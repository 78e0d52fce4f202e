"""CPU-side checks of the C-ABI boundary: the library loads, exports every symbol the header declares, the
parameter manifest equals the reference's checkpoint keys/shapes (pinned in the golden fixtures), the dry-run
workspace query works, and the product path fails loudly without a GPU (no fallback)."""
import ctypes as C
import os
import re

import pytest
import torch

from conftest import ROOT, golden_cases, load_golden, resolved_model_cfg


def test_library_exports_every_declared_symbol():
    from vidtok_b200 import _native as N
    hdr = open(os.path.join(ROOT, "include", "vidtok_b200.h")).read()
    declared = set(re.findall(r"\b(vt_[a-z0-9_]+)\s*\(", hdr))
    assert len(declared) >= 25
    lib = C.CDLL(N.LIB_PATH)
    for name in sorted(declared):
        assert hasattr(lib, name), f"{name} declared in include/vidtok_b200.h but not exported"
    assert declared == set(N.EXPORTS), declared ^ set(N.EXPORTS)
    assert N.lib().vt_abi_version() == 3


@pytest.mark.parametrize("case", golden_cases())
def test_manifest_matches_reference_checkpoint_keys(case):
    from vidtok_b200.compat_util import instantiate_from_config
    d, meta = load_golden(case)
    model = instantiate_from_config(resolved_model_cfg(meta))
    sd = model.state_dict()
    ref = meta["shapes"]  # state_dict() shapes of the unmodified reference model (oracle/make_golden.py)
    assert set(sd.keys()) == set(ref.keys())
    for k, v in ref.items():
        assert tuple(sd[k].shape) == tuple(v), k
    want = "AutoencodingEngineV11" if "v1_1" in meta["model"]["target"] else "AutoencodingEngine"
    assert type(model).__name__ == want
    assert model.is_causal == ("noncausal" not in meta["model"]["params"]["encoder_config"]["target"])   # README.md:335
    tdf = meta["model"]["params"]["encoder_config"]["params"]["time_downsample_factor"]
    assert model.encoder.time_downsample_factor == tdf
    if "v1_1" in meta["model"]["target"]:
        assert hasattr(model, "use_tiling") and model.t_chunk_dec == model.t_chunk_enc // tdf and model.use_overlap is False


def test_engine_surface_and_state_dict_roundtrip():
    from vidtok_b200.compat_util import instantiate_from_config
    from vidtok_b200.synth import synth_state_dict
    d, meta = load_golden("tiny_fsq_v10")
    model = instantiate_from_config(resolved_model_cfg(meta))
    sd = synth_state_dict({k: tuple(v) for k, v in meta["shapes"].items()})
    extra = dict(sd)
    extra["loss.logvar"] = torch.zeros(())  # released checkpoints carry loss.* keys (autoencoder.py:164 strict=False)
    missing, unexpected = model.load_state_dict(extra, strict=False)
    assert not missing and unexpected == ["loss.logvar"]
    for k, v in model.state_dict().items():
        assert torch.equal(v, sd[k])
    assert model.regularization.codebook_size == 32768
    for attr in ("encode", "decode", "forward", "indices_to_latent", "init_from_ckpt"):
        assert callable(getattr(model, attr))
    # zero-initialised temporal conv2 at construction (model_3dcausal.py:460-462)
    fresh = instantiate_from_config(resolved_model_cfg(meta))
    assert float(fresh.encoder.down_temporal[0].block[0].conv2.conv.weight.abs().sum()) == 0.0
    assert float(fresh.decoder.up_temporal[1].upsample.mix_factor) == 2.0


def test_instantiate_from_config_errors_like_reference():
    from vidtok_b200.compat_util import instantiate_from_config
    with pytest.raises(KeyError):
        instantiate_from_config({"params": {}})
    assert instantiate_from_config("__is_first_stage__") is None


def test_latent_geometry_and_workspace_dry_run():
    from vidtok_b200 import _native as N
    from vidtok_b200.engine import NativeModel, TokenizerSpec
    spec = TokenizerSpec(version=0, ch=128, ch_mult=(1, 2, 4, 4), num_res_blocks=2, z_channels=4, double_z=True,
                         norm_type="layernorm")
    nm = NativeModel(spec)
    assert nm.latent_shape(17, 256, 256) == (5, 32, 32)   # 17 -> pad 20 -> 10 -> 5 (SURVEY.md section 3.1)
    assert nm.latent_shape(16, 256, 256) == (4, 32, 32)
    assert nm.decoded_frames(5) == 17 and nm.decoded_frames(4) == 13
    assert nm.spatial_factor() == 8
    ws_bf16 = N.lib().vt_workspace_bytes(nm.handle, N.PREC_BF16, 8, 17, 256, 256)
    ws_fp32 = N.lib().vt_workspace_bytes(nm.handle, N.PREC_FMA32, 8, 17, 256, 256)
    ws_x3 = N.lib().vt_workspace_bytes(nm.handle, N.PREC_EXACT_TC, 8, 17, 256, 256)
    ws_mix = N.lib().vt_workspace_bytes(nm.handle, N.PREC_MIXED, 8, 17, 256, 256)
    assert 4e9 < ws_bf16 < 40e9 and ws_bf16 < ws_fp32 < 80e9
    assert ws_bf16 < ws_x3 < 80e9 and ws_bf16 <= ws_mix <= ws_x3
    assert N.lib().vt_workspace_bytes(nm.handle, 7, 8, 17, 256, 256) == -1
    assert N.lib().vt_workspace_bytes(nm.handle, N.PREC_BF16, 1, 17, 250, 256) == -1
    assert b"multiples of 8" in N.lib().vt_last_error()
    spec11 = TokenizerSpec(version=1, ch=128, ch_mult=(1, 2, 4, 4), num_res_blocks=2, z_channels=16, double_z=True,
                           norm_type="layernorm", interpolation_mode="trilinear")
    n11 = NativeModel(spec11)
    assert n11.latent_shape(1, 256, 256) == (1, 32, 32)    # 1-frame first chunk padded to 4 (model_3dcausal_v1_1.py:755-760)
    assert n11.latent_shape(16, 256, 256) == (4, 32, 32)
    assert n11.latent_shape(17, 256, 256) == (5, 32, 32)
    assert n11.decoded_frames(5) == 20
    spec5 = TokenizerSpec(version=0, ch=128, ch_mult=(1, 2, 4, 4, 4), num_res_blocks=2, z_channels=4, double_z=True,
                          norm_type="layernorm")
    assert NativeModel(spec5).latent_shape(17, 512, 512) == (5, 32, 32)


def test_load_refusals_name_the_parameter():
    from vidtok_b200 import _native as N
    from vidtok_b200.engine import NativeModel, TokenizerSpec
    nm = NativeModel(TokenizerSpec(version=0, ch=128, ch_mult=(1, 2, 4, 4), num_res_blocks=2, z_channels=4, double_z=True,
                                   norm_type="layernorm"))
    buf = (C.c_float * 128)()
    assert N.lib().vt_model_load_param(nm.handle, b"encoder.conv_in.bias", buf, 128, 0, None) == -1
    assert N.lib().vt_last_error() == b"unknown parameter encoder.conv_in.bias"
    assert N.lib().vt_model_load_param(nm.handle, b"encoder.conv_in.conv.bias", buf, 127, 0, None) == -1
    assert N.lib().vt_last_error() == b"parameter encoder.conv_in.conv.bias: expected 128 elements, got 127"


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_product_path_fails_loudly_without_gpu():
    from vidtok_b200.compat_util import instantiate_from_config
    d, meta = load_golden("tiny_kl_v10")
    model = instantiate_from_config(resolved_model_cfg(meta))
    with pytest.raises(RuntimeError, match="CUDA"):
        model(torch.zeros(meta["input"]))
    with pytest.raises(RuntimeError, match="CUDA"):
        model.regularization(torch.zeros(1, 8, 5, 4, 4))
    from vidtok_b200 import _native as N
    from vidtok_b200.engine import NativeModel
    nm = NativeModel(model.spec)
    buf = (C.c_float * 4)()
    rc = N.lib().vt_model_load_param(nm.handle, b"encoder.conv_in.conv.bias", buf, 16, 0, None)
    assert rc == -5 and b"no CPU fallback" in N.lib().vt_last_error()
