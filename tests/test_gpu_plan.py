"""-m gpu: the launch plans of a model depend on its geometry alone.

A workspace dry run plans every layer's kernel, fused epilogues included, from the geometry fixed when the model is built, so
the sizes it reports before vt_model_finalize are the sizes the finalized model runs with.  A decoder level at a channel
count without one N tile over Cout (192) plans its upsampling phase convolutions without the fused LayerNorm and normalises
after them."""
import ctypes as C
import gzip
import json
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

from conftest import golden_cases, load_golden, resolved_model_cfg  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ZOO = json.load(gzip.open(os.path.join(ROOT, "tests", "golden", "zoo_manifest.json.gz"), "rt"))
CONFIGS = ["golden/" + n for n in golden_cases()] + ["zoo/" + n for n in sorted(ZOO)]


def _config(name):
    from vidtok_b200.compat_util import instantiate_from_config
    kind, key = name.split("/", 1)
    if kind == "golden":
        _, meta = load_golden(key)
        B, _, T, H, W = meta["input"]
        return instantiate_from_config(resolved_model_cfg(meta)).spec, (B, T, H, W)
    return instantiate_from_config(ZOO[key]["model"]).spec, tuple(ZOO[key]["probe"])


def _finalize_synthetic(nm):
    from vidtok_b200.synth import synth_state_dict
    for k, v in synth_state_dict(dict(nm.manifest()), seed=0).items():
        nm.load(k, v.cuda())
    nm.finalize()


def _sizes(nm, spec, B, T, H, W):
    from vidtok_b200 import _native as N
    lib = N.lib()
    out = {}
    for prec in (N.PREC_FMA32, N.PREC_BF16, N.PREC_EXACT_TC, N.PREC_MIXED):
        out[("whole", prec)] = int(lib.vt_workspace_bytes(nm.handle, prec, B, T, H, W))
        if not spec.causal:
            continue
        _, Hz, Wz = nm.latent_shape(T, H, W)
        for dec, (h, w), chunks in ((0, (H, W), (1, 4, 17)), (1, (Hz, Wz), (1, 2))):
            st = C.c_void_p()
            N.check(lib.vt_chunk_state_create(nm.handle, prec, B, h, w, dec, 0, C.byref(st)))
            for tc in chunks:
                out[("chunk", prec, dec, tc)] = int(lib.vt_chunk_workspace_bytes(st, tc))
            lib.vt_chunk_state_destroy(st)
    return out


@pytest.mark.parametrize("name", CONFIGS)
def test_dry_run_sizes_do_not_change_with_finalize(name):
    from vidtok_b200.engine import NativeModel
    spec, (B, T, H, W) = _config(name)
    nm = NativeModel(spec)
    before = _sizes(nm, spec, B, T, H, W)
    _finalize_synthetic(nm)
    after = _sizes(nm, spec, B, T, H, W)
    assert all(v > 0 for v in after.values()), after
    assert before == after, {k: (before[k], after[k]) for k in before if before[k] != after[k]}


def test_layernorm_decoder_at_192_channels_normalises_after_the_phase_convs():
    from vidtok_b200 import _native as N
    from vidtok_b200.compat_util import compute_psnr
    from vidtok_b200.engine import NativeModel, TokenizerSpec
    from vidtok_b200.synth import synth_clip, synth_noise
    spec = TokenizerSpec(version=0, ch=64, ch_mult=(1, 2, 3), num_res_blocks=1, z_channels=4, double_z=True, norm_type="layernorm")
    nm = NativeModel(spec)
    _finalize_synthetic(nm)
    for prec in (N.PREC_BF16, N.PREC_EXACT_TC, N.PREC_MIXED):
        assert nm.lib.vt_workspace_bytes(nm.handle, prec, 1, 17, 64, 64) > 0, nm.lib.vt_last_error()
    x = synth_clip(1, 17, 64, 64).cuda()
    noise = synth_noise((1, 4) + nm.latent_shape(17, 64, 64)).cuda()
    dec = {}
    for prec in (N.PREC_FMA32, N.PREC_BF16):
        z, _, _, _ = nm.encode(x, noise, prec)
        dec[prec] = nm.decode(z, False, prec).cpu()
    torch.cuda.synchronize()
    ref, got = dec[N.PREC_FMA32], dec[N.PREC_BF16]
    assert got.shape == x.shape
    dmax, dmean = float((got - ref).abs().max()), float((got - ref).abs().mean())

    def psnr(y):
        return float(compute_psnr((x.cpu().clamp(-1, 1) + 1) / 2, (y.clamp(-1, 1) + 1) / 2))

    # the bf16 gate of test_gpu_model.py, against the fp32-FMA run
    assert abs(psnr(got) - psnr(ref)) <= 0.01 and dmax <= 0.25 and dmean <= 0.02, (psnr(got), psnr(ref), dmax, dmean)
