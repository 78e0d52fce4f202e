"""TEST INFRASTRUCTURE ONLY.  Walks every tokenizer YAML the reference ships (configs/*.yaml and configs/vidtok_v1_1/*.yaml:
causal / non-causal, KL / FSQ, 4x4x4 ... 8x8x8 ... 4x16x16 compression) and records, for each one,

  * the `model:` section (with the `${...}` interpolation of the decoder params resolved),
  * the checkpoint key -> shape table of the UNMODIFIED reference model (encoder.* / decoder.*),
  * the latent and reconstruction shapes the reference produces for a 1x3x17x64x64 clip,
  * the largest |reference - oracle| over latents and reconstruction on seeded weights (asserted <= 2e-5; FSQ indices equal),

into tests/golden/zoo_manifest.json.gz.  tests/test_zoo_cpu.py checks the engine's module tree, latent geometry and
workspace planning against it on any machine (the GPU box has no /root/reference), and regenerates the key tables when the
reference is present.

    python oracle/make_zoo_manifest.py
"""
import copy
import glob
import gzip
import json
import os
import sys

import torch
import yaml

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_shim  # noqa: E402
from oracle.vidtok_oracle import OracleModel, cfg_from_model_yaml  # noqa: E402
from vidtok_b200.synth import synth_clip, synth_state_dict  # noqa: E402

OUT = os.environ.get("VIDTOK_ZOO_OUT", os.path.join(ROOT, "tests", "golden", "zoo_manifest.json.gz"))
PROBE = (1, 17, 64, 64)   # B, T, H, W of the shape probe


def config_files():
    base = os.path.join(ref_shim.REFERENCE_ROOT, "configs")
    return sorted(glob.glob(os.path.join(base, "*.yaml")) + glob.glob(os.path.join(base, "vidtok_v1_1", "*.yaml")))


def model_section(path):
    cfg = yaml.safe_load(open(path))["model"]
    p = cfg["params"]
    if isinstance(p["decoder_config"].get("params"), str):   # ${model.params.encoder_config.params}
        p["decoder_config"]["params"] = copy.deepcopy(p["encoder_config"]["params"])
    p.pop("ckpt_path", None)
    p.pop("loss_config", None)    # training only (LPIPS / discriminator); the engines accept and skip it
    return cfg


def main(numerics=True):
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    out = {}
    for path in config_files():
        name = os.path.relpath(path, os.path.join(ref_shim.REFERENCE_ROOT, "configs"))
        my = model_section(path)
        ref = ref_shim.build_reference_model(copy.deepcopy(my))
        shapes = {k: list(v.shape) for k, v in ref.state_dict().items() if k.startswith(("encoder.", "decoder."))}
        rec = {"model": my, "shapes": shapes, "is_causal": bool(getattr(ref, "is_causal", True)), "engine": type(ref).__name__,
               "time_downsample_factor": int(ref.encoder.time_downsample_factor)}
        if numerics:
            sd = synth_state_dict({k: tuple(v) for k, v in shapes.items()}, seed=0)
            missing, unexpected = ref.load_state_dict(sd, strict=False)
            assert not unexpected, unexpected
            B, T, H, W = PROBE
            x = synth_clip(B, T, H, W, seed=1234)
            with torch.no_grad():
                torch.manual_seed(4321)
                z_ref, dec_ref, log_ref = ref(x)
            om = OracleModel(cfg_from_model_yaml(my), sd)
            torch.manual_seed(4321)
            z_o, dec_o, log_o = om.forward(x)
            dz = float((z_ref.double() - z_o.double()).abs().max())
            dd = float((dec_ref.double() - dec_o.double()).abs().max())
            assert tuple(z_ref.shape) == tuple(z_o.shape) and tuple(dec_ref.shape) == tuple(dec_o.shape), (name, z_ref.shape, z_o.shape)
            assert dz <= 2e-5 and dd <= 2e-5, (name, dz, dd)
            if "indices" in log_ref:
                assert torch.equal(log_ref["indices"], log_o["indices"]), name
            rec.update({"probe": list(PROBE), "z_shape": list(z_ref.shape), "dec_shape": list(dec_ref.shape),
                        "oracle_vs_reference": {"z": dz, "dec": dd}})
            print(f"{name}: {len(shapes)} tensors, z {tuple(z_ref.shape)}, dec {tuple(dec_ref.shape)}, oracle-vs-reference {dz:.1e} / {dd:.1e}")
        out[name] = rec
    with gzip.open(OUT, "wt") as f:
        json.dump(out, f, sort_keys=True)
    print("wrote", OUT, os.path.getsize(OUT), "bytes,", len(out), "configs")


if __name__ == "__main__":
    main()
