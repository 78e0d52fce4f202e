"""Every tokenizer configuration the reference ships (23 YAMLs: causal / non-causal, KL / FSQ, 4x4x4 ... 8x8x8 ... 4x16x16, v1.0 / v1.1)
against the engine's host side, from the committed manifest tests/golden/zoo_manifest.json.gz (written by
oracle/make_zoo_manifest.py from the UNMODIFIED reference; the same run asserts oracle == reference to 2e-5 on each of them)."""
import gzip
import json
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
MANIFEST = os.path.join(ROOT, "tests", "golden", "zoo_manifest.json.gz")
ZOO = json.load(gzip.open(MANIFEST, "rt"))


def test_manifest_covers_the_reference_zoo():
    assert len(ZOO) == 23
    assert sum(1 for r in ZOO.values() if not r["is_causal"]) == 6
    assert sum(1 for n in ZOO if n.startswith("vidtok_v1_1/")) == 7
    for name, rec in ZOO.items():
        assert rec["oracle_vs_reference"]["z"] <= 2e-5 and rec["oracle_vs_reference"]["dec"] <= 2e-5, name


@pytest.mark.parametrize("name", sorted(ZOO))
def test_engine_module_tree_geometry_and_workspace_plan(name):
    from vidtok_b200 import _native as N
    from vidtok_b200.compat_util import instantiate_from_config
    from vidtok_b200.engine import NativeModel
    rec = ZOO[name]
    model = instantiate_from_config(rec["model"])
    # checkpoint keys and shapes == the reference's state_dict (encoder.* / decoder.*)
    sd = {k: list(v.shape) for k, v in model.state_dict().items()}
    assert sd == rec["shapes"]
    assert model.is_causal == rec["is_causal"]                                               # README.md:335
    assert model.encoder.time_downsample_factor == rec["time_downsample_factor"]             # inference_evaluate.py:142,149
    assert hasattr(model, "use_tiling") == name.startswith("vidtok_v1_1/")                   # how the scripts tell v1.1 apart
    # latent / reconstruction geometry of the native model == what the reference produced for the probe clip
    nm = NativeModel(model.spec)
    B, T, H, W = rec["probe"]
    assert list(nm.latent_shape(T, H, W)) == rec["z_shape"][2:]
    frames = nm.decoded_frames(rec["z_shape"][2])
    assert frames >= rec["dec_shape"][2]             # v1.0 causal: equal; v1.1: the engine trims to the last T_in frames
    if not name.startswith("vidtok_v1_1/"):
        assert frames == rec["dec_shape"][2]
    assert model.spec.z_channels == rec["z_shape"][1]
    # every layer of this geometry has a launch plan in every precision (vt_workspace_bytes is a dry run of the executor)
    for prec in (N.PREC_BF16, N.PREC_EXACT_TC, N.PREC_MIXED, N.PREC_FMA32):
        ws = N.lib().vt_workspace_bytes(nm.handle, prec, B, T, H, W)
        assert ws > 0, (name, prec, N.lib().vt_last_error())
