import json
import os
import sys
import warnings

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
warnings.filterwarnings("ignore")

GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA (sm_90a, H100) device; run on an H100 machine with -m gpu")
    # make sure the CUDA library exists before anything imports it (nvcc cross-compiles without a GPU)
    import __graft_entry__ as ge
    ge.build()


def load_golden(name):
    d = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
    meta = json.loads(bytes(d["meta_json"]).decode())
    return d, meta


def golden_cases(prefix=None):
    names = sorted(f[:-4] for f in os.listdir(GOLDEN_DIR) if f.endswith(".npz"))
    return [n for n in names if prefix is None or n.startswith(prefix)]


def resolved_model_cfg(meta):
    import copy
    cfg = copy.deepcopy(meta["model"])
    cfg["params"]["decoder_config"]["params"] = copy.deepcopy(cfg["params"]["encoder_config"]["params"])
    return cfg


def synth_inputs(meta, d):
    import torch
    from vidtok_b200.synth import synth_clip
    B, _, T, H, W = meta["input"]
    x = synth_clip(B, T, H, W, seed=meta["input_seed"])
    assert abs(float(x.double().abs().sum()) - float(d["x_absum"])) < 1e-6 * float(d["x_absum"]), "input RNG differs from the fixture"
    if "x" in d:
        assert torch.equal(x, torch.from_numpy(d["x"]))
    return x


def synth_weights(meta, d):
    from vidtok_b200.synth import synth_state_dict, weights_fingerprint
    sd = synth_state_dict({k: tuple(v) for k, v in meta["shapes"].items()}, seed=meta["weights_seed"])
    fp = weights_fingerprint(sd)
    assert abs(fp - float(d["w_fingerprint"])) < 1e-9 * fp, "weight RNG differs from the fixture"
    return sd
