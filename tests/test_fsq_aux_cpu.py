"""The FSQ auxiliary loss without a GPU: the fp64 oracle (oracle/fsq_aux_oracle.py: fsq_aux_parts / fsq_aux_combine) against
the reference's values stored in tests/golden/fsq_aux (oracle/make_golden_fsq_aux.py), the entropy-weight annealing and
the regularizer's reference attributes."""
import glob
import json
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN_DIR

AUX_DIR = os.path.join(GOLDEN_DIR, "fsq_aux")
CASES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(AUX_DIR, "*.npz")))
COMPONENTS = ("per_sample_entropy", "codebook_entropy", "commit_loss", "aux_loss")


def load_aux(name):
    d = np.load(os.path.join(AUX_DIR, name + ".npz"))
    return d, json.loads(bytes(d["meta_json"]).decode())


def ref_bound(meta, k):
    """fp32 reference vs fp64 oracle: twice the deviation the recipe recorded, at least 1e-6 relative."""
    return max(2.0 * meta["deviation"][k], 1e-6)


def test_every_kind_of_case_is_present():
    kinds = {load_aux(c)[1]["kind"] for c in CASES}
    assert kinds == {"single", "tiled", "dist2"}, kinds
    assert {c for c in CASES if c.startswith("fix_")} == {"fix_tiny_fsq_v10", "fix_mid_fsq_v10", "fix_tiny_fsq_nc",
                                                          "fix_tiny_fsq_888_v11", "fix_cfg1_fsq_488_32768"}
    for digits in ("8888", "88888", "888888", "7555"):
        for kind in ("peaked", "encoder", "flat"):
            assert f"syn_{kind}_{digits}" in CASES


@pytest.mark.parametrize("case", CASES)
def test_oracle_matches_reference_fixture(case):
    from oracle.fsq_aux_oracle import fsq_aux_combine, fsq_aux_parts
    d, meta = load_aux(case)
    levels, w = meta["levels"], meta["weights"]
    if meta["kind"] == "single":
        got = {k: float(v) for k, v in fsq_aux_combine(*fsq_aux_parts(torch.from_numpy(d["h"]), levels), **w).items()}
        for k in COMPONENTS:
            assert abs(got[k] - meta["oracle"][k]) <= 1e-9 * abs(meta["oracle"][k]), (k, got[k], meta["oracle"][k])
            assert abs(got[k] - meta["reference"][k]) <= ref_bound(meta, k) * abs(got[k]), (k, got[k], meta["reference"][k])
    elif meta["kind"] == "tiled":
        chunks = [fsq_aux_combine(*fsq_aux_parts(torch.from_numpy(d[f"h{i}"]), levels), **w) for i in range(meta["n_chunks"])]
        aux = float(np.mean([float(c["aux_loss"]) for c in chunks]))
        assert abs(aux - meta["reference"]["aux_loss"]) <= ref_bound(meta, "aux_loss") * abs(aux)
    else:
        h = torch.from_numpy(d["h"])
        half = h.shape[0] // meta["world_size"]
        parts = [fsq_aux_parts(h[r * half:(r + 1) * half], levels) for r in range(meta["world_size"])]
        avg = sum(p[1] for p in parts) / meta["world_size"]
        for r, p in enumerate(parts):
            got = {k: float(v) for k, v in fsq_aux_combine(p[0], avg, p[2], **w).items()}
            for k in COMPONENTS:
                assert abs(got[k] - meta["reference_ranks"][r][k]) <= ref_bound(meta, k) * abs(got[k]), (r, k)


def _reference_weight(n_steps, weight, steps, factor):
    # regularizers.py:200-204
    if n_steps >= steps:
        return weight
    start = factor * weight
    return start - (n_steps / steps) * (start - weight)


@pytest.mark.parametrize("steps,factor", [(2000, 3), (2000, 1.2), (0, 3), (10, 1.0)])
def test_entropy_loss_weight_annealing(steps, factor):
    from vidtok_b200.engine import FSQRegularizer
    reg = FSQRegularizer([8, 8, 8, 8, 8], entropy_loss_weight=0.1, entropy_loss_annealing_steps=steps,
                         entropy_loss_annealing_factor=factor, commitment_loss_weight=0.25)
    for n in (0, 1, 7, 999, 1000, 1999, 2000, 5000):
        assert reg.calculate_entropy_loss_weight(n) == _reference_weight(n, 0.1, steps, factor)


def test_regularizer_keeps_reference_attributes():
    from vidtok_b200.engine import FSQRegularizer
    kw = dict(entropy_loss_weight=0.1, entropy_loss_annealing_steps=2000, entropy_loss_annealing_factor=3,
              commitment_loss_weight=0.25, diversity_gamma=0.7)
    reg = FSQRegularizer([8, 5, 5, 5], **kw)
    for k, v in kw.items():
        assert getattr(reg, k) == v, k
    assert reg.codebook_size == 1000 and reg.aux_enabled()
    assert not FSQRegularizer([8, 8, 8]).aux_enabled()   # the reference's defaults: both weights 0, aux_loss = 0
