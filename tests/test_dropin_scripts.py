"""Drop-in surface without the reference checkout: a v1.1 configuration from the committed zoo manifest
(tests/golden/zoo_manifest.json.gz, the `model:` section of the reference YAML) resolves to the tiling engine and takes the
tiling attributes exactly as scripts/inference_evaluate.py:144-150 sets them; the oracle's parameter table equals the
reference's state_dict (pinned in the golden fixtures), and compute_ssim equals the reference formula."""
import gzip
import json
import os

import pytest
import torch
import torch.nn.functional as F

from conftest import ROOT, golden_cases, load_golden

ZOO = json.load(gzip.open(os.path.join(ROOT, "tests", "golden", "zoo_manifest.json.gz"), "rt"))


def test_v11_config_resolves_to_the_tiling_engine():
    from vidtok_b200.compat_util import instantiate_from_config
    model = instantiate_from_config(ZOO["vidtok_v1_1/vidtok_kl_causal_488_16chn_v1_1.yaml"]["model"])
    # scripts/inference_evaluate.py:144-150
    assert hasattr(model, "use_tiling")
    model.use_tiling = True
    model.t_chunk_enc = 16
    model.t_chunk_dec = model.t_chunk_enc // model.encoder.time_downsample_factor
    model.use_overlap = True
    info = {"cls": type(model).__name__, "z": model.spec.z_channels, "interp": model.spec.interpolation_mode,
            "chunks": [list(c) for c in model.build_chunk_start_end(129)[:3]]}
    assert info == {"cls": "AutoencodingEngineV11", "z": 16, "interp": "trilinear", "chunks": [[0, 1], [1, 17], [17, 33]]}


@pytest.mark.parametrize("case", golden_cases())
def test_oracle_param_table_equals_reference_state_dict(case):
    from oracle.vidtok_oracle import cfg_from_model_yaml, reference_param_shapes
    d, meta = load_golden(case)   # meta["shapes"] = state_dict() shapes of the unmodified reference (oracle/make_golden.py)
    assert reference_param_shapes(cfg_from_model_yaml(meta["model"])) == {k: tuple(v) for k, v in meta["shapes"].items()}


def test_compute_ssim_matches_the_reference_formula():
    """vidtok/modules/util.py:157-178 stated directly (2-D 11x11 Gaussian window) vs the separable implementation."""
    from vidtok_b200.compat_util import compute_ssim
    g = torch.Generator().manual_seed(0)
    for shape in [(2, 3, 5, 64, 48), (1, 3, 2, 600, 520)]:   # the second exercises the avg-pool prefilter (f = 2)
        x = torch.rand(shape, generator=g)
        y = (x + 0.1 * torch.randn(shape, generator=g)).clamp(0, 1)
        a = x.permute(0, 2, 1, 3, 4).reshape(-1, 3, *shape[3:])
        b = y.permute(0, 2, 1, 3, 4).reshape(-1, 3, *shape[3:])
        f = max(1, round(min(shape[3:]) / 256))
        if f > 1:
            a, b = F.avg_pool2d(a, f), F.avg_pool2d(b, f)
        t = torch.arange(11, dtype=torch.float32) - 5.0
        k = torch.exp(-(t[None] ** 2 + t[:, None] ** 2) / (2 * 1.5 ** 2))
        k = (k / k.sum())[None, None].repeat(3, 1, 1, 1)
        blur = lambda v: F.conv2d(v, k, groups=3)  # noqa: E731
        mx, my = blur(a), blur(b)
        sxx, syy, sxy = blur(a * a) - mx * mx, blur(b * b) - my * my, blur(a * b) - mx * my
        cs = (2 * sxy + 0.03 ** 2) / (sxx + syy + 0.03 ** 2)
        ss = (2 * mx * my + 0.01 ** 2) / (mx * mx + my * my + 0.01 ** 2) * cs
        ref = ss.mean(dim=(-1, -2)).mean(1).mean(0)
        got = compute_ssim(x, y)
        assert abs(float(got) - float(ref)) < 2e-6, (float(got), float(ref))
        assert float(compute_ssim(x, x)) > 0.999999
