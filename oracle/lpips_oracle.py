"""TEST INFRASTRUCTURE ONLY -- never imported by the product path (vidtok_b200/).

LPIPS with VGG16 (vidtok/modules/lpips.py) as plain functions, for the fixtures and the GPU tests:

  synthetic_lpips_state(seed)   every weight of the reference's state dict drawn from one explicit torch.Generator in sorted
                                key order, so any machine regenerates the same tensors (the trained VGG16 is 59 MB: not
                                committed, and not available offline)
  lpips_fp64(state, x, y)       the evaluation script's preprocessing in fp32 (clamp of y, (v+1)/2, *2-1), then ScalingLayer,
                                VGG16 features[0:30] and the head in float64; returns the per-frame total and the five layer
                                terms

The lin weights are |N(0, 1)| * LIN_SCALE, non-negative like the trained ones; LIN_SCALE puts the fixtures' LPIPS values in the
trained metric's usual range (0.025 to 0.30 for the three larger distortions of tests/golden/lpips, 0.0014 for the small one)
rather than the ~0.003 that torchvision's default initialisation gives.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

CONV_IDX = (0, 2, 5, 7, 10, 12, 14, 17, 19, 21, 24, 26, 28)
SLICE = (1, 1, 2, 2, 3, 3, 3, 4, 4, 4, 5, 5, 5)
COUT = (64, 64, 128, 128, 256, 256, 256, 512, 512, 512, 512, 512, 512)
CHNS = (64, 128, 256, 512, 512)
TAPS = (1, 3, 6, 9, 12)              # relu1_2 .. relu5_3 follow these convolutions
POOL_BEFORE = (2, 4, 7, 10)
SHIFT = (-0.030, -0.088, -0.188)
SCALE = (0.458, 0.448, 0.450)
LIN_SCALE = 0.5


def state_shapes() -> dict:
    """The reference's LPIPS keys (net.slice*, lin*) and their shapes."""
    shapes, ci = {}, 3
    for s, i, co in zip(SLICE, CONV_IDX, COUT):
        shapes[f"net.slice{s}.{i}.weight"] = (co, ci, 3, 3)
        shapes[f"net.slice{s}.{i}.bias"] = (co,)
        ci = co
    for k, c in enumerate(CHNS):
        shapes[f"lin{k}.model.1.weight"] = (1, c, 1, 1)
    return shapes


def synthetic_lpips_state(seed: int) -> dict:
    """fp32 CPU tensors for every key of state_shapes(), drawn in sorted key order: conv weights N(0, 2 / fan_in) (He), biases
    N(0, 0.01^2), lin weights |N(0, 1)| * LIN_SCALE."""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for key, shape in sorted(state_shapes().items()):
        v = torch.randn(shape, generator=g, dtype=torch.float32)
        if key.startswith("lin"):
            v = v.abs() * LIN_SCALE
        elif key.endswith(".weight"):
            v = v * (2.0 / (shape[1] * 9)) ** 0.5
        else:
            v = v * 0.01
        out[key] = v
    return out


def script_inputs(x: torch.Tensor, y: torch.Tensor):
    """scripts/inference_evaluate.py:175-186 in fp32: clamp the reconstruction, (v + 1) / 2, then * 2 - 1 at the LPIPS call."""
    x, y = x.float(), y.float().clamp(-1, 1)
    x, y = (x + 1) / 2, (y + 1) / 2
    return x * 2 - 1, y * 2 - 1


def _features(state, v):
    feats, h = [], v
    for n, (s, i) in enumerate(zip(SLICE, CONV_IDX)):
        if n in POOL_BEFORE:
            h = F.max_pool2d(h, 2, 2)
        w = state[f"net.slice{s}.{i}.weight"].to(v)
        b = state[f"net.slice{s}.{i}.bias"].to(v)
        h = F.relu(F.conv2d(h, w, b, padding=1))
        if n in TAPS:
            feats.append(h)
    return feats


def lpips_fp64(state: dict, x: torch.Tensor, y: torch.Tensor):
    """x, y: frames [N,3,H,W] (any float dtype, y not yet clamped).  Returns (total [N], per_layer [N,5]) in float64."""
    a, b = script_inputs(x, y)
    shift = torch.tensor(SHIFT, dtype=torch.float32).double().view(1, 3, 1, 1).to(a.device)
    scale = torch.tensor(SCALE, dtype=torch.float32).double().view(1, 3, 1, 1).to(a.device)
    a = (a.double() - shift) / scale
    b = (b.double() - shift) / scale
    fa, fb = _features(state, a), _features(state, b)
    terms = []
    for k in range(5):
        na = fa[k] / (torch.sqrt((fa[k] ** 2).sum(1, keepdim=True)) + 1e-10)
        nb = fb[k] / (torch.sqrt((fb[k] ** 2).sum(1, keepdim=True)) + 1e-10)
        w = state[f"lin{k}.model.1.weight"].double().to(na.device)
        terms.append(F.conv2d((na - nb) ** 2, w).mean((1, 2, 3)))
    per_layer = torch.stack(terms, 1)
    total = terms[0]
    for t in terms[1:]:
        total = total + t
    return total, per_layer
