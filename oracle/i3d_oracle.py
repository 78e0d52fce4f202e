"""The FVD definition of vidtok_b200.metrics restated in torch.nn.functional: seeded I3D weights, the preprocessing, the network in
float64 with every end point, and the Frechet distance.  Test infrastructure only.

The reference reports FVD but ships no code for it, so there is nothing to pin a fixture against: this file *is* the
definition the library's kernels are tested against (VideoGPT's fvd module, TF-GAN's Frechet distance, the PyTorch port's
InceptionI3d layout).  It runs on whatever device the clips are on; pass "meta" tensors to get the end-point shapes alone."""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from vidtok_b200.metrics import I3D_ENDPOINTS, _I3D_MODULES, i3d_state_shapes

SIZE = 224


def synthetic_i3d_state(seed: int = 0) -> dict:
    """Every key of i3d_state_shapes() drawn in sorted order from one torch.Generator: He-initialised conv weights, BatchNorm
    statistics around the identity (gamma ~ 1, running_var ~ 1 +- 0.2, small means), and logits weights scaled so that the
    features spread by O(1)."""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for key, shape in sorted(i3d_state_shapes().items()):
        if key == "logits.conv3d.weight":
            v = torch.randn(shape, generator=g) * (4.0 / math.sqrt(shape[1]))
        elif key == "logits.conv3d.bias":
            v = torch.randn(shape, generator=g) * 0.1
        elif key.endswith("conv3d.weight"):
            fan_in = shape[1] * shape[2] * shape[3] * shape[4]
            v = torch.randn(shape, generator=g) * math.sqrt(2.0 / fan_in)
        elif key.endswith("bn.weight"):
            v = 1.0 + 0.1 * torch.randn(shape, generator=g)
        elif key.endswith("bn.bias"):
            v = 0.1 * torch.randn(shape, generator=g)
        elif key.endswith("running_mean"):
            v = 0.05 * torch.randn(shape, generator=g)
        else:
            v = 1.0 + 0.2 * (2 * torch.rand(shape, generator=g) - 1)
        out[key] = v.float()
    return out


def resized_size(H: int, W: int) -> tuple:
    """Short side 224, long side ceil(long * 224 / short)."""
    if H <= W:
        return SIZE, math.ceil(W * SIZE / H)
    return math.ceil(H * SIZE / W), SIZE


def preprocess(clips: torch.Tensor) -> torch.Tensor:
    """[B,3,T,H,W] in [-1,1] (any float dtype) -> fp32 [B,3,T,224,224]: clamp, (v+1)/2, F.interpolate bilinear
    (align_corners=False, no antialias) to resized_size, centre crop, (v-0.5)*2."""
    B, C, T, H, W = clips.shape
    v = (clips.float().clamp(-1, 1) + 1) / 2
    v = v.transpose(1, 2).reshape(B * T, C, H, W)
    h, w = resized_size(H, W)
    v = F.interpolate(v, size=(h, w), mode="bilinear", align_corners=False)
    oh, ow = (h - SIZE) // 2, (w - SIZE) // 2
    v = v[:, :, oh:oh + SIZE, ow:ow + SIZE]
    v = (v - 0.5) * 2
    return v.reshape(B, T, C, SIZE, SIZE).transpose(1, 2)


def _same_pad(x: torch.Tensor, k, s) -> torch.Tensor:
    pads = []
    for n, kk, ss in zip(x.shape[2:], k, s):
        pad = max(kk - ss, 0) if n % ss == 0 else max(kk - n % ss, 0)
        pads.append((pad // 2, pad - pad // 2))
    (t0, t1), (h0, h1), (w0, w1) = pads
    return F.pad(x, (w0, w1, h0, h1, t0, t1))


def _unit(x, sd, key, k, s=1):
    x = _same_pad(x, (k,) * 3, (s,) * 3)
    x = F.conv3d(x, sd[f"{key}.conv3d.weight"], stride=s)
    x = F.batch_norm(x, sd[f"{key}.bn.running_mean"], sd[f"{key}.bn.running_var"], sd[f"{key}.bn.weight"], sd[f"{key}.bn.bias"],
                     training=False, eps=1e-3)
    return F.relu(x)


def _pool(x, k, s):
    return F.max_pool3d(_same_pad(x, k, s), k, s)


def i3d_fp64(state: dict, clips: torch.Tensor):
    """(end points {name: float64 [B,C,T,H,W]}, features float64 [B,400]) of clips [B,3,T,H,W], T >= 9: preprocess in fp32,
    then the network in float64 on the clips' device."""
    if clips.shape[2] < 9:
        raise ValueError(f"I3D needs clips of at least 9 frames, got T = {clips.shape[2]}")
    sd = {k: v.to(clips.device, torch.float64) for k, v in state.items()}
    x = preprocess(clips).double()
    ep = {}
    x = _unit(x, sd, "Conv3d_1a_7x7", 7, 2); ep["Conv3d_1a_7x7"] = x
    x = _pool(x, (1, 3, 3), (1, 2, 2)); ep["MaxPool3d_2a_3x3"] = x
    x = _unit(x, sd, "Conv3d_2b_1x1", 1); ep["Conv3d_2b_1x1"] = x
    x = _unit(x, sd, "Conv3d_2c_3x3", 3); ep["Conv3d_2c_3x3"] = x
    x = _pool(x, (1, 3, 3), (1, 2, 2)); ep["MaxPool3d_3a_3x3"] = x
    for name, _ in _I3D_MODULES:
        if name == "Mixed_4b":
            x = _pool(x, (3, 3, 3), (2, 2, 2)); ep["MaxPool3d_4a_3x3"] = x
        if name == "Mixed_5b":
            x = _pool(x, (2, 2, 2), (2, 2, 2)); ep["MaxPool3d_5a_2x2"] = x
        b0 = _unit(x, sd, f"{name}.b0", 1)
        b1 = _unit(_unit(x, sd, f"{name}.b1a", 1), sd, f"{name}.b1b", 3)
        b2 = _unit(_unit(x, sd, f"{name}.b2a", 1), sd, f"{name}.b2b", 3)
        b3 = _unit(_pool(x, (3, 3, 3), (1, 1, 1)), sd, f"{name}.b3b", 1)
        x = torch.cat([b0, b1, b2, b3], dim=1)
        ep[name] = x
    assert tuple(ep) == I3D_ENDPOINTS
    x = F.avg_pool3d(x, (2, 7, 7), stride=1)
    x = F.conv3d(x, sd["logits.conv3d.weight"], sd["logits.conv3d.bias"])
    feats = x.squeeze(4).squeeze(3).mean(2)
    return ep, feats


def fvd_fp64(features_a: torch.Tensor, features_b: torch.Tensor) -> float:
    """FVD of two feature sets [n,400] in float64: unbiased covariances of the centred sets, tr((S1^1/2 S2 S1^1/2)^1/2) from
    eigh with eigenvalues clamped at 0 and those beyond the covariances' rank (n - 1) dropped."""
    def stats(f):
        f = f.detach().cpu().double()
        mu = f.mean(0)
        d = f - mu
        return mu, d.T @ d / (f.shape[0] - 1), f.shape[0] - 1

    def eig(a, rank):
        w, v = torch.linalg.eigh((a + a.T) / 2)
        w = w.clamp(min=0)
        w[: max(w.numel() - rank, 0)] = 0
        return w, v

    (m1, s1, r1), (m2, s2, r2) = stats(features_a), stats(features_b)
    w, v = eig(s1, r1)
    r = (v * w.sqrt()) @ v.T
    tr = eig(r @ s2 @ r, min(r1, r2))[0].sqrt().sum()
    return float(((m1 - m2) ** 2).sum() + s1.trace() + s2.trace() - 2 * tr)
