"""-m gpu: I3D features and FVD on the device (vidtok_b200.metrics.I3D / i3d_features / fvd / Scorer(i3d=...)) against the
float64 restatement of oracle/i3d_oracle.py run on the device, with the seeded weights of synthetic_i3d_state(0): trained
weights are not available offline, so every accuracy statement here is about seeded weights.

End points are compared relative to the end point's max |fp64| value, features relative to their max |fp64| value.  Each test
prints what it saw.  On an H100 the exact mode's deviation grows with depth: 1.3e-6 after the stem, 2.1e-6 after Conv3d_2c,
4.8e-6 after Mixed_3c, 8.3e-6 after Mixed_4b, 1.9e-5 after Mixed_4f, 2.2e-5 to 2.6e-5 after Mixed_5c, and the features
reach 2.1e-5 to 2.4e-5 of their max.  Each Inception module adds a few 1e-6: the split-operand convolutions of conv_tc are
fp32-class per layer, and I3D stacks 22 of them on its longest path.  The bounds below are about twice what was seen; bf16 features deviate by 4.2e-3 to 4.7e-3."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from gpu_util import _p, stream  # noqa: E402
from oracle.i3d_oracle import fvd_fp64, i3d_fp64, synthetic_i3d_state  # noqa: E402
from vidtok_b200 import _native as N  # noqa: E402
from vidtok_b200.metrics import (I3D, I3D_ENDPOINTS, Scorer, features_to_stats, fvd, fvd_from_stats, i3d_features,  # noqa: E402
                                 i3d_stats_empty)

EXACT_ENDPOINT, EXACT_FEATURES, BF16_FEATURES = 6e-5, 5e-5, 3e-2
_MODELS = {}


def model(precision):
    if precision not in _MODELS:
        _MODELS[precision] = I3D.from_state_dict(synthetic_i3d_state(0), precision=precision)
    return _MODELS[precision]


def clips(B, T, H, W, seed, dtype=torch.float32):
    """smooth random clips in [-1,1] with a little noise: the spatial structure a video has"""
    g = torch.Generator().manual_seed(seed)
    coarse = torch.rand((B * 3, T, max(2, H // 32), max(2, W // 32)), generator=g) * 2 - 1
    x = F.interpolate(coarse, size=(H, W), mode="bilinear", align_corners=False).reshape(B, 3, T, H, W) * 0.8
    x = (x + 0.05 * torch.randn(x.shape, generator=g)).clamp(-1, 1)
    return x.to(dtype).cuda().contiguous()


def rel_to_max(got, want):
    got, want = got.double(), want.double().to(got.device)
    return float((got - want).abs().max() / want.abs().max().clamp_min(1e-30))


def oracle(x, chunk=2):
    st = synthetic_i3d_state(0)
    eps, feats = {}, []
    with torch.no_grad():
        for i in range(0, x.shape[0], chunk):
            e, f = i3d_fp64(st, x[i:i + chunk])
            for k, v in e.items():
                eps.setdefault(k, []).append(v)
            feats.append(f)
    return {k: torch.cat(v) for k, v in eps.items()}, torch.cat(feats)


@pytest.mark.parametrize("shape,dtype", [((2, 17, 256, 256), torch.float32), ((1, 16, 224, 224), torch.float32),
                                         ((1, 9, 224, 400), torch.float32), ((1, 17, 256, 256), torch.bfloat16),
                                         ((1, 17, 1080, 1920), torch.float32)])
def test_exact_end_points_and_features_against_fp64(shape, dtype):
    B, T, H, W = shape
    x = clips(B, T, H, W, seed=sum(shape), dtype=dtype)
    m = model("exact")
    ref_ep, ref_f = oracle(x)
    worst = 0.0
    for name in I3D_ENDPOINTS:
        got = m.endpoint(x, name)
        assert tuple(got.shape) == tuple(ref_ep[name].shape), name
        e = rel_to_max(got, ref_ep[name])
        print(f"{shape} {dtype} {name}: {e:.2e}")
        worst = max(worst, e)
        assert e <= EXACT_ENDPOINT, f"{name} deviates by {e:.2e} of its max"
    f = i3d_features(m, x)
    ef = rel_to_max(f, ref_f)
    print(f"{shape} {dtype} features: {ef:.2e} (worst end point {worst:.2e}); feature spread {float(ref_f.std()):.3f}")
    assert ef <= EXACT_FEATURES


@pytest.mark.parametrize("shape", [(2, 17, 256, 256), (1, 17, 1080, 1920)])
def test_bf16_features_against_fp64(shape):
    B, T, H, W = shape
    x = clips(B, T, H, W, seed=7 + sum(shape))
    _, ref_f = oracle(x)
    e = rel_to_max(i3d_features(model("bf16"), x), ref_f)
    print(f"bf16 {shape}: features {e:.2e} of their max")
    assert e <= BF16_FEATURES


def _distort(x, seed):
    g = torch.Generator().manual_seed(seed)
    B, Cc, T, H, W = x.shape
    k = torch.tensor([1.0, 2.0, 1.0], dtype=torch.float32)
    k2 = (k[:, None] * k[None, :] / 16).to(x.device)[None, None].expand(Cc, 1, 3, 3)
    blurred = F.conv2d(x.transpose(1, 2).reshape(B * T, Cc, H, W), k2, padding=1, groups=Cc)
    y = blurred.reshape(B, T, Cc, H, W).transpose(1, 2) + 0.1 * torch.randn(x.shape, generator=g).to(x.device)
    return y.clamp(-1, 1).contiguous()


def test_fvd_against_fp64_and_the_scorer():
    x = clips(24, 9, 224, 224, seed=100)
    y = _distort(x, seed=101)
    m = model("exact")
    _, fx64 = oracle(x, chunk=4)
    _, fy64 = oracle(y, chunk=4)
    want = fvd_fp64(fx64, fy64)
    fx, fy = i3d_features(m, x), i3d_features(m, y)
    got = fvd(fx, fy)
    print(f"FVD device {got:.6f} fp64 {want:.6f} rel {abs(got - want) / abs(want):.2e}")
    assert abs(got - want) <= 1e-4 * abs(want)
    sx = features_to_stats(fx)
    zero = fvd_from_stats(sx, sx)
    trace = float(torch.cov(fx.double().T).trace())
    print(f"FVD(X, X) = {zero:.3e}, tr S = {trace:.3e}")
    assert abs(zero) <= 1e-9 * trace

    # three uneven updates give the bits of one update, without a host synchronisation before result()
    one, three = Scorer(i3d=m), Scorer(i3d=m)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        one.update(x, y)
        for a, b in ((0, 5), (5, 6), (6, 24)):
            three.update(x[a:b], y[a:b])
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert torch.equal(one.fvd_sums(), three.fvd_sums())
    r = three.result()
    print(f"scorer {r}")
    assert r["fvd_clips"] == 24 and abs(r["fvd"] - got) <= 1e-9 * abs(got)
    dev = i3d_stats_empty("cuda")
    i3d_features(m, x, stats=dev)
    assert torch.equal(dev.cpu(), one.fvd_sums()[0].cpu())
    assert torch.allclose(dev.cpu(), features_to_stats(fx).cpu(), rtol=1e-12, atol=1e-9)


def test_scorer_windows():
    m = model("bf16")
    x = clips(2, 20, 64, 64, seed=5)
    y = _distort(x, seed=6)
    s = Scorer(i3d=m, fvd_frames=9)
    s.update(x, y)
    want = i3d_features(m, x[:, :, :18].reshape(2, 3, 2, 9, 64, 64).transpose(1, 2).reshape(4, 3, 9, 64, 64).contiguous())
    assert torch.allclose(s.fvd_sums()[0].cpu(), features_to_stats(want).cpu(), rtol=1e-12, atol=1e-9)
    assert s.result()["fvd_clips"] == 4


@pytest.mark.parametrize("precision", ["exact", "bf16"])
def test_features_do_not_depend_on_the_pass_or_the_workspace(precision):
    m = model(precision)
    x = clips(10, 9, 96, 128, seed=11)          # two passes of 8 and 2 clips
    assert m.pass_clips(9, 96, 128) == 8
    full = i3d_features(m, x)
    again = i3d_features(m, x)
    alone = torch.cat([i3d_features(m, x[i:i + 1]) for i in (0, 9)])
    pair = i3d_features(m, x[8:10])
    ws = torch.full((m._workspace_bytes(tuple(x.shape)) // 4,), float("nan"), device="cuda")
    nan_ws = m._launch(x, None, ws.view(torch.uint8))
    torch.cuda.synchronize()
    assert torch.equal(full, again)
    assert torch.equal(alone, full[[0, 9]])
    assert torch.equal(pair, full[8:10])
    assert torch.equal(nan_ws, full)
    assert bool(torch.isfinite(full).all())


def test_abi_errors():
    m = model("bf16")
    lib = N.lib()
    x = torch.zeros(1, 3, 9, 32, 32, device="cuda")
    out = torch.zeros(1, 400, device="cuda")
    need = lib.vt_i3d_workspace_bytes(m._h, N.PREC_BF16, 1, 3, 9, 32, 32)
    assert need > 0
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    s = stream()

    def call(prec=N.PREC_BF16, C_=3, T=9, nbytes=need, h=m._h):
        lib.vt_launch_count(1)
        rc = lib.vt_i3d_features(h, prec, _p(x), 0, 1, C_, T, 32, 32, _p(out), None, _p(ws), nbytes, s)
        return rc, lib.vt_launch_count(0)

    rc, launched = call()
    assert rc == 0 and launched > 0
    for kw in ({"T": 8}, {"C_": 4}, {"prec": N.PREC_FMA32}, {"prec": N.PREC_MIXED}):
        assert call(**kw) == (-1, 0), kw
    assert call(nbytes=need - 1) == (-4, 0)
    assert lib.vt_i3d_workspace_bytes(m._h, N.PREC_BF16, 1, 3, 8, 32, 32) == -1
    with pytest.raises(RuntimeError):
        i3d_features(m, x.cpu())
    with pytest.raises(ValueError):
        i3d_features(m, x[:, :, :8].contiguous())
    h = C.c_void_p()
    N.check(lib.vt_i3d_create(0, C.byref(h)))
    try:
        assert call(h=h)[0] == -3
        assert lib.vt_i3d_finalize(h, s) == -3
    finally:
        lib.vt_i3d_destroy(h)
