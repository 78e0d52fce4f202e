"""-m gpu: op-level parity of the variants the tensor-core modes actually run (VERDICT r1 "make the fast path's tests
bite"): every fused epilogue, padding mode and weight transformation of conv_tc / conv_stem / the attention core,
in BOTH tensor-core precisions, against fp64 torch statements of the reference op:

  * BF16     -- operands rounded to bf16 first; bound 2^-7*|ref| + 2e-2 (bf16 output rounding + fp32 accumulation)
  * EXACT_TC -- fp32 operands as hi|lo fp16 planes (11 + 11 mantissa bits; three MMAs hi*hi + lo*hi + hi*lo per K step);
                bound 4e-5*(1 + |ref|): fp32-class, three orders of magnitude below bf16 rounding, so a silent bf16 path or a
                wrong gamma/beta slice cannot pass.  (A first version with bf16 planes measured 2e-5 .. 2.3e-4 here and
                3e-4 on model latents -- too coarse for bit-exact FSQ codes -- hence fp16 planes.)

Reference lines: model_3dcausal.py:62-80 (LayerNorm), :26-27 (SiLU), :193-197 (CausalConv3d), :208-212 (Upsample),
:267-273 (TimeUpsampleResCausal2x), :139-140 (attention); model_3dcausal_v1_1.py:216-236 (replicate / cache padding).
"""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from vidtok_b200 import _native as N  # noqa: E402

PRECS = [N.PREC_BF16, N.PREC_EXACT_TC]
PIDS = ["bf16", "exact_tc"]
X3_TOL = 4e-5


def rnd(*shape, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g) * scale


def prep(t, precision):
    """operand values as the kernel sees them"""
    return t.to(torch.bfloat16).float() if precision == N.PREC_BF16 else t


def check(got, ref, precision, what="", slack=1.0):
    assert got.shape == ref.shape, (got.shape, ref.shape)
    err = (got.double() - ref.double()).abs()
    if precision == N.PREC_BF16:
        tol = slack * (2.0 ** -7 * ref.abs().double() + 2e-2)
    else:
        tol = slack * X3_TOL * (1.0 + ref.abs().double())
    worst = float((err / tol).max())
    assert worst <= 1.0, f"{what}: max err {float(err.max()):.3e} (x{worst:.1f} the bound) at ref {float(ref.flatten()[(err / tol).argmax()]):.4f}"
    return float(err.max())


def conv3d_ref(x, w, b, stride=(1, 1, 1), pads=None, front=None):
    """causal conv in fp64; `front` = frames placed in front of x instead of zeros (replicate / cache padding)"""
    kt, kh, kw = w.shape[2:]
    tp = (kt - 1) + (1 - stride[0])
    if pads is None:
        hp, wp = (kh - 1) + (1 - stride[1]), (kw - 1) + (1 - stride[2])
        pads = (hp // 2, hp - hp // 2, wp // 2, wp - wp // 2)
    x = x.double()
    if front is not None:
        x = torch.cat([front.double(), x], dim=2)
        x = F.pad(x, (pads[2], pads[3], pads[0], pads[1], 0, 0))
    else:
        x = F.pad(x, (pads[2], pads[3], pads[0], pads[1], tp, 0))
    return F.conv3d(x, w.double(), b.double(), stride=stride)


def ln_ref(v, g, b, silu):
    """LayerNorm over channels of [B,C,T,H,W], eps 1e-6, optional x*sigmoid(x)"""
    y = F.layer_norm(v.double().permute(0, 2, 3, 4, 1), (v.shape[1],), g.double(), b.double(), eps=1e-6).permute(0, 4, 1, 2, 3)
    return y * torch.sigmoid(y) if silu else y


# ---------------------------------------------------------------------------------------------------------------
# plain geometries in EXACT_TC (the BF16 versions are tests/test_gpu_ops.py::test_conv_tc)
# ---------------------------------------------------------------------------------------------------------------
X3_CASES = [
    # name, Ci, Co, k, stride, (B,T,H,W), res_mode
    ("k333", 64, 64, (3, 3, 3), (1, 1, 1), (1, 3, 16, 16), 0),
    ("k133_n256", 128, 256, (1, 3, 3), (1, 1, 1), (1, 2, 32, 32), 0),
    ("k311_res", 64, 128, (3, 1, 1), (1, 1, 1), (1, 5, 8, 16), 1),
    ("k111_two_ntiles", 256, 512, (1, 1, 1), (1, 1, 1), (2, 1, 16, 16), 0),
    ("partial_tiles_n96", 64, 96, (1, 3, 3), (1, 1, 1), (1, 2, 12, 20), 0),
    ("tstride_avgpool", 64, 64, (3, 3, 3), (2, 1, 1), (2, 6, 16, 16), 3),
    ("many_tiles_res", 64, 64, (3, 3, 3), (1, 1, 1), (2, 4, 64, 64), 1),
    ("k333_c512_res", 512, 512, (3, 3, 3), (1, 1, 1), (1, 3, 16, 16), 1),
    ("halo_res", 64, 128, (1, 3, 3), (1, 1, 1), (1, 5, 128, 128), 1),
    ("halo_k233_n256", 128, 256, (2, 3, 3), (1, 1, 1), (1, 3, 128, 128), 0),
]


@pytest.mark.parametrize("case", X3_CASES, ids=[c[0] for c in X3_CASES])
def test_conv_exact_tc(case):
    from gpu_util import op_conv
    _, Ci, Co, k, stride, (B, T, H, W), res_mode = case
    K = Ci * k[0] * k[1] * k[2]
    x, w, b = rnd(B, Ci, T, H, W, seed=1), rnd(Co, Ci, *k, seed=2, scale=1 / math.sqrt(K)), rnd(Co, seed=3)
    conv = conv3d_ref(x, w, b, stride)
    alpha, res = 0.6, None
    if res_mode == 1:
        res = rnd(*conv.shape, seed=4)
        ref = res.double() + conv
    elif res_mode == 3:
        res = x
        ref = alpha * F.avg_pool3d(F.pad(x.double(), (0, 0, 0, 0, 1, 0)), (3, 1, 1), stride=(2, 1, 1)) + (1 - alpha) * conv
    else:
        ref = conv
    got = op_conv(x, w, b, stride=stride, res=res, res_mode=res_mode, alpha=alpha, precision=N.PREC_EXACT_TC)
    e = check(got, ref, N.PREC_EXACT_TC, case[0])
    print(f"[{case[0]}] exact_tc max err {e:.2e}")
    # the FMA kernel reading the same hi|lo operands agrees to fp32 rounding
    simt = op_conv(x, w, b, stride=stride, res=res, res_mode=res_mode, alpha=alpha, precision=N.PREC_EXACT_TC, force_simt=True)
    check(simt, ref, N.PREC_EXACT_TC, case[0] + " (fma on split operands)")


def test_conv_exact_tc_downsample_stride2():
    from gpu_util import op_conv
    for (B, T, H, W, Ci, Co) in [(1, 2, 32, 32, 64, 64), (2, 3, 64, 32, 128, 128)]:
        x, w, b = rnd(B, Ci, T, H, W, seed=1), rnd(Co, Ci, 1, 3, 3, seed=2, scale=1 / math.sqrt(9 * Ci)), rnd(Co, seed=3)
        ref = conv3d_ref(x, w, b, (1, 2, 2), pads=(0, 1, 0, 1))
        got = op_conv(x, w, b, stride=(1, 2, 2), pads=(0, 1, 0, 1), precision=N.PREC_EXACT_TC)
        check(got, ref, N.PREC_EXACT_TC, "downsample")


# ---------------------------------------------------------------------------------------------------------------
# LayerNorm(+SiLU) fused into the epilogue
# ---------------------------------------------------------------------------------------------------------------
LN_CASES = [
    # name, Ci, Co, k, (B,T,H,W), ln_mode, silu, residual
    ("ln1_c128_k133", 128, 128, (1, 3, 3), (1, 2, 32, 32), 1, True, False),     # conv1 -> norm2 of a ResnetBlock
    ("ln1_c256_k311", 256, 256, (3, 1, 1), (1, 4, 16, 16), 1, True, False),
    ("ln2_c128_k133_res", 128, 128, (1, 3, 3), (1, 2, 32, 32), 2, True, True),  # conv2 + skip -> next block's norm1
    ("ln2_c256_k311_res", 256, 256, (3, 1, 1), (2, 3, 16, 16), 2, True, True),
    ("ln2_c256_nosilu", 128, 256, (1, 1, 1), (1, 2, 16, 16), 2, False, False),  # -> attention norm (no SiLU)
    ("ln2_c128_halo_res", 128, 128, (1, 3, 3), (1, 3, 128, 128), 2, True, True),  # halo windows, residual through the MMA
    ("ln1_c64", 64, 64, (3, 3, 3), (1, 3, 16, 16), 1, True, False),
]


@pytest.mark.parametrize("precision", PRECS, ids=PIDS)
@pytest.mark.parametrize("case", LN_CASES, ids=[c[0] for c in LN_CASES])
def test_conv_fused_layernorm(case, precision):
    from gpu_util import op_conv_ex
    _, Ci, Co, k, (B, T, H, W), ln_mode, silu, with_res = case
    K = Ci * k[0] * k[1] * k[2]
    x = prep(rnd(B, Ci, T, H, W, seed=1), precision)
    w = prep(rnd(Co, Ci, *k, seed=2, scale=1 / math.sqrt(K)), precision)
    b = rnd(Co, seed=3)
    # distinct gamma/beta per channel: a shifted or truncated slice fails
    g = 1.0 + 0.5 * rnd(Co, seed=5)
    bt = 0.3 * rnd(Co, seed=6) + torch.linspace(-0.5, 0.5, Co)
    v = conv3d_ref(x, w, b)
    res = None
    if with_res:
        res = prep(rnd(*v.shape, seed=4), precision)
        v = v + res.double()
    y = ln_ref(v, g, bt, silu)
    out, out2 = op_conv_ex(x, w, b, precision=precision, res=res, res_mode=1 if with_res else 0, ln_mode=ln_mode, ln_silu=silu,
                           gamma=g, beta=bt)
    if ln_mode == 1:
        check(out, y, precision, case[0] + " act(LN(v))", slack=1.5)
    else:
        check(out, v, precision, case[0] + " v")
        check(out2, y, precision, case[0] + " act(LN(v))", slack=1.5)


# ---------------------------------------------------------------------------------------------------------------
# v1.1 time padding: replicated first frame / cache of the previous chunk
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", PRECS, ids=PIDS)
@pytest.mark.parametrize("k", [(3, 1, 1), (3, 3, 3)], ids=["k311", "k333"])
def test_conv_v11_time_padding(k, precision):
    from gpu_util import op_conv_ex
    B, Ci, Co, T, H, W = 2, 64, 64, 4, 16, 16
    K = Ci * k[0] * k[1] * k[2]
    x = prep(rnd(B, Ci, T, H, W, seed=1), precision)
    w = prep(rnd(Co, Ci, *k, seed=2, scale=1 / math.sqrt(K)), precision)
    b = rnd(Co, seed=3)
    # first chunk: x[:, :, :1] repeated time_pad times (model_3dcausal_v1_1.py:219-221)
    ref1 = conv3d_ref(x, w, b, front=x[:, :, :1].repeat(1, 1, 2, 1, 1))
    got1, _ = op_conv_ex(x, w, b, precision=precision, t_mode=1)
    check(got1, ref1, precision, "replicate")
    # later chunks: the cached tail of the previous chunk's padded input (:223-226)
    cache = prep(rnd(B, Ci, 2, H, W, seed=9), precision)
    ref2 = conv3d_ref(x, w, b, front=cache)
    got2, _ = op_conv_ex(x, w, b, precision=precision, t_mode=2, cache=cache)
    check(got2, ref2, precision, "cache")
    # and the zero-padded v1.0 result differs from both (the modes are not aliases of each other)
    ref0 = conv3d_ref(x, w, b)
    assert float((ref0 - ref1).abs().max()) > 0.1 and float((ref1 - ref2).abs().max()) > 0.1


@pytest.mark.parametrize("precision", PRECS, ids=PIDS)
def test_conv_v11_time_downsample_cache(precision):
    """TimeDownsampleResCausal2x in v1.1 (model_3dcausal_v1_1.py:289-302): conv cache 1 frame... here time_pad = 1 for the
    stride-2 conv, avg-pool branch front-padded with frame 0 (first chunk) or a 1-frame cache."""
    from gpu_util import op_conv_ex
    B, C_, T, H, W = 1, 64, 6, 16, 16
    alpha = 0.7
    x = prep(rnd(B, C_, T, H, W, seed=1), precision)
    w = prep(rnd(C_, C_, 3, 3, 3, seed=2, scale=1 / math.sqrt(27 * C_)), precision)
    b = rnd(C_, seed=3)

    def ref(front_conv, front_pool):
        conv = conv3d_ref(x, w, b, (2, 1, 1), front=front_conv)
        pool = F.avg_pool3d(torch.cat([front_pool.double(), x.double()], dim=2), (3, 1, 1), stride=(2, 1, 1))
        return alpha * pool + (1 - alpha) * conv

    got, _ = op_conv_ex(x, w, b, precision=precision, stride=(2, 1, 1), res=x, res_mode=3, alpha=alpha, t_mode=1, res_t_mode=1)
    check(got, ref(x[:, :, :1], x[:, :, :1]), precision, "first chunk")
    cache = prep(rnd(B, C_, 1, H, W, seed=8), precision)
    got, _ = op_conv_ex(x, w, b, precision=precision, stride=(2, 1, 1), res=x, res_mode=3, alpha=alpha, t_mode=2, cache=cache,
                        res_t_mode=2)
    check(got, ref(cache, cache), precision, "cached")


# ---------------------------------------------------------------------------------------------------------------
# stem, heads
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", PRECS, ids=PIDS)
@pytest.mark.parametrize("t_rep", [0, 3])
def test_conv_stem_kernel(precision, t_rep):
    """encoder conv_in 3 -> 128 on conv_stem_kernel from the caller's fp32 NCDHW tensor; t_rep: the encoder's replicated
    leading frames (model_3dcausal.py:685-689)"""
    from gpu_util import _p, empty_act, from_act, ncdhw, stream
    B, Ci, Co, T, H, W = 2, 3, 128, 5, 24, 40      # H, W not multiples of the 8x16 tile
    x = prep(rnd(B, Ci, T, H, W, seed=1), precision)
    w = prep(rnd(Co, Ci, 3, 3, 3, seed=2, scale=1 / math.sqrt(81)), precision)
    b = rnd(Co, seed=3)
    xp = torch.cat([x[:, :, :1].repeat(1, 1, t_rep, 1, 1), x], dim=2) if t_rep else x
    ref = conv3d_ref(xp, w, b)
    xd, wd, bd = x.cuda(), w.cuda(), b.cuda()
    out = empty_act((B, T + t_rep, H, W, Co), precision)
    N.check(N.lib().vt_op_conv_stem(precision, _p(xd), _p(wd), _p(bd), _p(out), B, Ci, T, H, W, Co, t_rep, stream()))
    torch.cuda.synchronize()
    check(ncdhw(from_act(out, precision)), ref, precision, "stem")


def test_head_tap_planes_gather():
    """BF16 decoder head: conv_out 128 -> 3 (k333, zero padding, first tdf-1 frames dropped, model_3dcausal.py:883-885) as
    a tap-planes GEMM + gather.  27 bf16-rounded partials per output: bound 27 * 2^-9 * max|partial| + bias rounding."""
    from gpu_util import _p, cl, stream
    B, Ci, Co, T, H, W, to_off = 1, 128, 3, 6, 16, 24, 3
    x = rnd(B, Ci, T, H, W, seed=1).to(torch.bfloat16).float()
    w = rnd(Co, Ci, 3, 3, 3, seed=2, scale=1 / math.sqrt(27 * Ci)).to(torch.bfloat16).float()
    b = rnd(Co, seed=3)
    ref = conv3d_ref(x, w, b)[:, :, to_off:]
    xd = cl(x).to(torch.bfloat16).cuda()
    wd, bd = w.cuda(), b.cuda()
    out = torch.empty((B, Co, T - to_off, H, W), dtype=torch.float32, device="cuda")
    N.check(N.lib().vt_op_head_planes(_p(xd), _p(wd), _p(bd), _p(out), B, T, H, W, Ci, Co, to_off, stream()))
    torch.cuda.synchronize()
    err = (out.cpu().double() - ref).abs()
    assert float(err.max()) <= 0.03, float(err.max())


@pytest.mark.parametrize("precision", PRECS, ids=PIDS)
def test_conv_head_fp32_ncdhw_with_dropped_frames(precision):
    """heads through conv_tc itself: fp32 [B,C,T,H,W] output, Cout padded to 32 internally, to_off leading frames dropped
    (EXACT_TC decoder conv_out; encoder conv_out 512 -> 2z in both modes)"""
    from gpu_util import op_conv_ex
    for (Ci, Co, to_off) in [(128, 3, 3), (512, 8, 0)]:
        B, T, H, W = 1, 5, 16, 16
        x = prep(rnd(B, Ci, T, H, W, seed=1), precision)
        w = prep(rnd(Co, Ci, 3, 3, 3, seed=2, scale=1 / math.sqrt(27 * Ci)), precision)
        b = rnd(Co, seed=3)
        ref = conv3d_ref(x, w, b)[:, :, to_off:]
        got, _ = op_conv_ex(x, w, b, precision=precision, to_off=to_off, out_f32=True)
        # fp32 output: no bf16 output rounding in BF16 mode either
        err = (got.double() - ref).abs()
        assert float(err.max()) <= (2e-3 if precision == N.PREC_BF16 else X3_TOL), float(err.max())


# ---------------------------------------------------------------------------------------------------------------
# phase-collapsed "upsample then conv"
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", PRECS, ids=PIDS)
@pytest.mark.parametrize("fuse_ln", [False, True], ids=["plain", "ln"])
def test_upsample_conv_four_phases(precision, fuse_ln):
    """Upsample (model_3dcausal.py:208-212): nearest 2x (H, W) then conv3x3 == four 1x2x2 convs on the low-res input"""
    from gpu_util import _p, empty_act, from_act, ncdhw, stream, to_act, cl
    B, Ci, Co, T, H, W = 1, 64, 128, 2, 16, 24
    x = prep(rnd(B, Ci, T, H, W, seed=1), precision)
    w = rnd(Co, Ci, 3, 3, seed=2, scale=1 / math.sqrt(9 * Ci))
    b = rnd(Co, seed=3)
    g, bt = 1.0 + 0.5 * rnd(Co, seed=5), 0.3 * rnd(Co, seed=6)
    xu = F.interpolate(x.double().permute(0, 2, 1, 3, 4).reshape(B * T, Ci, H, W), scale_factor=2.0, mode="nearest")
    v = F.conv2d(xu, w.double(), b.double(), padding=1).reshape(B, T, Co, 2 * H, 2 * W).permute(0, 2, 1, 3, 4)
    xd, wd, bd, gd, btd = to_act(cl(x), precision), w.cuda(), b.cuda(), g.cuda(), bt.cuda()
    out = empty_act((B, T, 2 * H, 2 * W, Co), precision)
    out2 = empty_act((B, T, 2 * H, 2 * W, Co), precision) if fuse_ln else None
    N.check(N.lib().vt_op_upsample_conv(precision, 0, _p(xd), _p(wd), _p(bd), 0.0, _p(gd) if fuse_ln else None,
                                        _p(btd) if fuse_ln else None, 1, _p(out), _p(out2), B, T, H, W, Ci, Co, stream()))
    torch.cuda.synchronize()
    # BF16: the collapsed weights are sums of up to 4 taps rounded once (not the sum of rounded taps): slack 2
    check(ncdhw(from_act(out, precision)), v, precision, "upsample conv", slack=2.0)
    if fuse_ln:
        check(ncdhw(from_act(out2, precision)), ln_ref(v, g, bt, True), precision, "upsample conv + LN", slack=2.5)


@pytest.mark.parametrize("precision", PRECS, ids=PIDS)
@pytest.mark.parametrize("fuse_ln", [False, True], ids=["plain", "ln"])
def test_time_upsample_conv_two_phases(precision, fuse_ln):
    """TimeUpsampleResCausal2x v1.0 (model_3dcausal.py:267-273): x' = nearest 2x in T; alpha*x' + (1-alpha)*cconv3(x')
    == even / odd output frames from 2x3x3 convs on x, mixed with x[t/2]"""
    from gpu_util import _p, empty_act, from_act, ncdhw, stream, to_act, cl
    B, C_, T, H, W = 1, 64, 3, 16, 16
    alpha = 0.88
    x = prep(rnd(B, C_, T, H, W, seed=1), precision)
    w = rnd(C_, C_, 3, 3, 3, seed=2, scale=1 / math.sqrt(27 * C_))
    b = rnd(C_, seed=3)
    g, bt = 1.0 + 0.5 * rnd(C_, seed=5), 0.3 * rnd(C_, seed=6)
    xu = F.interpolate(x.double(), scale_factor=[2.0, 1.0, 1.0], mode="nearest")
    v = alpha * xu + (1 - alpha) * conv3d_ref(xu, w, b)
    xd, wd, bd, gd, btd = to_act(cl(x), precision), w.cuda(), b.cuda(), g.cuda(), bt.cuda()
    out = empty_act((B, 2 * T, H, W, C_), precision)
    out2 = empty_act((B, 2 * T, H, W, C_), precision) if fuse_ln else None
    N.check(N.lib().vt_op_upsample_conv(precision, 1, _p(xd), _p(wd), _p(bd), alpha, _p(gd) if fuse_ln else None,
                                        _p(btd) if fuse_ln else None, 1, _p(out), _p(out2), B, T, H, W, C_, C_, stream()))
    torch.cuda.synchronize()
    check(ncdhw(from_act(out, precision)), v, precision, "time-upsample conv", slack=2.0)
    if fuse_ln:
        check(ncdhw(from_act(out2, precision)), ln_ref(v, g, bt, True), precision, "time-upsample conv + LN", slack=2.5)


# ---------------------------------------------------------------------------------------------------------------
# attention core on wgmma (per-frame K / V^T as the B operand), LayerNorm / GroupNorm on split rows
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", PRECS, ids=PIDS)
def test_attention_core_wgmma(precision):
    """small frames (16 x 16 tokens, C = 128); the production size (32 x 32 tokens, C = 512) is in
    tests/test_gpu_production_plans.py"""
    from gpu_util import _p, empty_act, from_act, stream, to_act
    frames, H, W, C_ = 3, 16, 16, 128
    tokens = H * W
    q, k, v = (prep(rnd(frames, tokens, C_, seed=s_), precision) for s_ in (1, 2, 3))
    ref = F.scaled_dot_product_attention(q.double().unsqueeze(0), k.double().unsqueeze(0), v.double().unsqueeze(0))[0]
    qd, kd, vd = (to_act(t, precision) for t in (q, k, v))
    o = empty_act((frames, tokens, C_), precision)
    ws = torch.empty(frames * tokens * (8 * tokens + 24 * C_) + 65536, dtype=torch.uint8, device="cuda")
    lib = N.lib()
    lib.vt_profile_start()
    N.check(lib.vt_op_attention_hw(precision, _p(qd), _p(kd), _p(vd), _p(o), frames, H, W, C_, _p(ws), ws.numel(), stream()))
    buf = C.create_string_buffer(1 << 14)
    lib.vt_profile_stop(buf, len(buf))
    assert b"conv_tc" in buf.value and b"gemm_simt" not in buf.value, buf.value   # the tensor-core formulation ran
    got = from_act(o, precision)
    err = (got.double() - ref).abs()
    # P is rounded to bf16 in BF16 mode: 2^-8 relative on probabilities that sum to 1
    assert float(err.max()) <= (3e-2 if precision == N.PREC_BF16 else X3_TOL), float(err.max())


@pytest.mark.parametrize("C_", [16, 128, 512])
@pytest.mark.parametrize("silu", [False, True])
def test_layernorm_split_rows(C_, silu):
    from gpu_util import _p, join_rows, split_rows, stream
    rows = 777
    x = rnd(rows, C_, seed=1, scale=2.0) + 0.3
    g, b = 1 + 0.1 * rnd(C_, seed=2), 0.1 * rnd(C_, seed=3)
    ref = F.layer_norm(x.double(), (C_,), g.double(), b.double(), eps=1e-6)
    if silu:
        ref = ref * torch.sigmoid(ref)
    xd, gd, bd = split_rows(x.cuda()), g.cuda(), b.cuda()
    y = torch.empty_like(xd)
    N.check(N.lib().vt_op_layernorm(N.PREC_EXACT_TC, _p(xd), _p(gd), _p(bd), _p(y), rows, C_, int(silu), stream()))
    torch.cuda.synchronize()
    # the split input itself carries ~2^-17 relative error
    assert float((join_rows(y).cpu().double() - ref).abs().max()) < 1e-4


@pytest.mark.parametrize("per_position", [False, True])
def test_groupnorm_split_rows(per_position):
    from gpu_util import _p, join_rows, split_rows, stream
    frames, H, W, C_ = 3, 5, 6, 64
    x = rnd(frames, C_, H, W, seed=1, scale=1.5) + 0.2
    g, b = 1 + 0.1 * rnd(C_, seed=2), 0.1 * rnd(C_, seed=3)
    if per_position:
        ref = F.group_norm(x.permute(0, 2, 3, 1).reshape(-1, C_, 1), 32, g, b, eps=1e-6).reshape(frames, H, W, C_)
    else:
        ref = F.group_norm(x, 32, g, b, eps=1e-6).permute(0, 2, 3, 1)
    ref = ref * torch.sigmoid(ref)
    xd, gd, bd = split_rows(x.permute(0, 2, 3, 1).contiguous().cuda()), g.cuda(), b.cuda()
    y = torch.empty_like(xd)
    ws = torch.empty(frames * 64 * 4, dtype=torch.uint8, device="cuda")
    N.check(N.lib().vt_op_groupnorm(N.PREC_EXACT_TC, _p(xd), _p(gd), _p(bd), _p(y), frames, H * W, C_,
                                    int(per_position), 1, _p(ws), ws.numel(), stream()))
    torch.cuda.synchronize()
    # per-position statistics over C/32 = 2 channels amplify the 2^-17 relative error of the split input
    assert float((join_rows(y).cpu() - ref).abs().max()) < (1e-3 if per_position else 1e-4)


# ---------------------------------------------------------------------------------------------------------------
# video I/O adjacent steps (scripts/inference_reconstruct.py:41-47,71-82)
# ---------------------------------------------------------------------------------------------------------------
def test_video_io_u8_to_clip_and_back_bit_exact():
    import numpy as np
    from torchvision import transforms
    from vidtok_b200.video_io import clip_to_frames_u8, frames_to_clip
    g = torch.Generator().manual_seed(0)
    frames = torch.randint(0, 256, (5, 70, 90, 3), generator=g, dtype=torch.uint8)
    H, W = 64, 80
    tf = transforms.Compose([transforms.CenterCrop((H, W)), transforms.Normalize(mean=(0.5, 0.5, 0.5), std=(0.5, 0.5, 0.5))])
    ref = tf(frames.permute(0, 3, 1, 2).float() / 255.0).permute(1, 0, 2, 3)          # [C,T,H,W], reference statement
    got = frames_to_clip(frames.cuda(), H, W)
    assert tuple(got.shape) == (1, 3, 5, H, W) and torch.equal(got[0].cpu(), ref)
    rec = ref * 1.3 + 0.05 * torch.randn(ref.shape, generator=g)                      # leaves [-1,1]: exercises the clamp
    t = torch.clamp(rec, -1.0, 1.0)
    ref_u8 = ((((t + 1.0) / 2.0).numpy() * 255).astype(np.uint8)).transpose(1, 2, 3, 0)   # tensor_to_uint8 + "t c h w -> t h w c"
    got_u8 = clip_to_frames_u8(rec.cuda())
    assert got_u8.dtype == torch.uint8 and np.array_equal(got_u8.cpu().numpy(), ref_u8)


# ---------------------------------------------------------------------------------------------------------------
# fused temporal residual block (tblock_tc.cu)
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("geom", [(1, 5, 8, 128), (2, 20, 16, 256), (1, 3, 64, 64), (3, 2, 8, 16)], ids=["w128", "w256_t20", "64x64", "w16"])
@pytest.mark.parametrize("with_ln", [False, True], ids=["plain", "ln_out"])
def test_fused_temporal_resblock(geom, with_ln):
    """ResnetCausalBlock1D (model_3dcausal.py:473-499) for 128 channels as one launch: out = x + conv2(silu(LN2(conv1(n1)))),
    optionally out2 = silu(LN3(out)).  Reference in fp64 on the bf16-rounded operands; the intermediate h is bf16 in the
    kernel (as it is in the unfused BF16 path), hence the slack."""
    from gpu_util import _p, cl, ncdhw, stream
    B, T, H, W = geom
    C_ = 128
    n1 = rnd(B, C_, T, H, W, seed=1).to(torch.bfloat16).float()
    x = rnd(B, C_, T, H, W, seed=2).to(torch.bfloat16).float()
    w1 = rnd(C_, C_, 3, seed=3, scale=1 / math.sqrt(3 * C_)).to(torch.bfloat16).float()
    w2 = rnd(C_, C_, 3, seed=4, scale=1 / math.sqrt(3 * C_)).to(torch.bfloat16).float()
    b1, b2 = rnd(C_, seed=5), rnd(C_, seed=6)
    g2, be2 = 1.0 + 0.5 * rnd(C_, seed=7), 0.3 * rnd(C_, seed=8) + torch.linspace(-0.5, 0.5, C_)
    g3, be3 = 1.0 + 0.5 * rnd(C_, seed=9), 0.3 * rnd(C_, seed=10)
    h = conv3d_ref(n1, w1[..., None, None], b1)
    hn = ln_ref(h, g2, be2, True)
    out = x.double() + conv3d_ref(hn.to(torch.bfloat16).double(), w2[..., None, None], b2)
    out2 = ln_ref(out, g3, be3, True)
    n1d, xd = cl(n1).to(torch.bfloat16).cuda(), cl(x).to(torch.bfloat16).cuda()
    o = torch.empty_like(xd)
    o2 = torch.empty_like(xd) if with_ln else None
    dev = lambda t: t.contiguous().cuda()  # noqa: E731
    w1d, w2d, b1d, b2d, g2d, be2d, g3d, be3d = map(dev, (w1, w2, b1, b2, g2, be2, g3, be3))
    N.check(N.lib().vt_op_tblock(_p(n1d), _p(xd), _p(w1d), _p(b1d), _p(g2d), _p(be2d), _p(w2d), _p(b2d), _p(g3d), _p(be3d), 1,
                                 _p(o), _p(o2), B, T, H, W, C_, stream()))
    torch.cuda.synchronize()
    check(ncdhw(o.float().cpu()), out, N.PREC_BF16, "tblock out", slack=2.0)
    if with_ln:
        check(ncdhw(o2.float().cpu()), out2, N.PREC_BF16, "tblock out2", slack=2.5)


def test_fused_temporal_resblock_many_frames_per_cta():
    """Same block at a size where every persistent CTA walks ~7 strips x 20 frames (barrier phases wrap many times, the
    3-frame shared-memory ring and the accumulators are recycled hundreds of times).
    The reference is plain PyTorch fp32 on the GPU (TF32 off) with h rounded to bf16 where the kernel rounds it."""
    from gpu_util import _p, stream
    import torch.nn.functional as F
    B, T, H, W, C_ = 4, 20, 128, 256, 128
    g = torch.Generator(device="cuda").manual_seed(11)
    n1 = torch.randn((B, T, H, W, C_), device="cuda", generator=g).to(torch.bfloat16)
    x = torch.randn((B, T, H, W, C_), device="cuda", generator=g).to(torch.bfloat16)
    w1 = (torch.randn((C_, C_, 3), device="cuda", generator=g) / math.sqrt(3 * C_)).to(torch.bfloat16).float()
    w2 = (torch.randn((C_, C_, 3), device="cuda", generator=g) / math.sqrt(3 * C_)).to(torch.bfloat16).float()
    b1, b2, g2, be2, g3, be3 = [torch.randn(C_, device="cuda", generator=g) * 0.3 for _ in range(6)]
    g2, g3 = 1.0 + g2, 1.0 + g3
    o, o2 = torch.empty_like(x), torch.empty_like(x)
    N.check(N.lib().vt_op_tblock(_p(n1), _p(x), _p(w1), _p(b1), _p(g2), _p(be2), _p(w2), _p(b2), _p(g3), _p(be3), 1,
                                 _p(o), _p(o2), B, T, H, W, C_, stream()))
    torch.cuda.synchronize()
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        worst = 0.0
        for bi in range(B):   # per clip to bound the fp32 temporaries
            sl = slice(bi, bi + 1)
            def tc1(a, w, b):   # [1,T,H,W,C]: causal conv over T (two zero frames in front), C -> C
                a = F.pad(a, (0, 0, 0, 0, 0, 0, 2, 0)).permute(0, 2, 3, 4, 1).reshape(-1, C_, T + 2)
                return F.conv1d(a, w, b).reshape(1, H, W, C_, T).permute(0, 4, 1, 2, 3)
            h = tc1(n1[sl].float(), w1, b1)
            hn = F.silu(F.layer_norm(h, (C_,), g2, be2, 1e-6)).to(torch.bfloat16).float()
            ref = x[sl].float() + tc1(hn, w2, b2)
            ref2 = F.silu(F.layer_norm(ref, (C_,), g3, be3, 1e-6))
            r1 = ((o[sl].float() - ref).abs() / (2.0 * (2.0 ** -7 * ref.abs() + 2e-2))).max().item()
            r2 = ((o2[sl].float() - ref2).abs() / (2.5 * (2.0 ** -7 * ref2.abs() + 2e-2))).max().item()
            worst = max(worst, r1, r2)
            assert r1 <= 1.0 and r2 <= 1.0, (bi, r1, r2)
        print(f"tblock stress: worst error / bound = {worst:.3f}")
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


# ---------------------------------------------------------------------------------------------------------------
# regularizers as the epilogue of the bottleneck convolution (encoder conv_out)
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", PRECS, ids=PIDS)
@pytest.mark.parametrize("zc", [4, 8, 16])
def test_conv_out_kl_epilogue(precision, zc):
    """conv_out 512 -> 2z (k333) + DiagonalGaussianRegularizer in one launch: z = mean + exp(.5*clamp(logvar))*noise and
    kl_loss = .5 * sum(mean^2 + var - 1 - logvar) / B (distributions.py:8-28, regularizers.py:82-92).  Every shipped z:
    4 and 16 channels, and 8 (the 8chn configurations), which the epilogue compiles as a separate instantiation."""
    from gpu_util import _p, cl, conv_desc, stream, to_act
    from oracle.vidtok_oracle import kl_regularize
    B, Ci, T, H, W = 2, 512, 3, 16, 16
    x = prep(rnd(B, Ci, T, H, W, seed=1), precision)
    w = prep(rnd(2 * zc, Ci, 3, 3, 3, seed=2, scale=1 / math.sqrt(27 * Ci)), precision)
    b = rnd(2 * zc, seed=3)
    noise = rnd(B, zc, T, H, W, seed=4)
    h_ref = conv3d_ref(x, w, b).float()
    d, _ = conv_desc(x.shape, w.shape)
    xd, wd, bd, nd = to_act(cl(x), precision), w.cuda(), b.cuda(), noise.cuda()
    h = torch.empty((B, 2 * zc, T, H, W), device="cuda")
    z = torch.empty((B, zc, T, H, W), device="cuda")
    kl = torch.zeros((), device="cuda")
    N.check(N.lib().vt_op_conv_regularize(precision, C.byref(d), _p(xd), _p(wd), _p(bd), 1, zc, None, _p(nd), _p(h), _p(z), None, _p(kl), stream()))
    torch.cuda.synchronize()
    tol = 2e-3 if precision == N.PREC_BF16 else X3_TOL
    assert float((h.cpu() - h_ref).abs().max()) <= tol
    # the regularizer itself is exact given the kernel's own h
    z_ref, log = kl_regularize(h.cpu(), noise, True)
    assert float((z.cpu() - z_ref).abs().max()) <= 1e-6 * max(1.0, float(z_ref.abs().max()))
    assert abs(float(kl) - float(log["kl_loss"])) <= 1e-5 * abs(float(log["kl_loss"]))
    # and without the optional h output
    z2 = torch.empty_like(z)
    N.check(N.lib().vt_op_conv_regularize(precision, C.byref(d), _p(xd), _p(wd), _p(bd), 1, zc, None, _p(nd), None, _p(z2), None, _p(kl), stream()))
    torch.cuda.synchronize()
    assert torch.equal(z, z2)


@pytest.mark.parametrize("precision", PRECS, ids=PIDS)
@pytest.mark.parametrize("levels", [(8,) * 4, (8,) * 5, (8,) * 6], ids=["4096", "32768", "262144"])
def test_conv_out_fsq_epilogue(precision, levels):
    """conv_out 512 -> len(levels) + FSQ bound / round / index (regularizers.py:153-178) in one launch, for every shipped
    codebook: 4, 5 and 6 levels of 8 (4096, 32768 and 262144 codes)"""
    from gpu_util import _p, cl, conv_desc, stream, to_act
    from oracle.vidtok_oracle import fsq_regularize
    B, Ci, T, H, W = 2, 512, 3, 16, 16
    d_ = len(levels)
    x = prep(rnd(B, Ci, T, H, W, seed=1), precision)
    w = prep(rnd(d_, Ci, 3, 3, 3, seed=2, scale=1.5 / math.sqrt(27 * Ci)), precision)
    b = rnd(d_, seed=3)
    d, _ = conv_desc(x.shape, w.shape)
    xd, wd, bd = to_act(cl(x), precision), w.cuda(), b.cuda()
    h = torch.empty((B, d_, T, H, W), device="cuda")
    z = torch.empty((B, d_, T, H, W), device="cuda")
    idx = torch.empty((B, T, H, W), dtype=torch.int32, device="cuda")
    lv = (C.c_int32 * d_)(*levels)
    N.check(N.lib().vt_op_conv_regularize(precision, C.byref(d), _p(xd), _p(wd), _p(bd), 2, d_, lv, None, _p(h), _p(z), _p(idx), None, stream()))
    torch.cuda.synchronize()
    codes_ref, log = fsq_regularize(h.cpu(), levels)      # bit-exact given the kernel's own h
    assert torch.equal(idx.cpu(), log["indices"]) and torch.equal(z.cpu(), codes_ref)
    assert int(idx.max()) >= 8 ** (d_ - 1)                # the last level's digit is in play
    if precision == N.PREC_EXACT_TC:                       # and against the fp64 conv: codes equal outside the tie band
        _, log64 = fsq_regularize(conv3d_ref(x, w, b).float(), levels)
        bad = idx.cpu() != log64["indices"]
        pre = log64["pre_round"]
        near = ((pre - pre.floor() - 0.5).abs() < 1e-4).any(dim=-1)
        assert not (bad & ~near).any() and int(bad.sum()) <= 2
