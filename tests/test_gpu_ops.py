"""-m gpu: every kernel of the path against a plain PyTorch fp32 CPU statement of the reference op
(the op-level layer of the test pyramid the reference lacks, SURVEY.md section 4)."""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from vidtok_b200 import _native as N  # noqa: E402


def rnd(*shape, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g) * scale


def ref_causal_conv(x, w, b, stride=(1, 1, 1), pads=None, tmode="zero"):
    """CausalConv3d.forward (model_3dcausal.py:193-197)."""
    kt, kh, kw = w.shape[2:]
    tp = (kt - 1) + (1 - stride[0])
    if pads is None:
        hp, wp = (kh - 1) + (1 - stride[1]), (kw - 1) + (1 - stride[2])
        pads = (hp // 2, hp - hp // 2, wp // 2, wp - wp // 2)
    x = F.pad(x, (pads[2], pads[3], pads[0], pads[1], tp, 0))
    return F.conv3d(x, w, b, stride=stride)


CONV_CASES = [
    # name, Ci, Co, (kt,kh,kw), stride, (B,T,H,W)
    ("k333", 16, 24, (3, 3, 3), (1, 1, 1), (2, 5, 9, 10)),
    ("k133", 32, 64, (1, 3, 3), (1, 1, 1), (2, 3, 8, 8)),
    ("k311", 64, 64, (3, 1, 1), (1, 1, 1), (1, 7, 6, 5)),
    ("k111", 20, 12, (1, 1, 1), (1, 1, 1), (1, 2, 5, 7)),
    ("stem_ci3", 3, 32, (3, 3, 3), (1, 1, 1), (1, 4, 8, 8)),
    ("head_co3", 32, 3, (3, 3, 3), (1, 1, 1), (1, 4, 8, 8)),
    ("head_co8", 64, 8, (3, 3, 3), (1, 1, 1), (2, 3, 4, 4)),
    ("tstride", 32, 32, (3, 3, 3), (2, 1, 1), (1, 10, 6, 6)),
    ("tstride_odd", 32, 32, (3, 3, 3), (2, 1, 1), (1, 5, 6, 6)),
]


@pytest.mark.parametrize("case", CONV_CASES, ids=[c[0] for c in CONV_CASES])
def test_conv_exact(case):
    from gpu_util import op_conv
    _, Ci, Co, k, stride, (B, T, H, W) = case
    x, w, b = rnd(B, Ci, T, H, W, seed=1), rnd(Co, Ci, *k, seed=2, scale=1 / math.sqrt(Ci * k[0] * k[1] * k[2])), rnd(Co, seed=3)
    ref = ref_causal_conv(x.double(), w.double(), b.double(), stride).float()
    got = op_conv(x, w, b, stride=stride)
    assert got.shape == ref.shape
    assert float((got - ref).abs().max()) < 2e-5


def test_conv_downsample_asymmetric_pad():
    """Downsample: pad (0,1,0,1) + conv3x3 stride 2 (model_3dcausal.py:223-227)."""
    from gpu_util import op_conv
    x, w, b = rnd(2, 16, 3, 8, 10, seed=1), rnd(16, 16, 1, 3, 3, seed=2, scale=0.1), rnd(16, seed=3)
    y = F.conv2d(F.pad(x.permute(0, 2, 1, 3, 4).reshape(6, 16, 8, 10), (0, 1, 0, 1)), w[:, :, 0], b, stride=2)
    ref = y.reshape(2, 3, 16, 4, 5).permute(0, 2, 1, 3, 4)
    got = op_conv(x, w, b, stride=(1, 2, 2), pads=(0, 1, 0, 1))
    assert float((got - ref).abs().max()) < 2e-5


def test_conv_upsample_folded():
    """Upsample: nearest 2x then conv3x3 pad 1 (model_3dcausal.py:208-212), upsampling folded into the gather."""
    from gpu_util import op_conv
    x, w, b = rnd(1, 16, 2, 5, 6, seed=1), rnd(16, 16, 1, 3, 3, seed=2, scale=0.1), rnd(16, seed=3)
    xu = F.interpolate(x.permute(0, 2, 1, 3, 4).reshape(2, 16, 5, 6), scale_factor=2.0, mode="nearest")
    ref = F.conv2d(xu, w[:, :, 0], b, padding=1).reshape(1, 2, 16, 10, 12).permute(0, 2, 1, 3, 4)
    got = op_conv(x, w, b, up=(1, 2, 2))
    assert float((got - ref).abs().max()) < 2e-5


def test_conv_time_upsample_mix():
    """TimeUpsampleResCausal2x (model_3dcausal.py:267-273): x' = nearest2x_T(x); alpha*x' + (1-alpha)*conv(x')."""
    from gpu_util import op_conv
    alpha = 0.7
    x, w, b = rnd(1, 16, 3, 4, 4, seed=1), rnd(16, 16, 3, 3, 3, seed=2, scale=0.05), rnd(16, seed=3)
    xu = F.interpolate(x, scale_factor=[2.0, 1.0, 1.0], mode="nearest")
    ref = alpha * xu + (1 - alpha) * ref_causal_conv(xu, w, b)
    got = op_conv(x, w, b, up=(2, 1, 1), res=x, res_mode=2, alpha=alpha)
    assert got.shape == ref.shape and float((got - ref).abs().max()) < 2e-5


def test_conv_time_downsample_mix():
    """TimeDownsampleResCausal2x (model_3dcausal.py:247-252)."""
    from gpu_util import op_conv
    alpha = 0.6
    for T in (10, 5):
        x, w, b = rnd(2, 16, T, 4, 4, seed=1), rnd(16, 16, 3, 3, 3, seed=2, scale=0.05), rnd(16, seed=3)
        x1 = F.avg_pool3d(F.pad(x, (0, 0, 0, 0, 1, 0)), (3, 1, 1), stride=(2, 1, 1))
        ref = alpha * x1 + (1 - alpha) * ref_causal_conv(x, w, b, stride=(2, 1, 1))
        got = op_conv(x, w, b, stride=(2, 1, 1), res=x, res_mode=3, alpha=alpha)
        assert got.shape == ref.shape and float((got - ref).abs().max()) < 2e-5


def test_conv_residual_add_and_linearity():
    from gpu_util import op_conv
    x, w, b = rnd(1, 32, 3, 6, 6, seed=1), rnd(32, 32, 3, 1, 1, seed=2, scale=0.1), rnd(32, seed=3)
    r = rnd(1, 32, 3, 6, 6, seed=4)
    ref = r + ref_causal_conv(x, w, b)
    got = op_conv(x, w, b, res=r, res_mode=1)
    assert float((got - ref).abs().max()) < 2e-5
    # linearity: conv(a*x1 + x2) - bias == a*(conv(x1)-bias) + (conv(x2)-bias)
    x2 = rnd(1, 32, 3, 6, 6, seed=5)
    zero = torch.zeros(32)
    lhs = op_conv(2.5 * x + x2, w, zero)
    rhs = 2.5 * op_conv(x, w, zero) + op_conv(x2, w, zero)
    assert float((lhs - rhs).abs().max()) < 1e-4


@pytest.mark.parametrize("C_", [16, 128, 256, 512])
@pytest.mark.parametrize("silu", [False, True])
def test_layernorm(C_, silu):
    rows = 777
    x = rnd(rows, C_, seed=1, scale=2.0) + 0.3
    g, b = 1 + 0.1 * rnd(C_, seed=2), 0.1 * rnd(C_, seed=3)
    ref = F.layer_norm(x, (C_,), g, b, eps=1e-6)
    if silu:
        ref = ref * torch.sigmoid(ref)
    xd, gd, bd = x.cuda(), g.cuda(), b.cuda()
    y = torch.empty_like(xd)
    N.check(N.lib().vt_op_layernorm(N.PREC_FMA32, C.c_void_p(xd.data_ptr()), C.c_void_p(gd.data_ptr()), C.c_void_p(bd.data_ptr()),
                                    C.c_void_p(y.data_ptr()), rows, C_, int(silu), None))
    torch.cuda.synchronize()
    assert float((y.cpu() - ref).abs().max()) < 1e-5
    # bf16 activations: result within bf16 rounding of the fp32 answer on the same (rounded) input
    xb = x.bfloat16()
    refb = F.layer_norm(xb.float(), (C_,), g, b, eps=1e-6)
    if silu:
        refb = refb * torch.sigmoid(refb)
    xbd = xb.cuda()
    yb = torch.empty_like(xbd)
    N.check(N.lib().vt_op_layernorm(N.PREC_BF16, C.c_void_p(xbd.data_ptr()), C.c_void_p(gd.data_ptr()), C.c_void_p(bd.data_ptr()),
                                    C.c_void_p(yb.data_ptr()), rows, C_, int(silu), None))
    torch.cuda.synchronize()
    assert float((yb.float().cpu() - refb).abs().max()) < 0.04


@pytest.mark.parametrize("per_position", [False, True])
def test_groupnorm(per_position):
    frames, H, W, C_ = 3, 5, 6, 64
    x = rnd(frames, C_, H, W, seed=1, scale=1.5) + 0.2
    g, b = 1 + 0.1 * rnd(C_, seed=2), 0.1 * rnd(C_, seed=3)
    if per_position:
        ref = F.group_norm(x.permute(0, 2, 3, 1).reshape(-1, C_, 1), 32, g, b, eps=1e-6).reshape(frames, H, W, C_)
    else:
        ref = F.group_norm(x, 32, g, b, eps=1e-6).permute(0, 2, 3, 1)
    ref = ref * torch.sigmoid(ref)
    xd = x.permute(0, 2, 3, 1).contiguous().cuda()
    gd, bd = g.cuda(), b.cuda()
    y = torch.empty_like(xd)
    ws = torch.empty(frames * 64 * 4, dtype=torch.uint8, device="cuda")
    N.check(N.lib().vt_op_groupnorm(N.PREC_FMA32, C.c_void_p(xd.data_ptr()), C.c_void_p(gd.data_ptr()), C.c_void_p(bd.data_ptr()),
                                    C.c_void_p(y.data_ptr()), frames, H * W, C_, int(per_position), 1,
                                    C.c_void_p(ws.data_ptr()), ws.numel(), None))
    torch.cuda.synchronize()
    assert float((y.cpu() - ref).abs().max()) < 2e-5


def test_attention_core():
    """per-frame single-head SDPA, scale C^-0.5 (model_3dcausal.py:139-140)."""
    frames, tokens, C_ = 3, 64, 128
    q, k, v = rnd(frames, tokens, C_, seed=1), rnd(frames, tokens, C_, seed=2), rnd(frames, tokens, C_, seed=3)
    ref = F.scaled_dot_product_attention(q.unsqueeze(0), k.unsqueeze(0), v.unsqueeze(0))[0]
    qd, kd, vd = q.cuda(), k.cuda(), v.cuda()
    o = torch.empty_like(qd)
    ws = torch.empty(frames * tokens * (8 * tokens + 24 * C_) + 65536, dtype=torch.uint8, device="cuda")
    N.check(N.lib().vt_op_attention(N.PREC_FMA32, C.c_void_p(qd.data_ptr()), C.c_void_p(kd.data_ptr()), C.c_void_p(vd.data_ptr()),
                                    C.c_void_p(o.data_ptr()), frames, tokens, C_, C.c_void_p(ws.data_ptr()), ws.numel(), None))
    torch.cuda.synchronize()
    assert float((o.cpu() - ref).abs().max()) < 2e-5


def test_fsq_bit_exact_and_inverse():
    from oracle.vidtok_oracle import fsq_indices_to_codes, fsq_regularize
    levels = (8, 8, 8, 8, 8)
    h = rnd(2, 5, 5, 16, 16, seed=7, scale=1.2)
    codes_ref, log = fsq_regularize(h, levels)
    hd = h.cuda()
    codes = torch.empty_like(hd)
    idx = torch.empty((2, 5, 16, 16), dtype=torch.int32, device="cuda")
    lv = (C.c_int32 * 5)(*levels)
    N.check(N.lib().vt_op_fsq(C.c_void_p(hd.data_ptr()), 5, lv, 5 * 16 * 16, 2, C.c_void_p(codes.data_ptr()), C.c_void_p(idx.data_ptr()), None))
    torch.cuda.synchronize()
    bad = (idx.cpu() != log["indices"])
    pre = log["pre_round"]
    near_tie = ((pre - pre.floor() - 0.5).abs() < 1e-4).any(dim=-1)
    assert not (bad & ~near_tie).any()
    assert int(bad.sum()) == 0, f"{int(bad.sum())} mismatches (all within the tie guard band)"
    assert torch.equal(codes.cpu(), codes_ref)
    back = torch.empty_like(hd)
    N.check(N.lib().vt_op_fsq_indices_to_codes(C.c_void_p(idx.data_ptr()), 5, lv, 5 * 16 * 16, 2, C.c_void_p(back.data_ptr()), None))
    torch.cuda.synchronize()
    assert torch.equal(back.cpu(), fsq_indices_to_codes(log["indices"], levels))
    assert torch.equal(back, codes)
    # saturating inputs stay inside the codebook
    big = torch.full((1, 5, 1, 2, 2), 40.0)
    big[0, :, 0, 0, 0] = -40.0
    bd = big.cuda()
    cb, ib = torch.empty_like(bd), torch.empty((1, 1, 2, 2), dtype=torch.int32, device="cuda")
    N.check(N.lib().vt_op_fsq(C.c_void_p(bd.data_ptr()), 5, lv, 4, 1, C.c_void_p(cb.data_ptr()), C.c_void_p(ib.data_ptr()), None))
    torch.cuda.synchronize()
    assert ib.cpu().flatten().tolist() == [0, 32767, 32767, 32767]


def test_kl_reparameterise():
    from oracle.vidtok_oracle import kl_regularize
    h = rnd(2, 8, 5, 8, 8, seed=3, scale=2.0)
    h[0, 4:, 0, 0, 0] = 50.0   # exercises the clamp(-30, 20) (distributions.py:9)
    h[1, 4:, 0, 0, 1] = -50.0
    noise = rnd(2, 4, 5, 8, 8, seed=4)
    z_ref, log = kl_regularize(h, noise, True)
    hd, nd = h.cuda(), noise.cuda()
    z = torch.empty_like(nd)
    kl = torch.empty((), device="cuda")
    N.check(N.lib().vt_op_kl(C.c_void_p(hd.data_ptr()), C.c_void_p(nd.data_ptr()), 4, 5 * 8 * 8, 2, 1, C.c_void_p(z.data_ptr()),
                             C.c_void_p(kl.data_ptr()), None))
    torch.cuda.synchronize()
    assert float((z.cpu() - z_ref).abs().max()) <= 1e-5 * float(z_ref.abs().max())
    assert abs(float(kl) - float(log["kl_loss"])) <= 1e-5 * abs(float(log["kl_loss"]))


# ---------------------------------------------------------------------------------------------------------------
# wgmma / TMA implicit-GEMM kernel (BF16 mode) against fp32 torch on the same bf16-rounded operands
# ---------------------------------------------------------------------------------------------------------------
TC_CASES = [
    # name, Ci, Co, k, stride, (B,T,H,W), res_mode
    ("tc_k333", 64, 64, (3, 3, 3), (1, 1, 1), (1, 3, 16, 16), 0),
    ("tc_k133_n256", 128, 256, (1, 3, 3), (1, 1, 1), (1, 2, 32, 32), 0),
    ("tc_k311", 64, 128, (3, 1, 1), (1, 1, 1), (1, 5, 8, 16), 1),
    ("tc_k111_two_ntiles", 256, 512, (1, 1, 1), (1, 1, 1), (2, 1, 16, 16), 0),
    ("tc_bt2", 64, 64, (3, 3, 3), (1, 1, 1), (1, 4, 8, 8), 1),
    ("tc_partial_tiles", 64, 96, (1, 3, 3), (1, 1, 1), (1, 2, 12, 20), 0),
    ("tc_tstride_avgpool", 64, 64, (3, 3, 3), (2, 1, 1), (2, 6, 16, 16), 3),
    ("tc_many_tiles", 64, 64, (3, 3, 3), (1, 1, 1), (2, 4, 64, 64), 1),
    ("tc_k333_c512", 512, 512, (3, 3, 3), (1, 1, 1), (1, 3, 16, 16), 1),
    # halo windows (8 x 16 output tiles): with the residual through the MMA / at N tile 256 with two time taps
    ("tc_halo_mt2", 64, 128, (1, 3, 3), (1, 1, 1), (1, 5, 128, 128), 1),
    ("tc_halo_k233_n256", 128, 256, (2, 3, 3), (1, 1, 1), (1, 3, 128, 128), 0),
]


@pytest.mark.parametrize("case", TC_CASES, ids=[c[0] for c in TC_CASES])
def test_conv_tc(case):
    from gpu_util import op_conv
    _, Ci, Co, k, stride, (B, T, H, W), res_mode = case
    K = Ci * k[0] * k[1] * k[2]
    x = rnd(B, Ci, T, H, W, seed=1).bfloat16().float()
    w = rnd(Co, Ci, *k, seed=2, scale=1 / math.sqrt(K)).bfloat16().float()
    b = rnd(Co, seed=3)
    conv = ref_causal_conv(x.double(), w.double(), b.double(), stride).float()
    alpha = 0.6
    res = None
    if res_mode == 1:
        res = rnd(*conv.shape, seed=4).bfloat16().float()
        ref = res + conv
    elif res_mode == 3:
        res = x
        x1 = F.avg_pool3d(F.pad(x, (0, 0, 0, 0, 1, 0)), (3, 1, 1), stride=(2, 1, 1))
        ref = alpha * x1 + (1 - alpha) * conv
    else:
        ref = conv
    got = op_conv(x, w, b, stride=stride, res=res, res_mode=res_mode, alpha=alpha, precision=N.PREC_BF16)
    assert got.shape == ref.shape
    err = (got - ref).abs()
    tol = 2.0 ** -7 * ref.abs() + 2e-2
    assert bool((err <= tol).all()), f"max err {float(err.max()):.4f} at ref {float(ref.flatten()[err.argmax()]):.4f}"
    # and the FMA kernel on the same bf16 operands agrees (same math, different engine)
    simt = op_conv(x, w, b, stride=stride, res=res, res_mode=res_mode, alpha=alpha, precision=N.PREC_BF16, force_simt=True)
    assert float((got - simt).abs().max()) <= 2.0 ** -6 * float(ref.abs().max()) + 2e-2


def test_conv_tc_downsample_stride2():
    """Downsample (pad (0,1,0,1), 3x3 stride 2) on the wgmma path: parity-view tensor maps."""
    from gpu_util import op_conv
    for (B, T, H, W, Ci, Co) in [(1, 2, 32, 32, 64, 64), (2, 3, 64, 32, 128, 128)]:
        x = rnd(B, Ci, T, H, W, seed=1).bfloat16().float()
        w = rnd(Co, Ci, 1, 3, 3, seed=2, scale=1 / math.sqrt(9 * Ci)).bfloat16().float()
        b = rnd(Co, seed=3)
        y = F.conv2d(F.pad(x.permute(0, 2, 1, 3, 4).reshape(B * T, Ci, H, W), (0, 1, 0, 1)), w[:, :, 0], b, stride=2)
        ref = y.reshape(B, T, Co, H // 2, W // 2).permute(0, 2, 1, 3, 4)
        got = op_conv(x, w, b, stride=(1, 2, 2), pads=(0, 1, 0, 1), precision=N.PREC_BF16)
        assert got.shape == ref.shape
        err = (got - ref).abs()
        assert bool((err <= 2.0 ** -7 * ref.abs() + 2e-2).all()), float(err.max())


def test_layernorm_bf16_large_rows():
    """persistent bf16 LayerNorm kernel: row counts that do not divide the per-pass row groups"""
    for C_ in (128, 256, 512):
        for rows in (1, 3, 31, 4099):
            x = (rnd(rows, C_, seed=rows, scale=2.0) + 0.5).bfloat16()
            g, b = 1 + 0.1 * rnd(C_, seed=2), 0.1 * rnd(C_, seed=3)
            ref = F.layer_norm(x.float(), (C_,), g, b, eps=1e-6)
            ref = ref * torch.sigmoid(ref)
            xd, gd, bd = x.cuda(), g.cuda(), b.cuda()
            y = torch.empty_like(xd)
            N.check(N.lib().vt_op_layernorm(N.PREC_BF16, C.c_void_p(xd.data_ptr()), C.c_void_p(gd.data_ptr()), C.c_void_p(bd.data_ptr()),
                                            C.c_void_p(y.data_ptr()), rows, C_, 1, None))
            torch.cuda.synchronize()
            assert float((y.float().cpu() - ref).abs().max()) < 0.04
