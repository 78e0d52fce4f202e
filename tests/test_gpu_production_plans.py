"""-m gpu: every kernel plan the four bench.py workloads launch, at production geometry, against fp64 references.

`launch_conv_tc` picks a plan per launch (N tile, halo windows or one A box per tap, stages, kparts, residual through the
MMA or in the epilogue, time padding), and conv_stem / tblock_tc have plans of their own.  The detailed profiler names
each launch by a plan key (tests/gpu_util.py: plan_keys).  PLAN_TABLE lists every key that one bf16 and one exact forward
of kl488, fsq488, v11long (tiled, chunk 16) and kl41616 launch at B = 1, and test_plan_case runs each of them once:

  * through the single-operator entry point that reaches it (vt_op_conv_ex, vt_op_upsample_conv, vt_op_tblock,
    vt_op_conv_stem, vt_op_conv_regularize_ex, vt_op_head_planes, vt_op_attention_hw), at the key's T x H x W, with B = 1
    (B = 2 for the keys in BATCH2), seeded random inputs and per-channel gamma / beta;
  * asserting that the launch carries exactly the key it was written for, so that a change of plan selection fails here
    instead of quietly moving the coverage elsewhere;
  * against fp64 torch on the GPU at full H x W with all channels for the first kt-1 output frames (causal padding /
    cache), one middle frame and the last frame, with the bounds of test_gpu_ops_tc.check (bf16: 2^-7 |ref| + 2e-2;
    exact: 4e-5 (1 + |ref|)), and over the whole tensor against fp32 torch with TF32 off, with 2e-5 (1 + |ref|) more for
    the fp32 reference's own rounding.

The same cases run the plans of the rest of the shipped configurations (test_gpu_zoo.py): keys of the non-causal family
carry their time padding (" pad<front>.<back>", " pool<off>"), and the regularizer heads take every shipped z / codebook.

test_bench_forward_keys_are_in_table re-derives the keys from the model forwards and lists any that the table misses.
"""
import ctypes as C
import gc
import math
import os
import re
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from vidtok_b200 import _native as N  # noqa: E402

X3_TOL = 4e-5
FP32_REF_TOL = 2e-5
ALPHA = 0.6
BENCH = ("kl488", "fsq488", "v11long", "kl41616")


@pytest.fixture(autouse=True)
def _no_tf32():
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old
    gc.collect()
    torch.cuda.empty_cache()      # the cases use up to a few tens of GB each; the library allocates outside torch


# ---------------------------------------------------------------------------------------------------------------
# inputs, activation formats, bounds
# ---------------------------------------------------------------------------------------------------------------
class Rng:
    def __init__(self, seed):
        self.g = torch.Generator(device="cuda").manual_seed(seed)

    def __call__(self, *shape, scale=1.0):
        return torch.randn(shape, device="cuda", generator=self.g) * scale


def prep(t, prec):
    """operand values as the kernel sees them"""
    return t.to(torch.bfloat16).float() if prec == N.PREC_BF16 else t


def act(x, prec):
    """[B,C,T,H,W] fp32 cuda -> channels-last activation in the precision's format"""
    from gpu_util import split_rows
    y = x.permute(0, 2, 3, 4, 1).contiguous()
    return y.to(torch.bfloat16) if prec == N.PREC_BF16 else split_rows(y)


def unact(y, prec):
    """channels-last activation -> [B,C,T,H,W] fp32"""
    if prec == N.PREC_EXACT_TC:
        c = y.shape[-1] // 2
        y = y[..., :c].float() + y[..., c:].float()
    return y.float().permute(0, 4, 1, 2, 3)


def empty(shape_cl, prec):
    shape = list(shape_cl)
    if prec == N.PREC_EXACT_TC:
        shape[-1] *= 2
    return torch.empty(shape, device="cuda", dtype=torch.bfloat16 if prec == N.PREC_BF16 else torch.float16)


def worst_ratio(got, ref, prec, slack, extra=0.0):
    worst = 0.0
    for t in range(got.shape[2]):       # frame by frame: the fp64 temporaries of a whole tensor do not fit
        g, r = got[:, :, t].double(), ref[:, :, t].double()
        a = r.abs()
        tol = slack * (2.0 ** -7 * a + 2e-2) if prec == N.PREC_BF16 else slack * X3_TOL * (1.0 + a)
        if extra:
            tol = tol + extra * (1.0 + a)
        worst = max(worst, float(((g - r).abs() / tol).max()))
    return worst


def pick_frames(T, kt):
    return sorted(set(range(min(kt - 1, T))) | {T // 2, T - 1})


def verify(key, prec, outs, T, kt):
    """outs: (name, got [B,C,T,H,W], ref(dtype, frames or None) -> [B,C,len(frames),H,W], slack)"""
    frames = pick_frames(T, kt)
    fails = []
    for name, got, ref, slack in outs:
        r64 = worst_ratio(got[:, :, frames], ref(torch.float64, frames), prec, slack)
        r32 = worst_ratio(got, ref(torch.float32, None), prec, slack, FP32_REF_TOL)
        print(f"[{key}] {name}: worst error / bound {r64:.3f} (fp64, frames {frames}), {r32:.3f} (fp32, all frames)")
        if not (r64 <= 1.0 and r32 <= 1.0):
            fails.append(f"{key} {name}: error / bound {r64:.3f} (fp64), {r32:.3f} (fp32)")
    return fails


def check_case(key, prec, res):
    """asserts the launched plan key and the bounds of one case; the large tensors are dropped before an assertion
    fails, so that a failing case does not keep them alive in its traceback"""
    keys, outs, T, kt = res
    launched = sorted(keys)
    fails = verify(key, prec, outs, T, kt) if key in keys else []
    del outs, res
    torch.cuda.empty_cache()
    assert key in launched, f"the case for {key!r} launched {launched}"
    assert not fails, "\n".join(fails)


def conv_frames(xp, w, b, stride, frames, dtype):
    """conv3d of a fully padded input at the given output frames (None: all)"""
    kt, st = w.shape[2], stride[0]
    w, b = w.to(dtype), b.to(dtype)
    if frames is None:
        return F.conv3d(xp.to(dtype), w, b, stride=stride)
    return torch.cat([F.conv3d(xp[:, :, t * st:t * st + kt].to(dtype), w, b, stride=stride) for t in frames], dim=2)


def ln_act(v, g, b, silu=True):
    y = F.layer_norm(v.permute(0, 2, 3, 4, 1), (v.shape[1],), g.to(v.dtype), b.to(v.dtype), eps=1e-6).permute(0, 4, 1, 2, 3)
    return y * torch.sigmoid(y) if silu else y


def ln_params(rng, C_):
    return 1.0 + 0.5 * rng(C_), 0.3 * rng(C_) + torch.linspace(-0.5, 0.5, C_, device="cuda")


# ---------------------------------------------------------------------------------------------------------------
# plan keys
# ---------------------------------------------------------------------------------------------------------------
KEY_RE = re.compile(r"(?P<kern>conv_tc3?) k(?P<kt>\d)(?P<kh>\d)(?P<kw>\d) s(?P<st>\d)(?P<sh>\d) (?P<ci>\d+)->(?P<co>\d+) "
                    r"@(?P<T>\d+)x(?P<H>\d+)x(?P<W>\d+) tile\S+ bn\d+( halo)? ln(?P<ln>\d) r(?P<r>\d)(?P<m>m?) p\d+ "
                    r"t(?P<t>\d) st\d+( pad(?P<pf>\d+)\.(?P<pb>\d+))?( pool(?P<pool>\d+))?$")
STEM_RE = re.compile(r"(?P<kern>conv_stem3?) k333 (?P<ci>\d+)->(?P<co>\d+) @(?P<T>\d+)x(?P<H>\d+)x(?P<W>\d+)"
                     r"( pad(?P<pf>\d+)\.(?P<pb>\d+))?$")
REG_CO = (4, 5, 6, 8, 16, 32)       # encoder conv_out: FSQ with 4 / 5 / 6 levels, KL with z = 4 / 8 / 16 (Co = 2 z)
TBLOCK_RE = re.compile(r"tblock_tc strip \S+ T(?P<T>\d+) ln_out(?P<ln>\d)$")


def parse(key):
    for rx in (KEY_RE, STEM_RE, TBLOCK_RE):
        m = rx.match(key)
        if m:
            d = {k: (int(v) if v is not None and v.isdigit() else v) for k, v in m.groupdict().items()}
            d["kind"] = key.split(" ", 1)[0]
            return d
    raise AssertionError(f"unparsed plan key: {key}")


def entry_of(p):
    """which single-operator entry point reaches the plan of key p (see Exec in model.cu)"""
    if p["kind"] == "tblock_tc":
        return "tblock"
    if p["kind"].startswith("conv_stem"):
        return "stem"
    tokens = p["H"] * p["W"]
    if (p["ci"], p["co"]) in ((512, tokens), (tokens, 512)) and p["kt"] * p["kh"] * p["kw"] == 1 and p["T"] == 1:
        return "attention"                     # S = Q K^T (C -> tokens) and O = P V (tokens -> C) of a 32 x 32 / 16 x 16 frame
    if (p["kt"], p["kh"], p["kw"]) == (1, 2, 2):
        return "upsample"                      # one of the four phase convolutions of Upsample
    if (p["kt"], p["kh"], p["kw"]) == (2, 3, 3):
        return "time_upsample"                 # one of the two phase convolutions of TimeUpsampleResCausal2x (v1.0)
    if p["co"] in REG_CO:
        return "regularize"                    # encoder conv_out + FSQ (4, 5, 6) / KL (2 z = 8, 16, 32) in the epilogue
    if p["co"] == 3:
        return "head"                          # decoder conv_out, fp32 [B,C,T,H,W] output
    if p["kind"] == "conv_tc" and (p["kt"], p["ci"], p["co"]) == (1, 128, 128) and p["kh"] == 1:
        return "head_planes"                   # BF16 decoder conv_out: 27 tap planes by one GEMM, then a gather
    return "conv"


def prec_of(p):
    return N.PREC_EXACT_TC if p["kind"] in ("conv_tc3", "conv_stem3") else N.PREC_BF16


# ---------------------------------------------------------------------------------------------------------------
# one case per entry point
# ---------------------------------------------------------------------------------------------------------------
def _p(t):
    return C.c_void_p(0 if t is None else t.data_ptr())


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def time_pads(p):
    """(front, back) zero frames of the key's conv: the causal (kt-1)+(1-st) in front unless the key names its padding"""
    if p.get("pf") is not None:
        return p["pf"], p["pb"]
    if p["kind"].startswith("conv_stem"):
        return 2, 0
    return (p["kt"] - 1) + (1 - p["st"]), 0


def _desc(B, Ci, Co, k, stride, Ti, Hi, Wi, pads, res_mode=0, alpha=0.0, pt=None):
    d = N.ConvDesc()
    d.B, d.Ti, d.Hi, d.Wi, d.Ci, d.Co = B, Ti, Hi, Wi, Ci, Co
    d.kt, d.kh, d.kw = k
    d.st, d.sh, d.sw = stride
    d.pt = (k[0] - 1) + (1 - stride[0]) if pt is None else pt
    d.ph0, d.ph1, d.pw0, d.pw1 = pads
    d.ut = d.uh = d.uw = 1
    d.res_mode, d.alpha = res_mode, alpha
    return d


def _front(x, t_mode, pt, rng, prec):
    """time front padding of x: zeros (t0), replicated frame 0 (t1) or a cache of pt frames (t2); -> (front, cache)"""
    if pt == 0 or t_mode == 0:
        return x[:, :, :0].new_zeros(x.shape[0], x.shape[1], pt, *x.shape[3:]), None
    if t_mode == 1:
        return x[:, :, :1].repeat(1, 1, pt, 1, 1), None
    cache = prep(rng(x.shape[0], x.shape[1], pt, *x.shape[3:]), prec)
    return cache, cache


def case_conv(p, prec, B, rng, weight_scale=1.0):
    """vt_op_conv_ex: plain / residual (r1m: + x through the MMA; r1: alpha-mix of v1.1 TimeUpsample) / time-downsample
    avg-pool mix (r3, window shifted by one frame with pool1), fused LayerNorm+SiLU (ln1 / ln2), v1.1 replicate / cache
    time padding, the non-causal family's zero padding behind the end (pad<front>.<back>), stride-2 Downsample"""
    kt, kh, kw, st, sh = p["kt"], p["kh"], p["kw"], p["st"], p["sh"]
    Ci, Co, To, Ho, Wo = p["ci"], p["co"], p["T"], p["H"], p["W"]
    head = entry_of(p) == "head"
    # v1.0 causal decoder conv_out drops its first tdf-1 = 3 frames (the non-causal family drops none)
    to_off = 3 if head and p["t"] == 0 and p.get("pf") is None else 0
    pt, pt_back = time_pads(p)
    pool_off = p.get("pool") or 0
    Ti, Hi, Wi = (To - 1 + to_off) * st + kt - pt - pt_back, Ho * sh, Wo * sh
    pads = (0, 1, 0, 1) if sh == 2 else ((kh - 1) // 2, kh // 2, (kw - 1) // 2, kw // 2)
    K = Ci * kt * kh * kw
    x = prep(rng(B, Ci, Ti, Hi, Wi), prec)
    w = prep(rng(Co, Ci, kt, kh, kw, scale=weight_scale / math.sqrt(K)), prec)
    b = rng(Co)
    front, cache = _front(x, p["t"], pt, rng, prec)
    back = x.new_zeros(B, Ci, pt_back, Hi, Wi)
    xp = F.pad(torch.cat([front, x, back], dim=2), (pads[2], pads[3], pads[0], pads[1], 0, 0))
    res, mix, res_mode, res_t_mode = None, False, p["r"], 0
    if res_mode == 1:
        res = prep(rng(B, Co, To, Ho, Wo), prec)
        mix = p["m"] != "m"
    elif res_mode == 3:
        res, res_t_mode = x, p["t"]
        if p["t"] == 2:
            cache = cache[:, :, -1:]          # the stride-2 conv pads one frame: the conv and pool caches are one frame
            front = cache
    g = bt = None
    if p["ln"]:
        g, bt = ln_params(rng, Co)

    def v_ref(dtype, frames):
        y = conv_frames(xp, w, b, (st, sh, sh), [to_off + t for t in frames] if frames is not None else None, dtype)
        if frames is None and to_off:
            y = y[:, :, to_off:]
        if res_mode == 1:
            r = res.to(dtype) if frames is None else res[:, :, frames].to(dtype)
            y = ALPHA * r + (1 - ALPHA) * y if mix else r + y
        elif res_mode == 3:
            if pool_off:                      # frames 2t .. 2t+2, one zero frame behind the end
                pool_in = torch.cat([x, torch.zeros_like(x[:, :, :1])], dim=2).to(dtype)
            else:
                pool_in = torch.cat([front if p["t"] else torch.zeros_like(x[:, :, :1]), x], dim=2).to(dtype)
            pool = F.avg_pool3d(pool_in, (3, 1, 1), stride=(2, 1, 1))
            y = ALPHA * (pool if frames is None else pool[:, :, frames]) + (1 - ALPHA) * y
        return y

    e = N.ConvEx()
    e.d = _desc(B, Ci, Co, (kt, kh, kw), (st, sh, sh), Ti, Hi, Wi, pads, res_mode, ALPHA if (mix or res_mode == 3) else 0.0, pt)
    e.force_simt, e.t_mode, e.ln_mode, e.ln_silu, e.to_off = 0, p["t"], p["ln"], 1, to_off
    e.pt_back, e.res_pool_off = pt_back, pool_off
    e.out_f32_ncdhw, e.res_mix, e.res_t_mode = int(head), int(mix), res_t_mode
    e.cacheT = 0 if cache is None else cache.shape[2]
    xd, cd = act(x, prec), (act(cache, prec) if cache is not None else None)
    rd = act(res, prec) if res is not None else None
    out = torch.empty((B, Co, To, Ho, Wo), device="cuda") if head else empty((B, To, Ho, Wo, Co), prec)
    out2 = empty((B, To, Ho, Wo, Co), prec) if p["ln"] == 2 else None
    from gpu_util import plan_keys
    _, keys = plan_keys(lambda: N.check(N.lib().vt_op_conv_ex(prec, C.byref(e), _p(xd), _p(cd), _p(w), _p(b), _p(rd), _p(g), _p(bt),
                                                               _p(out), _p(out2), _stream())))
    got = out if head else unact(out, prec)
    if p["ln"] == 1:
        outs = [("act(LN(v))", got, lambda dt, fr: ln_act(v_ref(dt, fr), g, bt), 1.5)]
    else:
        outs = [("v", got, v_ref, 1.0)]
        if p["ln"] == 2:
            outs.append(("act(LN(v))", unact(out2, prec), lambda dt, fr: ln_act(v_ref(dt, fr), g, bt), 1.5))
    return keys, outs, To, kt


def case_regularize(p, prec, B, rng):
    """vt_op_conv_regularize_ex: encoder conv_out with KL (Co = 2 z, z = 4, 8, 16) or FSQ (Co = 4, 5, 6 levels of 8) in the
    epilogue; the head h against the conv reference, z / indices / kl_loss against the oracle's regularizer on the
    kernel's own h"""
    from oracle.vidtok_oracle import fsq_regularize, kl_regularize
    Ci, Co, To, H, W = p["ci"], p["co"], p["T"], p["H"], p["W"]
    pt, pt_back = time_pads(p)
    Ti = To + 2 - pt - pt_back
    x = prep(rng(B, Ci, Ti, H, W), prec)
    w = prep(rng(Co, Ci, 3, 3, 3, scale=1.5 / math.sqrt(27 * Ci)), prec)
    b = rng(Co)
    front, cache = _front(x, p["t"], pt, rng, prec)
    xp = F.pad(torch.cat([front, x, x.new_zeros(B, Ci, pt_back, H, W)], dim=2), (1, 1, 1, 1, 0, 0))
    fsq = Co in (4, 5, 6)
    zc = Co if fsq else Co // 2
    levels = (8,) * Co if fsq else None
    e = N.ConvEx()
    e.d = _desc(B, Ci, Co, (3, 3, 3), (1, 1, 1), Ti, H, W, (1, 1, 1, 1), pt=pt)
    e.t_mode, e.cacheT, e.pt_back = p["t"], 0 if cache is None else pt, pt_back
    h = torch.empty((B, Co, To, H, W), device="cuda")
    z = torch.empty((B, zc, To, H, W), device="cuda")
    idx = torch.empty((B, To, H, W), dtype=torch.int32, device="cuda") if fsq else None
    kl = torch.zeros((), device="cuda")
    noise = None if fsq else rng(B, zc, To, H, W)
    lv = (C.c_int32 * Co)(*levels) if fsq else None
    xd, cd = act(x, prec), (act(cache, prec) if cache is not None else None)
    from gpu_util import plan_keys
    _, keys = plan_keys(lambda: N.check(N.lib().vt_op_conv_regularize_ex(prec, C.byref(e), _p(xd), _p(cd), _p(w), _p(b), 2 if fsq else 1, zc,
                                                                       lv, _p(noise), _p(h), _p(z), _p(idx), _p(None if fsq else kl),
                                                                       _stream())))
    if fsq:
        codes, log = fsq_regularize(h.cpu(), levels)
        assert torch.equal(idx.cpu(), log["indices"]) and torch.equal(z.cpu(), codes)
    else:
        z_ref, log = kl_regularize(h.cpu(), noise.cpu(), True)
        assert float((z.cpu() - z_ref).abs().max()) <= 1e-6 * max(1.0, float(z_ref.abs().max()))
        assert abs(float(kl) - float(log["kl_loss"])) <= 1e-5 * abs(float(log["kl_loss"]))
    return keys, [("h", h, lambda dt, fr: conv_frames(xp, w, b, (1, 1, 1), fr, dt), 1.0)], To, 3


def case_head_planes(p, prec, B, rng):
    """vt_op_head_planes: BF16 v1.0 decoder conv_out 128 -> 3 (k333, first 3 frames dropped) as tap planes + gather.
    27 bf16-rounded partials per output: absolute bound 0.03 (test_gpu_ops_tc.test_head_tap_planes_gather)"""
    T, H, W, Ci, Co, to_off = p["T"], p["H"], p["W"], 128, 3, 3
    x = prep(rng(B, Ci, T, H, W), prec)
    w = prep(rng(Co, Ci, 3, 3, 3, scale=1 / math.sqrt(27 * Ci)), prec)
    b = rng(Co)
    xp = F.pad(x, (1, 1, 1, 1, 2, 0))
    out = torch.empty((B, Co, T - to_off, H, W), device="cuda")
    xd = act(x, prec)
    from gpu_util import plan_keys
    _, keys = plan_keys(lambda: N.check(N.lib().vt_op_head_planes(_p(xd), _p(w), _p(b), _p(out), B, T, H, W, Ci, Co, to_off, _stream())))
    ref = conv_frames(xp, w, b, (1, 1, 1), list(range(to_off, T)), torch.float64)
    err = float((out.double() - ref).abs().max())
    print(f"[head planes] max err {err:.3e} (bound 0.03)")
    assert err <= 0.03
    return keys, [], T - to_off, 3


def case_stem(p, prec, B, rng):
    """vt_op_conv_stem (vt_op_conv_stem_ex for pad1.1): encoder conv_in 3 -> 128 from the caller's fp32 [B,3,T,H,W]; t_rep replicated leading frames
    (the v1.0 clip of 17 frames and the first v1.1 chunk of 1 frame get 3), or one zero frame at each end (pad1.1: the
    non-causal family)"""
    To, H, W, Ci, Co = p["T"], p["H"], p["W"], p["ci"], p["co"]
    pt, pt_back = time_pads(p)
    t_rep = 3 if To in (20, 4) and pt == 2 else 0
    T = To - t_rep
    x = prep(rng(B, Ci, T, H, W), prec)
    w = prep(rng(Co, Ci, 3, 3, 3, scale=1 / math.sqrt(27 * Ci)), prec)
    b = rng(Co)
    xr = torch.cat([x[:, :, :1].repeat(1, 1, t_rep, 1, 1), x], dim=2)
    xp = F.pad(xr, (1, 1, 1, 1, pt, pt_back))
    out = empty((B, To, H, W, Co), prec)
    from gpu_util import plan_keys
    if pt == 2:
        run = lambda: N.lib().vt_op_conv_stem(prec, _p(x), _p(w), _p(b), _p(out), B, Ci, T, H, W, Co, t_rep, _stream())  # noqa: E731
    else:
        run = lambda: N.lib().vt_op_conv_stem_ex(prec, _p(x), _p(w), _p(b), _p(out), B, Ci, T, H, W, Co, t_rep, pt, _stream())  # noqa: E731
    _, keys = plan_keys(lambda: N.check(run()))
    return keys, [("stem", unact(out, prec), lambda dt, fr: conv_frames(xp, w, b, (1, 1, 1), fr, dt), 1.0)], To, 3


def case_upsample(p, prec, B, rng):
    """vt_op_upsample_conv: kind 0 = Upsample (nearest 2x in H, W, then 3x3: four 1x2x2 phase convs on the low-resolution
    input), kind 1 = TimeUpsampleResCausal2x v1.0 (nearest 2x in T, alpha-mix with a causal 3x3x3: two 2x3x3 phase convs),
    kind 2 = the non-causal TimeUpsampleRes2x (the 3x3x3 zero-padded by one frame at each end; its odd phase is the key
    with pad0.1).  Collapsed bf16 weights are sums of up to 4 taps rounded once: slack 2 (2.5 after the LayerNorm)"""
    kind = 0 if p["kt"] == 1 else (2 if p.get("pf") is not None else 1)
    C_, T, H, W = p["ci"], p["T"], p["H"], p["W"]
    x = prep(rng(B, C_, T, H, W), prec)
    b = rng(C_)
    g = bt = out2 = None
    if kind == 0:
        w = rng(C_, C_, 3, 3, scale=1 / math.sqrt(9 * C_))
        To, Ho, Wo = T, 2 * H, 2 * W
        xu = F.interpolate(x.permute(0, 2, 1, 3, 4).reshape(B * T, C_, H, W), scale_factor=2.0, mode="nearest")
        xu = xu.reshape(B, T, C_, Ho, Wo).permute(0, 2, 1, 3, 4)
        xp = F.pad(xu, (1, 1, 1, 1, 0, 0))
        w3 = w[:, :, None]

        def v_ref(dt, fr):
            return conv_frames(xp, w3, b, (1, 1, 1), fr, dt)
    else:
        w = rng(C_, C_, 3, 3, 3, scale=1 / math.sqrt(27 * C_))
        To, Ho, Wo = 2 * T, H, W
        xu = x.repeat_interleave(2, dim=2)
        xp = F.pad(xu, (1, 1, 1, 1, 2, 0) if kind == 1 else (1, 1, 1, 1, 1, 1))

        def v_ref(dt, fr):
            u = xu.to(dt) if fr is None else xu[:, :, fr].to(dt)
            return ALPHA * u + (1 - ALPHA) * conv_frames(xp, w, b, (1, 1, 1), fr, dt)
    if p["ln"]:
        g, bt = ln_params(rng, C_)
        out2 = empty((B, To, Ho, Wo, C_), prec)
    out = empty((B, To, Ho, Wo, C_), prec)
    xd = act(x, prec)
    from gpu_util import plan_keys
    _, keys = plan_keys(lambda: N.check(N.lib().vt_op_upsample_conv(prec, kind, _p(xd), _p(w), _p(b), ALPHA if kind else 0.0, _p(g), _p(bt), 1,
                                                                     _p(out), _p(out2), B, T, H, W, C_, C_, _stream())))
    outs = [("v", unact(out, prec), v_ref, 2.0)]
    if p["ln"]:
        outs.append(("act(LN(v))", unact(out2, prec), lambda dt, fr: ln_act(v_ref(dt, fr), g, bt), 2.5))
    return keys, outs, To, 3 if kind else 1


def case_attention(p, prec, frames, rng, C_=512):
    """vt_op_attention_hw on frames of H x W tokens: S = Q K^T / sqrt(C) and O = P V on wgmma (per-frame K / V^T as the B
    operand), softmax in between; BF16 rounds P to bf16 (2^-8 relative on probabilities that sum to 1)"""
    H, W = p["H"], p["W"]
    tokens = H * W
    q, k, v = (prep(rng(frames, C_, 1, H, W), prec) for _ in range(3))
    qd, kd, vd = (act(t, prec) for t in (q, k, v))
    o = empty((frames, 1, H, W, C_), prec)
    ws = torch.empty(frames * tokens * (8 * tokens + 24 * C_) + 65536, dtype=torch.uint8, device="cuda")
    from gpu_util import plan_keys
    _, keys = plan_keys(lambda: N.check(N.lib().vt_op_attention_hw(prec, _p(qd), _p(kd), _p(vd), _p(o), frames, H, W, C_, _p(ws), ws.numel(),
                                                                 _stream())))

    def ref(dt, fr):
        sel = (lambda t: t) if fr is None else (lambda t: t[fr])
        tok = [sel(t).to(dt).reshape(-1, C_, tokens).transpose(1, 2) for t in (q, k, v)]
        y = F.scaled_dot_product_attention(*tok)                     # [frames, tokens, C]
        return y.transpose(1, 2).reshape(-1, C_, H, W).permute(1, 0, 2, 3)[None]   # frames on the T axis

    got = unact(o, prec).permute(2, 1, 0, 3, 4)                      # [1, C, frames, H, W]
    return keys, [("o", got, ref, 1.0)], frames, 1


def case_tblock(p, prec, B, rng, H=256, W=256):
    """vt_op_tblock: the fused temporal ResnetBlock (128 channels, BF16): out = x + conv2(silu(LN2(conv1(n1)))), optionally
    out2 = silu(LN3(out)); h is bf16 inside the kernel, hence the slack (test_gpu_ops_tc.test_fused_temporal_resblock)"""
    T, C_ = p["T"], 128
    n1, x = prep(rng(B, C_, T, H, W), prec), prep(rng(B, C_, T, H, W), prec)
    w1, w2 = (prep(rng(C_, C_, 3, scale=1 / math.sqrt(3 * C_)), prec) for _ in range(2))
    b1, b2 = rng(C_), rng(C_)
    g2, be2 = ln_params(rng, C_)
    g3, be3 = ln_params(rng, C_)
    o = empty((B, T, H, W, C_), prec)
    o2 = empty((B, T, H, W, C_), prec) if p["ln"] else None
    n1d, xd = act(n1, prec), act(x, prec)
    from gpu_util import plan_keys
    _, keys = plan_keys(lambda: N.check(N.lib().vt_op_tblock(_p(n1d), _p(xd), _p(w1), _p(b1), _p(g2), _p(be2), _p(w2), _p(b2), _p(g3), _p(be3),
                                                              1, _p(o), _p(o2), B, T, H, W, C_, _stream())))

    def tconv(a, w, b):   # causal conv over T (two zero frames in front)
        return F.conv3d(F.pad(a, (0, 0, 0, 0, 2, 0)), w[..., None, None].to(a.dtype), b.to(a.dtype))

    def out_ref(dt, fr):
        if fr is None:
            hn = ln_act(tconv(n1.to(dt), w1, b1), g2, be2).to(torch.bfloat16).to(dt)
            return x.to(dt) + tconv(hn, w2, b2)
        res = []
        for t in fr:
            # output frame t reads h of frames t-2..t, which read n1 of frames t-4..t; h of frames < 0 is zero padding
            lo = max(0, t - 2)
            a = n1[:, :, max(0, lo - 2):t + 1].to(dt)
            a = F.pad(a, (0, 0, 0, 0, 2 - (lo - max(0, lo - 2)), 0))
            h = F.conv3d(a, w1[..., None, None].to(dt), b1.to(dt))          # h of frames lo..t
            hn = ln_act(h, g2, be2).to(torch.bfloat16).to(dt)
            hn = F.pad(hn, (0, 0, 0, 0, 2 - (t - lo), 0))
            res.append(x[:, :, t:t + 1].to(dt) + F.conv3d(hn, w2[..., None, None].to(dt), b2.to(dt)))
        return torch.cat(res, dim=2)

    outs = [("out", unact(o, prec), out_ref, 2.0)]
    if p["ln"]:
        outs.append(("out2", unact(o2, prec), lambda dt, fr: ln_act(out_ref(dt, fr), g3, be3), 2.5))
    return keys, outs, T, 5


CASES = {"conv": case_conv, "head": case_conv, "regularize": case_regularize, "head_planes": case_head_planes,
         "stem": case_stem, "upsample": case_upsample, "time_upsample": case_upsample, "attention": case_attention,
         "tblock": case_tblock}


# ---------------------------------------------------------------------------------------------------------------
# the table: every plan key one bf16 and one exact forward of the four bench.py workloads launch at B = 1
# (test_bench_forward_keys_are_in_table lists any key missing here)
# ---------------------------------------------------------------------------------------------------------------
PLAN_TABLE = [
    "conv_stem k333 3->128 @16x256x256",
    "conv_stem k333 3->128 @20x256x256",
    "conv_stem k333 3->128 @20x512x512",
    "conv_stem k333 3->128 @4x256x256",
    "conv_stem3 k333 3->128 @16x256x256",
    "conv_stem3 k333 3->128 @20x256x256",
    "conv_stem3 k333 3->128 @20x512x512",
    "conv_stem3 k333 3->128 @4x256x256",
    "conv_tc k111 s11 1024->512 @1x32x32 tile1x8x16 bn256 ln0 r0 p1 t0 st4",
    "conv_tc k111 s11 128->128 @20x256x256 tile1x8x16 bn128 ln0 r0 p1 t0 st6",
    "conv_tc k111 s11 128->128 @20x512x512 tile1x8x16 bn128 ln0 r0 p1 t0 st6",
    "conv_tc k111 s11 128->256 @16x128x128 tile1x8x16 bn256 ln0 r0 p1 t0 st4",
    "conv_tc k111 s11 128->256 @20x128x128 tile1x8x16 bn256 ln0 r0 p1 t0 st4",
    "conv_tc k111 s11 128->256 @20x256x256 tile1x8x16 bn256 ln0 r0 p1 t0 st4",
    "conv_tc k111 s11 128->256 @4x128x128 tile1x8x16 bn256 ln0 r0 p1 t0 st4",
    "conv_tc k111 s11 256->128 @16x256x256 tile1x8x16 bn128 ln0 r0 p1 t0 st6",
    "conv_tc k111 s11 256->128 @20x256x256 tile1x8x16 bn128 ln0 r0 p1 t0 st6",
    "conv_tc k111 s11 256->128 @20x512x512 tile1x8x16 bn128 ln0 r0 p1 t0 st6",
    "conv_tc k111 s11 256->128 @8x256x256 tile1x8x16 bn128 ln0 r0 p1 t0 st6",
    "conv_tc k111 s11 256->512 @10x64x64 tile1x8x16 bn256 ln0 r0 p1 t0 st4",
    "conv_tc k111 s11 256->512 @20x128x128 tile1x8x16 bn256 ln0 r0 p1 t0 st4",
    "conv_tc k111 s11 256->512 @2x64x64 tile1x8x16 bn256 ln0 r0 p1 t0 st4",
    "conv_tc k111 s11 256->512 @8x64x64 tile1x8x16 bn256 ln0 r0 p1 t0 st4",
    "conv_tc k111 s11 512->1024 @1x32x32 tile1x8x16 bn256 ln0 r0 p1 t0 st4",
    "conv_tc k111 s11 512->256 @10x128x128 tile1x8x16 bn256 ln0 r0 p1 t0 st4",
    "conv_tc k111 s11 512->256 @10x256x256 tile1x8x16 bn256 ln0 r0 p1 t0 st4",
    "conv_tc k111 s11 512->256 @4x128x128 tile1x8x16 bn256 ln0 r0 p1 t0 st4",
    "conv_tc k111 s11 512->256 @8x128x128 tile1x8x16 bn256 ln0 r0 p1 t0 st4",
    "conv_tc k111 s11 512->512 @1x32x32 tile1x8x16 bn256 ln0 r0 p1 t0 st4",
    "conv_tc k111 s11 512->512 @1x32x32 tile1x8x16 bn256 ln0 r1m p1 t0 st4",
    "conv_tc k111 s11 512->512 @2x32x32 tile1x8x16 bn256 ln0 r0 p1 t0 st4",
    "conv_tc k111 s11 512->512 @2x32x32 tile1x8x16 bn256 ln0 r1m p1 t0 st4",
    "conv_tc k111 s11 512->512 @4x32x32 tile1x8x16 bn256 ln0 r0 p1 t0 st4",
    "conv_tc k111 s11 512->512 @4x32x32 tile1x8x16 bn256 ln0 r1m p1 t0 st4",
    "conv_tc k111 s11 512->512 @5x32x32 tile1x8x16 bn256 ln0 r0 p1 t0 st4",
    "conv_tc k111 s11 512->512 @5x32x32 tile1x8x16 bn256 ln0 r1m p1 t0 st4",
    "conv_tc k122 s11 256->256 @10x128x128 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4",
    "conv_tc k122 s11 256->256 @10x256x256 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4",
    "conv_tc k122 s11 256->256 @4x128x128 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4",
    "conv_tc k122 s11 256->256 @8x128x128 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4",
    "conv_tc k122 s11 512->512 @2x32x32 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4",
    "conv_tc k122 s11 512->512 @2x64x64 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4",
    "conv_tc k122 s11 512->512 @4x32x32 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4",
    "conv_tc k122 s11 512->512 @4x64x64 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4",
    "conv_tc k122 s11 512->512 @5x128x128 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4",
    "conv_tc k122 s11 512->512 @5x32x32 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4",
    "conv_tc k122 s11 512->512 @5x64x64 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4",
    "conv_tc k133 s11 128->128 @16x256x256 tile1x16x8 bn128 halo ln1 r0 p1 t0 st8",
    "conv_tc k133 s11 128->128 @16x256x256 tile1x16x8 bn128 halo ln2 r1m p1 t0 st8",
    "conv_tc k133 s11 128->128 @20x256x256 tile1x16x8 bn128 halo ln1 r0 p1 t0 st8",
    "conv_tc k133 s11 128->128 @20x256x256 tile1x16x8 bn128 halo ln2 r1m p1 t0 st8",
    "conv_tc k133 s11 128->128 @20x512x512 tile1x16x8 bn128 halo ln1 r0 p1 t0 st8",
    "conv_tc k133 s11 128->128 @20x512x512 tile1x16x8 bn128 halo ln2 r1m p1 t0 st8",
    "conv_tc k133 s11 128->128 @4x256x256 tile1x16x8 bn128 halo ln1 r0 p1 t0 st8",
    "conv_tc k133 s11 128->128 @4x256x256 tile1x16x8 bn128 halo ln2 r1m p1 t0 st8",
    "conv_tc k133 s11 128->128 @8x256x256 tile1x16x8 bn128 halo ln1 r0 p1 t0 st8",
    "conv_tc k133 s11 128->128 @8x256x256 tile1x16x8 bn128 halo ln2 r1m p1 t0 st8",
    "conv_tc k133 s11 128->256 @16x128x128 tile1x16x8 bn256 halo ln1 r0 p1 t0 st4",
    "conv_tc k133 s11 128->256 @20x128x128 tile1x16x8 bn256 halo ln1 r0 p1 t0 st4",
    "conv_tc k133 s11 128->256 @20x256x256 tile1x16x8 bn256 halo ln1 r0 p1 t0 st4",
    "conv_tc k133 s11 128->256 @4x128x128 tile1x16x8 bn256 halo ln1 r0 p1 t0 st4",
    "conv_tc k133 s11 256->128 @16x256x256 tile1x16x8 bn128 halo ln1 r0 p1 t0 st8",
    "conv_tc k133 s11 256->128 @20x256x256 tile1x16x8 bn128 halo ln1 r0 p1 t0 st8",
    "conv_tc k133 s11 256->128 @20x512x512 tile1x16x8 bn128 halo ln1 r0 p1 t0 st8",
    "conv_tc k133 s11 256->128 @8x256x256 tile1x16x8 bn128 halo ln1 r0 p1 t0 st8",
    "conv_tc k133 s11 256->256 @10x128x128 tile1x16x8 bn256 halo ln1 r0 p1 t0 st4",
    "conv_tc k133 s11 256->256 @10x128x128 tile1x16x8 bn256 halo ln2 r1m p1 t0 st4",
    "conv_tc k133 s11 256->256 @10x256x256 tile1x16x8 bn256 halo ln1 r0 p1 t0 st4",
    "conv_tc k133 s11 256->256 @10x256x256 tile1x16x8 bn256 halo ln2 r1m p1 t0 st4",
    "conv_tc k133 s11 256->256 @16x128x128 tile1x16x8 bn256 halo ln1 r0 p1 t0 st4",
    "conv_tc k133 s11 256->256 @16x128x128 tile1x16x8 bn256 halo ln2 r1m p1 t0 st4",
    "conv_tc k133 s11 256->256 @20x128x128 tile1x16x8 bn256 halo ln1 r0 p1 t0 st4",
    "conv_tc k133 s11 256->256 @20x128x128 tile1x16x8 bn256 halo ln2 r1m p1 t0 st4",
    "conv_tc k133 s11 256->256 @20x256x256 tile1x16x8 bn256 halo ln1 r0 p1 t0 st4",
    "conv_tc k133 s11 256->256 @20x256x256 tile1x16x8 bn256 halo ln2 r1m p1 t0 st4",
    "conv_tc k133 s11 256->256 @4x128x128 tile1x16x8 bn256 halo ln1 r0 p1 t0 st4",
    "conv_tc k133 s11 256->256 @4x128x128 tile1x16x8 bn256 halo ln2 r1m p1 t0 st4",
    "conv_tc k133 s11 256->256 @8x128x128 tile1x16x8 bn256 halo ln1 r0 p1 t0 st4",
    "conv_tc k133 s11 256->256 @8x128x128 tile1x16x8 bn256 halo ln2 r1m p1 t0 st4",
    "conv_tc k133 s11 256->512 @10x64x64 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4",
    "conv_tc k133 s11 256->512 @20x128x128 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4",
    "conv_tc k133 s11 256->512 @2x64x64 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4",
    "conv_tc k133 s11 256->512 @8x64x64 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4",
    "conv_tc k133 s11 512->256 @10x128x128 tile1x16x8 bn256 halo ln1 r0 p1 t0 st4",
    "conv_tc k133 s11 512->256 @10x256x256 tile1x16x8 bn256 halo ln1 r0 p1 t0 st4",
    "conv_tc k133 s11 512->256 @4x128x128 tile1x16x8 bn256 halo ln1 r0 p1 t0 st4",
    "conv_tc k133 s11 512->256 @8x128x128 tile1x16x8 bn256 halo ln1 r0 p1 t0 st4",
    "conv_tc k133 s11 512->512 @10x64x64 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4",
    "conv_tc k133 s11 512->512 @10x64x64 tile1x16x8 bn256 halo ln0 r1m p1 t0 st4",
    "conv_tc k133 s11 512->512 @1x32x32 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4",
    "conv_tc k133 s11 512->512 @1x32x32 tile1x16x8 bn256 halo ln0 r1m p1 t0 st4",
    "conv_tc k133 s11 512->512 @20x128x128 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4",
    "conv_tc k133 s11 512->512 @20x128x128 tile1x16x8 bn256 halo ln0 r1m p1 t0 st4",
    "conv_tc k133 s11 512->512 @2x32x32 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4",
    "conv_tc k133 s11 512->512 @2x32x32 tile1x16x8 bn256 halo ln0 r1m p1 t0 st4",
    "conv_tc k133 s11 512->512 @2x64x64 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4",
    "conv_tc k133 s11 512->512 @2x64x64 tile1x16x8 bn256 halo ln0 r1m p1 t0 st4",
    "conv_tc k133 s11 512->512 @4x32x32 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4",
    "conv_tc k133 s11 512->512 @4x32x32 tile1x16x8 bn256 halo ln0 r1m p1 t0 st4",
    "conv_tc k133 s11 512->512 @4x64x64 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4",
    "conv_tc k133 s11 512->512 @4x64x64 tile1x16x8 bn256 halo ln0 r1m p1 t0 st4",
    "conv_tc k133 s11 512->512 @5x128x128 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4",
    "conv_tc k133 s11 512->512 @5x128x128 tile1x16x8 bn256 halo ln0 r1m p1 t0 st4",
    "conv_tc k133 s11 512->512 @5x32x32 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4",
    "conv_tc k133 s11 512->512 @5x32x32 tile1x16x8 bn256 halo ln0 r1m p1 t0 st4",
    "conv_tc k133 s11 512->512 @5x64x64 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4",
    "conv_tc k133 s11 512->512 @5x64x64 tile1x16x8 bn256 halo ln0 r1m p1 t0 st4",
    "conv_tc k133 s11 512->512 @8x64x64 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4",
    "conv_tc k133 s11 512->512 @8x64x64 tile1x16x8 bn256 halo ln0 r1m p1 t0 st4",
    "conv_tc k133 s12 128->128 @16x128x128 tile1x8x16 bn128 ln2 r0 p1 t0 st6",
    "conv_tc k133 s12 128->128 @20x128x128 tile1x8x16 bn128 ln2 r0 p1 t0 st6",
    "conv_tc k133 s12 128->128 @20x256x256 tile1x8x16 bn128 ln2 r0 p1 t0 st6",
    "conv_tc k133 s12 128->128 @4x128x128 tile1x8x16 bn128 ln2 r0 p1 t0 st6",
    "conv_tc k133 s12 256->256 @16x64x64 tile1x8x16 bn256 ln0 r0 p1 t0 st4",
    "conv_tc k133 s12 256->256 @20x128x128 tile1x8x16 bn256 ln2 r0 p1 t0 st4",
    "conv_tc k133 s12 256->256 @20x64x64 tile1x8x16 bn256 ln0 r0 p1 t0 st4",
    "conv_tc k133 s12 256->256 @4x64x64 tile1x8x16 bn256 ln0 r0 p1 t0 st4",
    "conv_tc k133 s12 512->512 @10x32x32 tile1x8x16 bn256 ln0 r0 p1 t0 st4",
    "conv_tc k133 s12 512->512 @20x64x64 tile1x8x16 bn256 ln0 r0 p1 t0 st4",
    "conv_tc k133 s12 512->512 @2x32x32 tile1x8x16 bn256 ln0 r0 p1 t0 st4",
    "conv_tc k133 s12 512->512 @8x32x32 tile1x8x16 bn256 ln0 r0 p1 t0 st4",
    "conv_tc k233 s11 256->256 @10x256x256 tile1x16x8 bn256 halo ln2 r1 p1 t0 st4",
    "conv_tc k233 s11 256->256 @10x512x512 tile1x16x8 bn256 halo ln2 r1 p1 t0 st4",
    "conv_tc k233 s11 512->512 @5x128x128 tile1x16x8 bn256 halo ln0 r1 p1 t0 st4",
    "conv_tc k233 s11 512->512 @5x256x256 tile1x16x8 bn256 halo ln0 r1 p1 t0 st4",
    "conv_tc k311 s11 128->128 @16x256x256 tile1x8x16 bn128 ln0 r1m p1 t2 st6",
    "conv_tc k311 s11 128->128 @16x256x256 tile1x8x16 bn128 ln1 r0 p1 t2 st6",
    "conv_tc k311 s11 128->128 @16x256x256 tile1x8x16 bn128 ln2 r1m p1 t2 st6",
    "conv_tc k311 s11 128->128 @20x256x256 tile1x8x16 bn128 ln1 r0 p1 t2 st6",
    "conv_tc k311 s11 128->128 @20x256x256 tile1x8x16 bn128 ln2 r1m p1 t2 st6",
    "conv_tc k311 s11 128->128 @4x256x256 tile1x8x16 bn128 ln0 r1m p1 t1 st6",
    "conv_tc k311 s11 128->128 @4x256x256 tile1x8x16 bn128 ln1 r0 p1 t1 st6",
    "conv_tc k311 s11 128->128 @4x256x256 tile1x8x16 bn128 ln2 r1m p1 t1 st6",
    "conv_tc k311 s11 128->128 @8x256x256 tile1x8x16 bn128 ln1 r0 p1 t1 st6",
    "conv_tc k311 s11 128->128 @8x256x256 tile1x8x16 bn128 ln2 r1m p1 t1 st6",
    "conv_tc k311 s11 256->256 @10x128x128 tile1x8x16 bn256 ln0 r1m p1 t0 st4",
    "conv_tc k311 s11 256->256 @10x128x128 tile1x8x16 bn256 ln0 r1m p1 t2 st4",
    "conv_tc k311 s11 256->256 @10x128x128 tile1x8x16 bn256 ln1 r0 p1 t0 st4",
    "conv_tc k311 s11 256->256 @10x128x128 tile1x8x16 bn256 ln1 r0 p1 t2 st4",
    "conv_tc k311 s11 256->256 @10x128x128 tile1x8x16 bn256 ln2 r1m p1 t0 st4",
    "conv_tc k311 s11 256->256 @10x128x128 tile1x8x16 bn256 ln2 r1m p1 t2 st4",
    "conv_tc k311 s11 256->256 @10x256x256 tile1x8x16 bn256 ln0 r1m p1 t0 st4",
    "conv_tc k311 s11 256->256 @10x256x256 tile1x8x16 bn256 ln1 r0 p1 t0 st4",
    "conv_tc k311 s11 256->256 @10x256x256 tile1x8x16 bn256 ln2 r1m p1 t0 st4",
    "conv_tc k311 s11 256->256 @16x128x128 tile1x8x16 bn256 ln0 r1m p1 t2 st4",
    "conv_tc k311 s11 256->256 @16x128x128 tile1x8x16 bn256 ln1 r0 p1 t2 st4",
    "conv_tc k311 s11 256->256 @16x128x128 tile1x8x16 bn256 ln2 r1m p1 t2 st4",
    "conv_tc k311 s11 256->256 @20x128x128 tile1x8x16 bn256 ln0 r1m p1 t0 st4",
    "conv_tc k311 s11 256->256 @20x128x128 tile1x8x16 bn256 ln1 r0 p1 t0 st4",
    "conv_tc k311 s11 256->256 @20x128x128 tile1x8x16 bn256 ln2 r1m p1 t0 st4",
    "conv_tc k311 s11 256->256 @20x256x256 tile1x8x16 bn256 ln0 r1m p1 t0 st4",
    "conv_tc k311 s11 256->256 @20x256x256 tile1x8x16 bn256 ln1 r0 p1 t0 st4",
    "conv_tc k311 s11 256->256 @20x256x256 tile1x8x16 bn256 ln2 r1m p1 t0 st4",
    "conv_tc k311 s11 256->256 @4x128x128 tile1x8x16 bn256 ln0 r1m p1 t1 st4",
    "conv_tc k311 s11 256->256 @4x128x128 tile1x8x16 bn256 ln1 r0 p1 t1 st4",
    "conv_tc k311 s11 256->256 @4x128x128 tile1x8x16 bn256 ln2 r1m p1 t1 st4",
    "conv_tc k311 s11 256->256 @8x128x128 tile1x8x16 bn256 ln0 r1m p1 t2 st4",
    "conv_tc k311 s11 256->256 @8x128x128 tile1x8x16 bn256 ln1 r0 p1 t2 st4",
    "conv_tc k311 s11 256->256 @8x128x128 tile1x8x16 bn256 ln2 r1m p1 t2 st4",
    "conv_tc k311 s11 512->512 @10x64x64 tile1x8x16 bn256 ln0 r0 p1 t0 st4",
    "conv_tc k311 s11 512->512 @10x64x64 tile1x8x16 bn256 ln0 r1m p1 t0 st4",
    "conv_tc k311 s11 512->512 @1x32x32 tile1x8x16 bn256 ln0 r0 p1 t1 st4",
    "conv_tc k311 s11 512->512 @1x32x32 tile1x8x16 bn256 ln0 r1m p1 t1 st4",
    "conv_tc k311 s11 512->512 @20x128x128 tile1x8x16 bn256 ln0 r0 p1 t0 st4",
    "conv_tc k311 s11 512->512 @20x128x128 tile1x8x16 bn256 ln0 r1m p1 t0 st4",
    "conv_tc k311 s11 512->512 @2x32x32 tile1x8x16 bn256 ln0 r0 p1 t1 st4",
    "conv_tc k311 s11 512->512 @2x32x32 tile1x8x16 bn256 ln0 r1m p1 t1 st4",
    "conv_tc k311 s11 512->512 @2x64x64 tile1x8x16 bn256 ln0 r0 p1 t1 st4",
    "conv_tc k311 s11 512->512 @2x64x64 tile1x8x16 bn256 ln0 r1m p1 t1 st4",
    "conv_tc k311 s11 512->512 @4x32x32 tile1x8x16 bn256 ln0 r0 p1 t2 st4",
    "conv_tc k311 s11 512->512 @4x32x32 tile1x8x16 bn256 ln0 r1m p1 t2 st4",
    "conv_tc k311 s11 512->512 @4x64x64 tile1x8x16 bn256 ln0 r0 p1 t2 st4",
    "conv_tc k311 s11 512->512 @4x64x64 tile1x8x16 bn256 ln0 r1m p1 t2 st4",
    "conv_tc k311 s11 512->512 @5x128x128 tile1x8x16 bn256 ln0 r0 p1 t0 st4",
    "conv_tc k311 s11 512->512 @5x128x128 tile1x8x16 bn256 ln0 r1m p1 t0 st4",
    "conv_tc k311 s11 512->512 @5x32x32 tile1x8x16 bn256 ln0 r0 p1 t0 st4",
    "conv_tc k311 s11 512->512 @5x32x32 tile1x8x16 bn256 ln0 r0 p1 t2 st4",
    "conv_tc k311 s11 512->512 @5x32x32 tile1x8x16 bn256 ln0 r1m p1 t0 st4",
    "conv_tc k311 s11 512->512 @5x32x32 tile1x8x16 bn256 ln0 r1m p1 t2 st4",
    "conv_tc k311 s11 512->512 @5x64x64 tile1x8x16 bn256 ln0 r0 p1 t0 st4",
    "conv_tc k311 s11 512->512 @5x64x64 tile1x8x16 bn256 ln0 r0 p1 t2 st4",
    "conv_tc k311 s11 512->512 @5x64x64 tile1x8x16 bn256 ln0 r1m p1 t0 st4",
    "conv_tc k311 s11 512->512 @5x64x64 tile1x8x16 bn256 ln0 r1m p1 t2 st4",
    "conv_tc k311 s11 512->512 @8x64x64 tile1x8x16 bn256 ln0 r0 p1 t2 st4",
    "conv_tc k311 s11 512->512 @8x64x64 tile1x8x16 bn256 ln0 r1m p1 t2 st4",
    "conv_tc k333 s11 128->3 @16x256x256 tile1x16x8 bn32 halo ln0 r0 p1 t2 st8",
    "conv_tc k333 s11 128->3 @20x256x256 tile1x16x8 bn32 halo ln0 r0 p1 t2 st8",
    "conv_tc k333 s11 128->3 @8x256x256 tile1x16x8 bn32 halo ln0 r0 p1 t1 st8",
    "conv_tc k333 s11 256->256 @16x256x256 tile1x16x8 bn256 halo ln2 r1 p1 t2 st4",
    "conv_tc k333 s11 256->256 @20x256x256 tile1x16x8 bn256 halo ln2 r1 p1 t2 st4",
    "conv_tc k333 s11 256->256 @8x256x256 tile1x16x8 bn256 halo ln2 r1 p1 t1 st4",
    "conv_tc k333 s11 512->32 @1x32x32 tile1x16x8 bn32 halo ln0 r0 p1 t1 st8",
    "conv_tc k333 s11 512->32 @4x32x32 tile1x16x8 bn32 halo ln0 r0 p1 t2 st8",
    "conv_tc k333 s11 512->5 @5x32x32 tile1x16x8 bn32 halo ln0 r0 p1 t0 st8",
    "conv_tc k333 s11 512->512 @10x128x128 tile1x16x8 bn256 halo ln0 r1 p1 t2 st4",
    "conv_tc k333 s11 512->512 @1x32x32 tile1x16x8 bn256 halo ln0 r0 p1 t1 st4",
    "conv_tc k333 s11 512->512 @1x32x32 tile1x16x8 bn256 halo ln0 r1m p1 t1 st4",
    "conv_tc k333 s11 512->512 @2x32x32 tile1x16x8 bn256 halo ln0 r0 p1 t1 st4",
    "conv_tc k333 s11 512->512 @2x32x32 tile1x16x8 bn256 halo ln0 r1m p1 t1 st4",
    "conv_tc k333 s11 512->512 @4x128x128 tile1x16x8 bn256 halo ln0 r1 p1 t1 st4",
    "conv_tc k333 s11 512->512 @4x32x32 tile1x16x8 bn256 halo ln0 r0 p1 t2 st4",
    "conv_tc k333 s11 512->512 @4x32x32 tile1x16x8 bn256 halo ln0 r1m p1 t2 st4",
    "conv_tc k333 s11 512->512 @5x32x32 tile1x16x8 bn256 halo ln0 r0 p1 t0 st4",
    "conv_tc k333 s11 512->512 @5x32x32 tile1x16x8 bn256 halo ln0 r0 p1 t2 st4",
    "conv_tc k333 s11 512->512 @5x32x32 tile1x16x8 bn256 halo ln0 r1m p1 t0 st4",
    "conv_tc k333 s11 512->512 @5x32x32 tile1x16x8 bn256 halo ln0 r1m p1 t2 st4",
    "conv_tc k333 s11 512->512 @8x128x128 tile1x16x8 bn256 halo ln0 r1 p1 t2 st4",
    "conv_tc k333 s11 512->8 @5x32x32 tile1x16x8 bn32 halo ln0 r0 p1 t0 st8",
    "conv_tc k333 s21 256->256 @10x64x64 tile1x16x8 bn256 halo ln2 r3 p1 t0 st4",
    "conv_tc k333 s21 256->256 @2x64x64 tile1x16x8 bn256 halo ln2 r3 p1 t1 st4",
    "conv_tc k333 s21 256->256 @8x64x64 tile1x16x8 bn256 halo ln2 r3 p1 t2 st4",
    "conv_tc k333 s21 512->512 @10x64x64 tile1x16x8 bn256 halo ln0 r3 p1 t0 st4",
    "conv_tc k333 s21 512->512 @1x32x32 tile1x16x8 bn256 halo ln0 r3 p1 t1 st4",
    "conv_tc k333 s21 512->512 @4x32x32 tile1x16x8 bn256 halo ln0 r3 p1 t2 st4",
    "conv_tc k333 s21 512->512 @5x32x32 tile1x16x8 bn256 halo ln0 r3 p1 t0 st4",
    "conv_tc3 k111 s11 1024->512 @1x32x32 tile1x8x16 bn128 ln0 r0 p4 t0 st3",
    "conv_tc3 k111 s11 1024->512 @1x32x32 tile1x8x16 bn256 ln0 r0 p1 t0 st2",
    "conv_tc3 k111 s11 128->256 @16x128x128 tile1x8x16 bn256 ln0 r0 p1 t0 st2",
    "conv_tc3 k111 s11 128->256 @20x128x128 tile1x8x16 bn256 ln0 r0 p1 t0 st2",
    "conv_tc3 k111 s11 128->256 @20x256x256 tile1x8x16 bn256 ln0 r0 p1 t0 st2",
    "conv_tc3 k111 s11 128->256 @4x128x128 tile1x8x16 bn256 ln0 r0 p1 t0 st2",
    "conv_tc3 k111 s11 256->128 @16x256x256 tile1x8x16 bn128 ln0 r0 p1 t0 st3",
    "conv_tc3 k111 s11 256->128 @20x256x256 tile1x8x16 bn128 ln0 r0 p1 t0 st3",
    "conv_tc3 k111 s11 256->128 @20x512x512 tile1x8x16 bn128 ln0 r0 p1 t0 st3",
    "conv_tc3 k111 s11 256->128 @8x256x256 tile1x8x16 bn128 ln0 r0 p1 t0 st3",
    "conv_tc3 k111 s11 256->512 @10x64x64 tile1x8x16 bn256 ln0 r0 p1 t0 st2",
    "conv_tc3 k111 s11 256->512 @20x128x128 tile1x8x16 bn256 ln0 r0 p1 t0 st2",
    "conv_tc3 k111 s11 256->512 @2x64x64 tile1x8x16 bn256 ln0 r0 p1 t0 st2",
    "conv_tc3 k111 s11 256->512 @8x64x64 tile1x8x16 bn256 ln0 r0 p1 t0 st2",
    "conv_tc3 k111 s11 512->1024 @1x32x32 tile1x8x16 bn256 ln0 r0 p1 t0 st2",
    "conv_tc3 k111 s11 512->256 @10x128x128 tile1x8x16 bn256 ln0 r0 p1 t0 st2",
    "conv_tc3 k111 s11 512->256 @10x256x256 tile1x8x16 bn256 ln0 r0 p1 t0 st2",
    "conv_tc3 k111 s11 512->256 @4x128x128 tile1x8x16 bn256 ln0 r0 p1 t0 st2",
    "conv_tc3 k111 s11 512->256 @8x128x128 tile1x8x16 bn256 ln0 r0 p1 t0 st2",
    "conv_tc3 k111 s11 512->512 @1x32x32 tile1x8x16 bn256 ln0 r0 p1 t0 st2",
    "conv_tc3 k111 s11 512->512 @1x32x32 tile1x8x16 bn256 ln0 r1m p1 t0 st2",
    "conv_tc3 k111 s11 512->512 @2x32x32 tile1x8x16 bn256 ln0 r0 p1 t0 st2",
    "conv_tc3 k111 s11 512->512 @2x32x32 tile1x8x16 bn256 ln0 r1m p1 t0 st2",
    "conv_tc3 k111 s11 512->512 @4x32x32 tile1x8x16 bn256 ln0 r0 p1 t0 st2",
    "conv_tc3 k111 s11 512->512 @4x32x32 tile1x8x16 bn256 ln0 r1m p1 t0 st2",
    "conv_tc3 k111 s11 512->512 @5x32x32 tile1x8x16 bn256 ln0 r0 p1 t0 st2",
    "conv_tc3 k111 s11 512->512 @5x32x32 tile1x8x16 bn256 ln0 r1m p1 t0 st2",
    "conv_tc3 k122 s11 256->256 @10x128x128 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2",
    "conv_tc3 k122 s11 256->256 @10x256x256 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2",
    "conv_tc3 k122 s11 256->256 @4x128x128 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2",
    "conv_tc3 k122 s11 256->256 @8x128x128 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2",
    "conv_tc3 k122 s11 512->512 @2x32x32 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2",
    "conv_tc3 k122 s11 512->512 @2x64x64 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2",
    "conv_tc3 k122 s11 512->512 @4x32x32 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2",
    "conv_tc3 k122 s11 512->512 @4x64x64 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2",
    "conv_tc3 k122 s11 512->512 @5x128x128 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2",
    "conv_tc3 k122 s11 512->512 @5x32x32 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2",
    "conv_tc3 k122 s11 512->512 @5x64x64 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2",
    "conv_tc3 k133 s11 128->128 @16x256x256 tile1x16x8 bn128 halo ln1 r0 p4 t0 st2",
    "conv_tc3 k133 s11 128->128 @16x256x256 tile1x16x8 bn128 halo ln2 r1m p4 t0 st2",
    "conv_tc3 k133 s11 128->128 @20x256x256 tile1x16x8 bn128 halo ln1 r0 p4 t0 st2",
    "conv_tc3 k133 s11 128->128 @20x256x256 tile1x16x8 bn128 halo ln2 r1m p4 t0 st2",
    "conv_tc3 k133 s11 128->128 @20x512x512 tile1x16x8 bn128 halo ln1 r0 p4 t0 st2",
    "conv_tc3 k133 s11 128->128 @20x512x512 tile1x16x8 bn128 halo ln2 r1m p4 t0 st2",
    "conv_tc3 k133 s11 128->128 @4x256x256 tile1x16x8 bn128 halo ln1 r0 p4 t0 st2",
    "conv_tc3 k133 s11 128->128 @4x256x256 tile1x16x8 bn128 halo ln2 r1m p4 t0 st2",
    "conv_tc3 k133 s11 128->128 @8x256x256 tile1x16x8 bn128 halo ln1 r0 p4 t0 st2",
    "conv_tc3 k133 s11 128->128 @8x256x256 tile1x16x8 bn128 halo ln2 r1m p4 t0 st2",
    "conv_tc3 k133 s11 128->256 @16x128x128 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2",
    "conv_tc3 k133 s11 128->256 @20x128x128 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2",
    "conv_tc3 k133 s11 128->256 @20x256x256 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2",
    "conv_tc3 k133 s11 128->256 @4x128x128 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2",
    "conv_tc3 k133 s11 256->128 @16x256x256 tile1x16x8 bn128 halo ln1 r0 p4 t0 st2",
    "conv_tc3 k133 s11 256->128 @20x256x256 tile1x16x8 bn128 halo ln1 r0 p4 t0 st2",
    "conv_tc3 k133 s11 256->128 @20x512x512 tile1x16x8 bn128 halo ln1 r0 p4 t0 st2",
    "conv_tc3 k133 s11 256->128 @8x256x256 tile1x16x8 bn128 halo ln1 r0 p4 t0 st2",
    "conv_tc3 k133 s11 256->256 @10x128x128 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2",
    "conv_tc3 k133 s11 256->256 @10x128x128 tile1x16x8 bn128 halo ln0 r1m p4 t0 st2",
    "conv_tc3 k133 s11 256->256 @10x256x256 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2",
    "conv_tc3 k133 s11 256->256 @10x256x256 tile1x16x8 bn128 halo ln0 r1m p4 t0 st2",
    "conv_tc3 k133 s11 256->256 @16x128x128 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2",
    "conv_tc3 k133 s11 256->256 @16x128x128 tile1x16x8 bn128 halo ln0 r1m p4 t0 st2",
    "conv_tc3 k133 s11 256->256 @20x128x128 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2",
    "conv_tc3 k133 s11 256->256 @20x128x128 tile1x16x8 bn128 halo ln0 r1m p4 t0 st2",
    "conv_tc3 k133 s11 256->256 @20x256x256 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2",
    "conv_tc3 k133 s11 256->256 @20x256x256 tile1x16x8 bn128 halo ln0 r1m p4 t0 st2",
    "conv_tc3 k133 s11 256->256 @4x128x128 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2",
    "conv_tc3 k133 s11 256->256 @4x128x128 tile1x16x8 bn128 halo ln0 r1m p4 t0 st2",
    "conv_tc3 k133 s11 256->256 @8x128x128 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2",
    "conv_tc3 k133 s11 256->256 @8x128x128 tile1x16x8 bn128 halo ln0 r1m p4 t0 st2",
    "conv_tc3 k133 s11 256->512 @10x64x64 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2",
    "conv_tc3 k133 s11 256->512 @20x128x128 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2",
    "conv_tc3 k133 s11 256->512 @2x64x64 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2",
    "conv_tc3 k133 s11 256->512 @8x64x64 tile1x16x8 bn128 halo ln0 r0 p4 t0 st2",
    "conv_tc3 k133 s11 512->256 @10x128x128 tile1x16x8 bn128 halo ln0 r0 p8 t0 st2",
    "conv_tc3 k133 s11 512->256 @10x256x256 tile1x16x8 bn128 halo ln0 r0 p8 t0 st2",
    "conv_tc3 k133 s11 512->256 @4x128x128 tile1x16x8 bn128 halo ln0 r0 p8 t0 st2",
    "conv_tc3 k133 s11 512->256 @8x128x128 tile1x16x8 bn128 halo ln0 r0 p8 t0 st2",
    "conv_tc3 k133 s11 512->512 @10x64x64 tile1x16x8 bn128 halo ln0 r0 p8 t0 st2",
    "conv_tc3 k133 s11 512->512 @10x64x64 tile1x16x8 bn128 halo ln0 r1m p8 t0 st2",
    "conv_tc3 k133 s11 512->512 @1x32x32 tile1x16x8 bn128 halo ln0 r0 p8 t0 st2",
    "conv_tc3 k133 s11 512->512 @1x32x32 tile1x16x8 bn128 halo ln0 r1m p8 t0 st2",
    "conv_tc3 k133 s11 512->512 @20x128x128 tile1x16x8 bn128 halo ln0 r0 p8 t0 st2",
    "conv_tc3 k133 s11 512->512 @20x128x128 tile1x16x8 bn128 halo ln0 r1m p8 t0 st2",
    "conv_tc3 k133 s11 512->512 @2x32x32 tile1x16x8 bn128 halo ln0 r0 p8 t0 st2",
    "conv_tc3 k133 s11 512->512 @2x32x32 tile1x16x8 bn128 halo ln0 r1m p8 t0 st2",
    "conv_tc3 k133 s11 512->512 @2x64x64 tile1x16x8 bn128 halo ln0 r0 p8 t0 st2",
    "conv_tc3 k133 s11 512->512 @2x64x64 tile1x16x8 bn128 halo ln0 r1m p8 t0 st2",
    "conv_tc3 k133 s11 512->512 @4x32x32 tile1x16x8 bn128 halo ln0 r0 p8 t0 st2",
    "conv_tc3 k133 s11 512->512 @4x32x32 tile1x16x8 bn128 halo ln0 r1m p8 t0 st2",
    "conv_tc3 k133 s11 512->512 @4x64x64 tile1x16x8 bn128 halo ln0 r0 p8 t0 st2",
    "conv_tc3 k133 s11 512->512 @4x64x64 tile1x16x8 bn128 halo ln0 r1m p8 t0 st2",
    "conv_tc3 k133 s11 512->512 @5x128x128 tile1x16x8 bn128 halo ln0 r0 p8 t0 st2",
    "conv_tc3 k133 s11 512->512 @5x128x128 tile1x16x8 bn128 halo ln0 r1m p8 t0 st2",
    "conv_tc3 k133 s11 512->512 @5x32x32 tile1x16x8 bn128 halo ln0 r0 p8 t0 st2",
    "conv_tc3 k133 s11 512->512 @5x32x32 tile1x16x8 bn128 halo ln0 r1m p8 t0 st2",
    "conv_tc3 k133 s11 512->512 @5x64x64 tile1x16x8 bn128 halo ln0 r0 p8 t0 st2",
    "conv_tc3 k133 s11 512->512 @5x64x64 tile1x16x8 bn128 halo ln0 r1m p8 t0 st2",
    "conv_tc3 k133 s11 512->512 @8x64x64 tile1x16x8 bn128 halo ln0 r0 p8 t0 st2",
    "conv_tc3 k133 s11 512->512 @8x64x64 tile1x16x8 bn128 halo ln0 r1m p8 t0 st2",
    "conv_tc3 k133 s12 128->128 @16x128x128 tile1x8x16 bn128 ln2 r0 p4 t0 st3",
    "conv_tc3 k133 s12 128->128 @20x128x128 tile1x8x16 bn128 ln2 r0 p4 t0 st3",
    "conv_tc3 k133 s12 128->128 @20x256x256 tile1x8x16 bn128 ln2 r0 p4 t0 st3",
    "conv_tc3 k133 s12 128->128 @4x128x128 tile1x8x16 bn128 ln2 r0 p4 t0 st3",
    "conv_tc3 k133 s12 256->256 @16x64x64 tile1x8x16 bn128 ln0 r0 p4 t0 st3",
    "conv_tc3 k133 s12 256->256 @20x128x128 tile1x8x16 bn128 ln0 r0 p4 t0 st3",
    "conv_tc3 k133 s12 256->256 @20x64x64 tile1x8x16 bn128 ln0 r0 p4 t0 st3",
    "conv_tc3 k133 s12 256->256 @4x64x64 tile1x8x16 bn128 ln0 r0 p4 t0 st3",
    "conv_tc3 k133 s12 512->512 @10x32x32 tile1x8x16 bn128 ln0 r0 p8 t0 st3",
    "conv_tc3 k133 s12 512->512 @20x64x64 tile1x8x16 bn128 ln0 r0 p8 t0 st3",
    "conv_tc3 k133 s12 512->512 @2x32x32 tile1x8x16 bn128 ln0 r0 p8 t0 st3",
    "conv_tc3 k133 s12 512->512 @8x32x32 tile1x8x16 bn128 ln0 r0 p8 t0 st3",
    "conv_tc3 k233 s11 256->256 @10x256x256 tile1x16x8 bn128 halo ln0 r1 p8 t0 st2",
    "conv_tc3 k233 s11 256->256 @10x512x512 tile1x16x8 bn128 halo ln0 r1 p8 t0 st2",
    "conv_tc3 k233 s11 512->512 @5x128x128 tile1x16x8 bn64 halo ln0 r1 p8 t0 st4",
    "conv_tc3 k233 s11 512->512 @5x256x256 tile1x16x8 bn64 halo ln0 r1 p8 t0 st4",
    "conv_tc3 k311 s11 128->128 @16x256x256 tile1x8x16 bn128 ln0 r1m p1 t2 st3",
    "conv_tc3 k311 s11 128->128 @16x256x256 tile1x8x16 bn128 ln1 r0 p1 t2 st3",
    "conv_tc3 k311 s11 128->128 @16x256x256 tile1x8x16 bn128 ln2 r1m p1 t2 st3",
    "conv_tc3 k311 s11 128->128 @20x256x256 tile1x8x16 bn128 ln0 r1m p1 t0 st3",
    "conv_tc3 k311 s11 128->128 @20x256x256 tile1x8x16 bn128 ln1 r0 p1 t0 st3",
    "conv_tc3 k311 s11 128->128 @20x256x256 tile1x8x16 bn128 ln1 r0 p1 t2 st3",
    "conv_tc3 k311 s11 128->128 @20x256x256 tile1x8x16 bn128 ln2 r1m p1 t0 st3",
    "conv_tc3 k311 s11 128->128 @20x256x256 tile1x8x16 bn128 ln2 r1m p1 t2 st3",
    "conv_tc3 k311 s11 128->128 @20x512x512 tile1x8x16 bn128 ln0 r1m p1 t0 st3",
    "conv_tc3 k311 s11 128->128 @20x512x512 tile1x8x16 bn128 ln1 r0 p1 t0 st3",
    "conv_tc3 k311 s11 128->128 @20x512x512 tile1x8x16 bn128 ln2 r1m p1 t0 st3",
    "conv_tc3 k311 s11 128->128 @4x256x256 tile1x8x16 bn128 ln0 r1m p1 t1 st3",
    "conv_tc3 k311 s11 128->128 @4x256x256 tile1x8x16 bn128 ln1 r0 p1 t1 st3",
    "conv_tc3 k311 s11 128->128 @4x256x256 tile1x8x16 bn128 ln2 r1m p1 t1 st3",
    "conv_tc3 k311 s11 128->128 @8x256x256 tile1x8x16 bn128 ln1 r0 p1 t1 st3",
    "conv_tc3 k311 s11 128->128 @8x256x256 tile1x8x16 bn128 ln2 r1m p1 t1 st3",
    "conv_tc3 k311 s11 256->256 @10x128x128 tile1x8x16 bn256 ln0 r1m p1 t0 st2",
    "conv_tc3 k311 s11 256->256 @10x128x128 tile1x8x16 bn256 ln0 r1m p1 t2 st2",
    "conv_tc3 k311 s11 256->256 @10x128x128 tile1x8x16 bn256 ln1 r0 p1 t0 st2",
    "conv_tc3 k311 s11 256->256 @10x128x128 tile1x8x16 bn256 ln1 r0 p1 t2 st2",
    "conv_tc3 k311 s11 256->256 @10x128x128 tile1x8x16 bn256 ln2 r1m p1 t0 st2",
    "conv_tc3 k311 s11 256->256 @10x128x128 tile1x8x16 bn256 ln2 r1m p1 t2 st2",
    "conv_tc3 k311 s11 256->256 @10x256x256 tile1x8x16 bn256 ln0 r1m p1 t0 st2",
    "conv_tc3 k311 s11 256->256 @10x256x256 tile1x8x16 bn256 ln1 r0 p1 t0 st2",
    "conv_tc3 k311 s11 256->256 @10x256x256 tile1x8x16 bn256 ln2 r1m p1 t0 st2",
    "conv_tc3 k311 s11 256->256 @16x128x128 tile1x8x16 bn256 ln0 r1m p1 t2 st2",
    "conv_tc3 k311 s11 256->256 @16x128x128 tile1x8x16 bn256 ln1 r0 p1 t2 st2",
    "conv_tc3 k311 s11 256->256 @16x128x128 tile1x8x16 bn256 ln2 r1m p1 t2 st2",
    "conv_tc3 k311 s11 256->256 @20x128x128 tile1x8x16 bn256 ln0 r1m p1 t0 st2",
    "conv_tc3 k311 s11 256->256 @20x128x128 tile1x8x16 bn256 ln1 r0 p1 t0 st2",
    "conv_tc3 k311 s11 256->256 @20x128x128 tile1x8x16 bn256 ln2 r1m p1 t0 st2",
    "conv_tc3 k311 s11 256->256 @20x256x256 tile1x8x16 bn256 ln0 r1m p1 t0 st2",
    "conv_tc3 k311 s11 256->256 @20x256x256 tile1x8x16 bn256 ln1 r0 p1 t0 st2",
    "conv_tc3 k311 s11 256->256 @20x256x256 tile1x8x16 bn256 ln2 r1m p1 t0 st2",
    "conv_tc3 k311 s11 256->256 @4x128x128 tile1x8x16 bn256 ln0 r1m p1 t1 st2",
    "conv_tc3 k311 s11 256->256 @4x128x128 tile1x8x16 bn256 ln1 r0 p1 t1 st2",
    "conv_tc3 k311 s11 256->256 @4x128x128 tile1x8x16 bn256 ln2 r1m p1 t1 st2",
    "conv_tc3 k311 s11 256->256 @8x128x128 tile1x8x16 bn256 ln0 r1m p1 t2 st2",
    "conv_tc3 k311 s11 256->256 @8x128x128 tile1x8x16 bn256 ln1 r0 p1 t2 st2",
    "conv_tc3 k311 s11 256->256 @8x128x128 tile1x8x16 bn256 ln2 r1m p1 t2 st2",
    "conv_tc3 k311 s11 512->512 @10x64x64 tile1x8x16 bn128 ln0 r0 p4 t0 st3",
    "conv_tc3 k311 s11 512->512 @10x64x64 tile1x8x16 bn128 ln0 r1m p4 t0 st3",
    "conv_tc3 k311 s11 512->512 @1x32x32 tile1x8x16 bn128 ln0 r0 p4 t1 st3",
    "conv_tc3 k311 s11 512->512 @1x32x32 tile1x8x16 bn128 ln0 r1m p4 t1 st3",
    "conv_tc3 k311 s11 512->512 @20x128x128 tile1x8x16 bn128 ln0 r0 p4 t0 st3",
    "conv_tc3 k311 s11 512->512 @20x128x128 tile1x8x16 bn128 ln0 r1m p4 t0 st3",
    "conv_tc3 k311 s11 512->512 @2x32x32 tile1x8x16 bn128 ln0 r0 p4 t1 st3",
    "conv_tc3 k311 s11 512->512 @2x32x32 tile1x8x16 bn128 ln0 r1m p4 t1 st3",
    "conv_tc3 k311 s11 512->512 @2x64x64 tile1x8x16 bn128 ln0 r0 p4 t1 st3",
    "conv_tc3 k311 s11 512->512 @2x64x64 tile1x8x16 bn128 ln0 r1m p4 t1 st3",
    "conv_tc3 k311 s11 512->512 @4x32x32 tile1x8x16 bn128 ln0 r0 p4 t2 st3",
    "conv_tc3 k311 s11 512->512 @4x32x32 tile1x8x16 bn128 ln0 r1m p4 t2 st3",
    "conv_tc3 k311 s11 512->512 @4x64x64 tile1x8x16 bn128 ln0 r0 p4 t2 st3",
    "conv_tc3 k311 s11 512->512 @4x64x64 tile1x8x16 bn128 ln0 r1m p4 t2 st3",
    "conv_tc3 k311 s11 512->512 @5x128x128 tile1x8x16 bn128 ln0 r0 p4 t0 st3",
    "conv_tc3 k311 s11 512->512 @5x128x128 tile1x8x16 bn128 ln0 r1m p4 t0 st3",
    "conv_tc3 k311 s11 512->512 @5x32x32 tile1x8x16 bn128 ln0 r0 p4 t0 st3",
    "conv_tc3 k311 s11 512->512 @5x32x32 tile1x8x16 bn128 ln0 r0 p4 t2 st3",
    "conv_tc3 k311 s11 512->512 @5x32x32 tile1x8x16 bn128 ln0 r1m p4 t0 st3",
    "conv_tc3 k311 s11 512->512 @5x32x32 tile1x8x16 bn128 ln0 r1m p4 t2 st3",
    "conv_tc3 k311 s11 512->512 @5x64x64 tile1x8x16 bn128 ln0 r0 p4 t0 st3",
    "conv_tc3 k311 s11 512->512 @5x64x64 tile1x8x16 bn128 ln0 r0 p4 t2 st3",
    "conv_tc3 k311 s11 512->512 @5x64x64 tile1x8x16 bn128 ln0 r1m p4 t0 st3",
    "conv_tc3 k311 s11 512->512 @5x64x64 tile1x8x16 bn128 ln0 r1m p4 t2 st3",
    "conv_tc3 k311 s11 512->512 @8x64x64 tile1x8x16 bn128 ln0 r0 p4 t2 st3",
    "conv_tc3 k311 s11 512->512 @8x64x64 tile1x8x16 bn128 ln0 r1m p4 t2 st3",
    "conv_tc3 k333 s11 128->3 @16x256x256 tile1x16x8 bn32 halo ln0 r0 p4 t2 st8",
    "conv_tc3 k333 s11 128->3 @17x256x256 tile1x16x8 bn32 halo ln0 r0 p4 t0 st8",
    "conv_tc3 k333 s11 128->3 @17x512x512 tile1x16x8 bn32 halo ln0 r0 p4 t0 st8",
    "conv_tc3 k333 s11 128->3 @20x256x256 tile1x16x8 bn32 halo ln0 r0 p4 t2 st8",
    "conv_tc3 k333 s11 128->3 @8x256x256 tile1x16x8 bn32 halo ln0 r0 p4 t1 st8",
    "conv_tc3 k333 s11 256->256 @16x256x256 tile1x16x8 bn128 halo ln0 r1 p8 t2 st2",
    "conv_tc3 k333 s11 256->256 @20x256x256 tile1x16x8 bn128 halo ln0 r1 p8 t2 st2",
    "conv_tc3 k333 s11 256->256 @8x256x256 tile1x16x8 bn128 halo ln0 r1 p8 t1 st2",
    "conv_tc3 k333 s11 512->32 @1x32x32 tile1x16x8 bn32 halo ln0 r0 p8 t1 st7",
    "conv_tc3 k333 s11 512->32 @4x32x32 tile1x16x8 bn32 halo ln0 r0 p8 t2 st7",
    "conv_tc3 k333 s11 512->5 @5x32x32 tile1x16x8 bn32 halo ln0 r0 p8 t0 st7",
    "conv_tc3 k333 s11 512->512 @10x128x128 tile1x16x8 bn64 halo ln0 r1 p8 t2 st4",
    "conv_tc3 k333 s11 512->512 @1x32x32 tile1x16x8 bn64 halo ln0 r0 p8 t1 st4",
    "conv_tc3 k333 s11 512->512 @1x32x32 tile1x16x8 bn64 halo ln0 r1m p8 t1 st4",
    "conv_tc3 k333 s11 512->512 @2x32x32 tile1x16x8 bn64 halo ln0 r0 p8 t1 st4",
    "conv_tc3 k333 s11 512->512 @2x32x32 tile1x16x8 bn64 halo ln0 r1m p8 t1 st4",
    "conv_tc3 k333 s11 512->512 @4x128x128 tile1x16x8 bn64 halo ln0 r1 p8 t1 st4",
    "conv_tc3 k333 s11 512->512 @4x32x32 tile1x16x8 bn64 halo ln0 r0 p8 t2 st4",
    "conv_tc3 k333 s11 512->512 @4x32x32 tile1x16x8 bn64 halo ln0 r1m p8 t2 st4",
    "conv_tc3 k333 s11 512->512 @5x32x32 tile1x16x8 bn64 halo ln0 r0 p8 t0 st4",
    "conv_tc3 k333 s11 512->512 @5x32x32 tile1x16x8 bn64 halo ln0 r0 p8 t2 st4",
    "conv_tc3 k333 s11 512->512 @5x32x32 tile1x16x8 bn64 halo ln0 r1m p8 t0 st4",
    "conv_tc3 k333 s11 512->512 @5x32x32 tile1x16x8 bn64 halo ln0 r1m p8 t2 st4",
    "conv_tc3 k333 s11 512->512 @8x128x128 tile1x16x8 bn64 halo ln0 r1 p8 t2 st4",
    "conv_tc3 k333 s11 512->8 @5x32x32 tile1x16x8 bn32 halo ln0 r0 p8 t0 st7",
    "conv_tc3 k333 s21 256->256 @10x64x64 tile1x16x8 bn128 halo ln0 r3 p8 t0 st2",
    "conv_tc3 k333 s21 256->256 @2x64x64 tile1x16x8 bn128 halo ln0 r3 p8 t1 st2",
    "conv_tc3 k333 s21 256->256 @8x64x64 tile1x16x8 bn128 halo ln0 r3 p8 t2 st2",
    "conv_tc3 k333 s21 512->512 @10x64x64 tile1x16x8 bn64 halo ln0 r3 p8 t0 st4",
    "conv_tc3 k333 s21 512->512 @1x32x32 tile1x16x8 bn64 halo ln0 r3 p8 t1 st4",
    "conv_tc3 k333 s21 512->512 @4x32x32 tile1x16x8 bn64 halo ln0 r3 p8 t2 st4",
    "conv_tc3 k333 s21 512->512 @5x32x32 tile1x16x8 bn64 halo ln0 r3 p8 t0 st4",
    "tblock_tc strip 1x128 T20 ln_out0",
    "tblock_tc strip 1x128 T20 ln_out1",
]

# run at B = 2 (batch strides of the activation, residual, cache and output maps)
BATCH2 = {
    "conv_stem k333 3->128 @20x256x256",
    "conv_tc k133 s11 128->128 @4x256x256 tile1x16x8 bn128 halo ln2 r1m p1 t0 st8",
    "conv_tc k333 s21 256->256 @8x64x64 tile1x16x8 bn256 halo ln2 r3 p1 t2 st4",
    "conv_tc3 k311 s11 256->256 @8x128x128 tile1x8x16 bn256 ln2 r1m p1 t2 st2",
    "conv_tc3 k333 s11 512->512 @5x32x32 tile1x16x8 bn64 halo ln0 r1m p8 t0 st4",
}
ATTENTION_FRAMES = 10


def run_case(key, B=None, **kw):
    import zlib
    p = parse(key)
    entry = entry_of(p)
    if B is None and entry == "attention":
        # several frames share the launch (per-frame weights); one frame (a v1.1 chunk of one latent frame) plans like a
        # plain GEMM, with the narrow N tile and kparts of a long split K
        B = 1 if re.search(r" p[48] ", key) else ATTENTION_FRAMES
    elif B is None:
        B = 2 if key in BATCH2 else 1
    return CASES[entry](p, prec_of(p), B, Rng(zlib.crc32(key.encode())), **kw)


def test_table_is_well_formed():
    assert len(set(PLAN_TABLE)) == len(PLAN_TABLE) and BATCH2 <= set(PLAN_TABLE)
    for key in PLAN_TABLE:
        entry_of(parse(key))


@pytest.mark.parametrize("key", PLAN_TABLE)
def test_plan_case(key):
    check_case(key, prec_of(parse(key)), run_case(key))


def test_bias_buffer_switches_between_n_tiles():
    """The epilogue double-buffers bias / gamma / beta (cbuf) and switches when a CTA's next tile has another n0: 512
    channels in N tiles of 64 (exact, long K) give 8 N tiles, and 132 persistent CTAs step through the tiles by 132, so
    consecutive tiles of a CTA differ in n0 whenever there are more than 132 tiles."""
    key = "conv_tc3 k333 s11 512->512 @5x32x32 tile1x16x8 bn64 halo ln0 r1m p8 t0 st4"
    p = parse(key)
    n_tiles = 512 // 64
    for B in (1, 2):
        tiles = B * p["T"] * (p["H"] // 16) * (p["W"] // 8) * n_tiles
        assert tiles > 132 and 132 % n_tiles != 0
        check_case(key, N.PREC_EXACT_TC, run_case(key, B=B))


def test_split_residual_through_mma_and_in_epilogue():
    """EXACT_TC weights carry a power-of-two scale 2^s.  With s <= 15 the residual is added by the tensor core as
    2^s I x R (r1m); with max|w| < 1/64 the scale is 2^16, whose identity is not exact in fp16, and the epilogue adds
    the residual instead (r1).  Both against fp64."""
    key = "conv_tc3 k333 s11 512->512 @5x32x32 tile1x16x8 bn64 halo ln0 r1m p8 t0 st4"
    check_case(key, N.PREC_EXACT_TC, run_case(key, B=1))
    check_case(key.replace(" r1m ", " r1 "), N.PREC_EXACT_TC, run_case(key, B=1, weight_scale=0.25))


# ---------------------------------------------------------------------------------------------------------------
# pipeline depth: the K order of a tile does not depend on the number of stages, so VT_TC_STAGES=2 is bit-identical
# ---------------------------------------------------------------------------------------------------------------
STAGE_KEYS = [   # one per conv_tc_kernel<BN, split> instantiation, halo and non-halo
    "conv_tc k333 s11 128->3 @8x256x256 tile1x16x8 bn32 halo ln0 r0 p1 t1 st8",
    "conv_tc k333 s11 64->64 @5x32x32 tile1x16x8 bn64 halo ln0 r1m p1 t0 st8",      # (not a production layer)
    "conv_tc k311 s11 128->128 @4x256x256 tile1x8x16 bn128 ln1 r0 p1 t1 st6",
    "conv_tc k133 s11 256->256 @10x128x128 tile1x16x8 bn256 halo ln2 r1m p1 t0 st4",
    "conv_tc k311 s11 512->512 @5x32x32 tile1x8x16 bn256 ln0 r1m p1 t2 st4",
    "conv_tc3 k333 s11 128->3 @8x256x256 tile1x16x8 bn32 halo ln0 r0 p4 t1 st8",
    "conv_tc3 k333 s11 512->512 @5x32x32 tile1x16x8 bn64 halo ln0 r1m p8 t0 st4",
    "conv_tc3 k311 s11 512->512 @5x32x32 tile1x8x16 bn128 ln0 r1m p4 t2 st3",
    "conv_tc3 k311 s11 256->256 @8x128x128 tile1x8x16 bn256 ln2 r1m p1 t2 st2",    # 2 stages already by default
]


def stage_digests():
    """{key: ([sha256 of each output], [launched plan keys])} of the STAGE_KEYS cases in this process"""
    import hashlib
    res = {}
    for key in STAGE_KEYS:
        keys, outs, _, _ = run_case(key, B=1)
        res[key] = ([hashlib.sha256(got.contiguous().cpu().numpy().tobytes()).hexdigest() for _, got, _, _ in outs], sorted(keys))
    return res


def test_two_stage_pipeline_is_bit_identical():
    import json
    here = os.path.dirname(os.path.abspath(__file__))
    code = ("import json, sys; sys.path[:0] = [%r, %r]; import test_gpu_production_plans as m; "
            "print('DIGESTS ' + json.dumps(m.stage_digests()))" % (here, os.path.dirname(here)))
    env = dict(os.environ, VT_TC_STAGES="2")
    torch.cuda.empty_cache()
    r = subprocess.run([sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code], env=env,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    line = [s for s in r.stdout.splitlines() if s.startswith("DIGESTS ")]
    assert len(line) == 1, r.stdout[-2000:]
    two = json.loads(line[0][len("DIGESTS "):])
    default = stage_digests()
    for key in STAGE_KEYS:
        d_out, d_keys = default[key]
        t_out, t_keys = two[key]
        conv_keys = [k for k in t_keys if k.startswith("conv_tc")]
        assert conv_keys and all(k.endswith(" st2") for k in conv_keys), t_keys
        print(f"[{key}] default {[k.rsplit(' ', 1)[1] for k in d_keys]} vs {[k.rsplit(' ', 1)[1] for k in t_keys]}")
        assert d_out == t_out, f"{key}: VT_TC_STAGES=2 changes the result"


# ---------------------------------------------------------------------------------------------------------------
# model level: coverage of the table, kl41616 batch independence
# ---------------------------------------------------------------------------------------------------------------
def bench_model(name):
    import bench
    from vidtok_b200.compat_util import instantiate_from_config
    from vidtok_b200.synth import synth_state_dict
    c = bench.CONFIGS[name]
    model = instantiate_from_config(bench.model_cfg(c))
    model.load_state_dict(synth_state_dict({k: tuple(v.shape) for k, v in model.state_dict().items()}, seed=0))
    model = model.cuda().eval()
    if c["tiling"]:
        model.use_tiling = True
        model.t_chunk_enc, model.t_chunk_dec, model.use_overlap = c["tiling"]
    return model, c


def test_bench_forward_keys_are_in_table():
    """one bf16 and one exact forward of each bench.py workload at B = 1 launches only plans that PLAN_TABLE tests"""
    from gpu_util import plan_keys
    from vidtok_b200.synth import synth_clip
    table, missing = set(PLAN_TABLE), {}
    for name in BENCH:
        model, c = bench_model(name)
        x = synth_clip(1, c["T"], c["H"], c["W"], seed=1234).cuda()
        for prec in ("bf16", "exact"):
            model.precision = prec
            torch.manual_seed(4321)
            with torch.no_grad():
                _, keys = plan_keys(lambda: model(x))
            assert keys, (name, prec)
            miss = sorted(set(keys) - table)
            print(f"[{name} {prec}] {len(keys)} plan keys, {len(miss)} not in the table")
            if miss:
                missing[f"{name} {prec}"] = miss
        del model
        torch.cuda.empty_cache()
    assert not missing, "plan keys without a production case:\n" + "\n".join(f"  {k}: {v}" for k, vs in missing.items() for v in vs)


def test_kl41616_batch_of_four_clips_is_independent():
    """bench.py kl41616: 4 clips of 17x512x512 in bf16 (level-0 activations of 2.28e9 elements, past 2^31).  Clip 3 run
    alone, with the noise it saw inside the batch, is bit-identical to clip 3 of the batch."""
    from vidtok_b200.synth import synth_clip
    model, c = bench_model("kl41616")
    model.precision = "bf16"
    x = synth_clip(4, c["T"], c["H"], c["W"], seed=5).cuda()
    with torch.no_grad():
        torch.manual_seed(99)
        noise = torch.randn(4, 4, 5, 32, 32)
        torch.manual_seed(99)
        za, da, _ = model(x)
        assert tuple(za.shape) == (4, 4, 5, 32, 32) and torch.isfinite(da).all()
        nat = model._rt.sync()
        z3, _, _, _ = nat.encode(x[3:4].contiguous(), noise[3:4].cuda().contiguous(), N.PREC_BF16)
        d3 = nat.decode(z3, False, N.PREC_BF16)
    assert torch.equal(z3, za[3:4]), "the latent of clip 3 depends on its batch neighbours"
    assert torch.equal(d3, da[3:4]), "the reconstruction of clip 3 depends on its batch neighbours"
