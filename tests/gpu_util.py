"""Helpers for the -m gpu parity tests: thin ctypes callers of the single-operator entry points."""
import ctypes as C

import torch

from vidtok_b200 import _native as N


def _p(t):
    return C.c_void_p(0 if t is None else t.data_ptr())


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def split_rows(x):
    """fp32 [..., C] -> the EXACT_TC activation format [..., hi(C) | lo(C)]: two fp16 planes, value = hi + lo
    (11 + 11 mantissa bits; saturating at the fp16 range)."""
    hi = x.clamp(-65504.0, 65504.0).to(torch.float16)
    lo = (x - hi.float()).clamp(-65504.0, 65504.0).to(torch.float16)
    return torch.cat([hi, lo], dim=-1).contiguous()


def join_rows(y):
    c = y.shape[-1] // 2
    return y[..., :c].float() + y[..., c:].float()


def act_dtype(precision):
    return {N.PREC_FMA32: torch.float32, N.PREC_BF16: torch.bfloat16, N.PREC_EXACT_TC: torch.float16}[precision]


def to_act(x_cl, precision):
    """channels-last fp32 tensor (cpu or cuda) -> cuda tensor in the precision's activation format."""
    x_cl = x_cl.contiguous().cuda()
    if precision == N.PREC_FMA32:
        return x_cl.float()
    if precision == N.PREC_BF16:
        return x_cl.to(torch.bfloat16)
    return split_rows(x_cl.float())


def from_act(y, precision):
    """activation-format cuda tensor -> fp32 cpu tensor (channels-last)."""
    if precision == N.PREC_EXACT_TC:
        return join_rows(y).cpu()
    return y.float().cpu()


def empty_act(shape_cl, precision):
    """uninitialised channels-last activation [..., C] in the precision's format"""
    shape = list(shape_cl)
    if precision == N.PREC_EXACT_TC:
        shape[-1] *= 2
    return torch.empty(shape, dtype=act_dtype(precision), device="cuda")


def to_cl(x, dtype):
    """[B,C,T,H,W] cpu -> channels-last [B,T,H,W,C] cuda"""
    return x.permute(0, 2, 3, 4, 1).contiguous().to("cuda", dtype)


def from_cl(y):
    return y.float().cpu().permute(0, 4, 1, 2, 3).contiguous()


def cl(x):
    """[B,C,T,H,W] -> [B,T,H,W,C]"""
    return x.permute(0, 2, 3, 4, 1).contiguous()


def ncdhw(y_cl):
    return y_cl.permute(0, 4, 1, 2, 3).contiguous()


def conv_desc(x_shape, w_shape, stride=(1, 1, 1), pt=None, pads=None, up=(1, 1, 1), res_mode=0, alpha=0.0):
    B, Ci, T, H, W = x_shape
    Co, _, kt, kh, kw = w_shape
    d = N.ConvDesc()
    d.B, d.Ti, d.Hi, d.Wi, d.Ci, d.Co = B, T, H, W, Ci, Co
    d.kt, d.kh, d.kw = kt, kh, kw
    d.st, d.sh, d.sw = stride
    d.pt = (kt - 1) + (1 - stride[0]) if pt is None else pt
    if pads is None:
        hp, wp = (kh - 1) + (1 - stride[1]), (kw - 1) + (1 - stride[2])
        pads = (hp // 2, hp - hp // 2, wp // 2, wp - wp // 2)
    d.ph0, d.ph1, d.pw0, d.pw1 = pads
    d.ut, d.uh, d.uw = up
    d.res_mode, d.alpha = res_mode, alpha
    To = (up[0] * T + d.pt - kt) // stride[0] + 1
    Ho = (up[1] * H + pads[0] + pads[1] - kh) // stride[1] + 1
    Wo = (up[2] * W + pads[2] + pads[3] - kw) // stride[2] + 1
    return d, (To, Ho, Wo)


def op_conv(x, w, b, *, stride=(1, 1, 1), pt=None, pads=None, up=(1, 1, 1), res=None, res_mode=0, alpha=0.0,
            precision=N.PREC_FMA32, force_simt=False):
    """x [B,Ci,T,H,W], w [Co,Ci,kt,kh,kw] (cpu fp32) -> [B,Co,To,Ho,Wo] cpu fp32 via vt_op_conv."""
    d, (To, Ho, Wo) = conv_desc(x.shape, w.shape, stride, pt, pads, up, res_mode, alpha)
    B, Co = x.shape[0], w.shape[0]
    xc = to_act(cl(x), precision)
    wd, bd = w.contiguous().cuda(), b.contiguous().cuda()
    rc_ = to_act(cl(res), precision) if res is not None else None
    out = empty_act((B, To, Ho, Wo, Co), precision)
    N.check(N.lib().vt_op_conv(precision, int(force_simt), C.byref(d), _p(xc), _p(wd), _p(bd), _p(rc_), _p(out), stream()))
    torch.cuda.synchronize()
    return ncdhw(from_act(out, precision))


def op_conv_ex(x, w, b, *, precision, stride=(1, 1, 1), pads=None, res=None, res_mode=0, alpha=0.0, t_mode=0, cache=None,
               ln_mode=0, ln_silu=True, gamma=None, beta=None, to_off=0, out_f32=False, res_mix=False, res_t_mode=0,
               force_simt=False):
    """vt_op_conv_ex; returns (out, out2) as [B,Co,To,Ho,Wo] cpu fp32 (out2 None unless ln_mode == 2)."""
    d, (To, Ho, Wo) = conv_desc(x.shape, w.shape, stride, None, pads, (1, 1, 1), res_mode, alpha)
    e = N.ConvEx()
    e.d = d
    e.force_simt, e.t_mode, e.ln_mode, e.ln_silu, e.to_off = int(force_simt), t_mode, ln_mode, int(ln_silu), to_off
    e.out_f32_ncdhw, e.res_mix, e.res_t_mode = int(out_f32), int(res_mix), res_t_mode
    e.cacheT = 0 if cache is None else cache.shape[2]
    B, Co = x.shape[0], w.shape[0]
    To -= to_off
    xc = to_act(cl(x), precision)
    cc = to_act(cl(cache), precision) if cache is not None else None
    wd, bd = w.contiguous().cuda(), b.contiguous().cuda()
    rc_ = to_act(cl(res), precision) if res is not None else None
    gd = gamma.contiguous().cuda() if gamma is not None else None
    btd = beta.contiguous().cuda() if beta is not None else None
    if out_f32:
        out = torch.empty((B, Co, To, Ho, Wo), dtype=torch.float32, device="cuda")
    else:
        out = empty_act((B, To, Ho, Wo, Co), precision)
    out2 = empty_act((B, To, Ho, Wo, Co), precision) if ln_mode == 2 else None
    N.check(N.lib().vt_op_conv_ex(precision, C.byref(e), _p(xc), _p(cc), _p(wd), _p(bd), _p(rc_), _p(gd), _p(btd), _p(out),
                                  _p(out2), stream()))
    torch.cuda.synchronize()
    o1 = out.cpu() if out_f32 else ncdhw(from_act(out, precision))
    o2 = ncdhw(from_act(out2, precision)) if out2 is not None else None
    return o1, o2


def bf16_round(x):
    return x.to(torch.bfloat16).float()


# kernels whose launch plan (tile, N tile, halo windows, stages, kparts, residual path, ...) the detailed profiler names
PLAN_KERNELS = ("conv_tc", "conv_tc3", "tblock_tc", "conv_stem", "conv_stem3")


def plan_keys(fn):
    """run fn() under the library's detailed profiler -> (fn's result, {plan key: launches}) for the PLAN_KERNELS launches.
    A key is the kernel name and its detail string, e.g. 'conv_tc k333 s11 128->128 @17x256x256 tile1x16x8 bn128 halo ln1
    r0 p1 t0 st8'."""
    import json
    lib = N.lib()
    lib.vt_profile_start_detailed()
    try:
        out = fn()
    finally:
        buf = C.create_string_buffer(1 << 22)
        n = lib.vt_profile_stop(buf, len(buf))
    assert n > 0, "profile did not fit the buffer"
    prof = json.loads(buf.value.decode())
    return out, {k: v["launches"] for k, v in prof.items() if k.split(" ", 1)[0] in PLAN_KERNELS}
