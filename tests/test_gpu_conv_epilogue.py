"""conv_tc's bf16 output tiles through shared memory and bulk tensor stores (TcPlan::stage_out: the 256-channel N tiles),
next to the per-thread stores of the narrower N tiles, against fp64 torch with the bounds of test_gpu_ops_tc.py.

The staged epilogue hands whole 64-row x 64-channel boxes to TMA, which clips them at the tensor's edge, where the
per-thread stores tested every row.  So every case writes into the middle of a larger poisoned buffer that must come back
untouched around the tensor, and the geometries include outputs whose T, H, W are not multiples of the tile box.

The host-only part pins the dry-run workspace of the benchmark's four configurations: the staging buffers come out of
shared memory the plans left unused, so no plan, and no workspace, may change because of them."""
import ctypes as C
import math

import pytest
import torch

from vidtok_b200 import _native as N

BF16 = N.PREC_BF16
POISON = -12345.0
PAD = 4096           # poisoned elements in front of and behind the tensor (a multiple of 8: the tensor stays 16-byte aligned)


def _run(Ci, Co, k, shape, *, ln_mode=0, silu=True, res=0, out_shift=0):
    """one vt_op_conv_ex launch in bf16; res: 0 none, 1 `+ r` (through the MMA), 2 alpha-mix (added in the epilogue).
    out_shift: elements by which the output tensors are moved off 16-byte alignment.  Returns the fp64 references and
    the kernel's v / act(LN(v))."""
    from gpu_util import _p, cl, conv_desc, ncdhw, stream
    from test_gpu_ops_tc import conv3d_ref, ln_ref, prep, rnd
    B, T, H, W = shape
    K = Ci * k[0] * k[1] * k[2]
    x = prep(rnd(B, Ci, T, H, W, seed=1), BF16)
    w = prep(rnd(Co, Ci, *k, seed=2, scale=1 / math.sqrt(K)), BF16)
    b = rnd(Co, seed=3)
    g = 1.0 + 0.5 * rnd(Co, seed=5)
    bt = 0.3 * rnd(Co, seed=6) + torch.linspace(-0.5, 0.5, Co)
    v = conv3d_ref(x, w, b)
    r, alpha = None, 0.6
    if res:
        r = prep(rnd(*v.shape, seed=4), BF16)
        v = alpha * r.double() + (1 - alpha) * v if res == 2 else v + r.double()
    y = ln_ref(v, g, bt, silu) if ln_mode else None

    d, (To, Ho, Wo) = conv_desc(x.shape, w.shape, res_mode=1 if res else 0, alpha=alpha if res == 2 else 0.0)
    e = N.ConvEx()
    e.d = d
    e.ln_mode, e.ln_silu, e.res_mix = ln_mode, int(silu), int(res == 2)
    n = B * To * Ho * Wo * Co
    xd = cl(x).to("cuda", torch.bfloat16)
    rd = cl(r).to("cuda", torch.bfloat16) if r is not None else None
    wd, bd, gd, btd = w.cuda(), b.cuda(), g.cuda(), bt.cuda()
    bufs = [torch.full((n + 2 * PAD,), POISON, device="cuda", dtype=torch.bfloat16) for _ in range(2 if ln_mode == 2 else 1)]
    lo = PAD + out_shift
    ptrs = [C.c_void_p(t.data_ptr() + 2 * lo) for t in bufs]
    N.check(N.lib().vt_op_conv_ex(BF16, C.byref(e), _p(xd), None, _p(wd), _p(bd), _p(rd), _p(gd) if ln_mode else None,
                                  _p(btd) if ln_mode else None, ptrs[0], ptrs[1] if ln_mode == 2 else None, stream()))
    torch.cuda.synchronize()
    outs = []
    for t in bufs:
        assert bool((t[:lo] == POISON).all()) and bool((t[lo + n:] == POISON).all()), "stored outside the output tensor"
        outs.append(ncdhw(t[lo:lo + n].view(B, To, Ho, Wo, Co).float().cpu()))
    return v, y, outs


def _check(v, y, outs, ln_mode, what):
    from test_gpu_ops_tc import check
    if ln_mode == 1:
        check(outs[0], y, BF16, what + " act(LN(v))", slack=1.5)
    else:
        check(outs[0], v, BF16, what + " v")
        if ln_mode == 2:
            check(outs[1], y, BF16, what + " act(LN(v))", slack=1.5)


# name, Ci, Co, k, (B,T,H,W): N tiles of 256 (cooperative, staged) and of 64 / 128 (ping-pong, per-thread stores), two N
# tiles, halo windows and dense tiles, outputs that end inside a box in W, H and T
GEOMS = [
    ("bn64_halo", 64, 64, (1, 3, 3), (1, 2, 32, 32)),
    ("bn128_halo", 128, 128, (1, 3, 3), (2, 2, 48, 24)),
    ("bn256_halo_k233", 128, 256, (2, 3, 3), (1, 3, 32, 40)),
    ("bn256_two_ntiles", 64, 512, (1, 1, 1), (1, 2, 16, 16)),
    ("bn64_dense_ragged", 64, 64, (3, 3, 3), (1, 3, 12, 20)),
    ("bn128_dense_ragged_k311", 64, 128, (3, 1, 1), (2, 5, 10, 12)),
    ("bn256_dense_ragged", 128, 256, (1, 3, 3), (1, 3, 20, 28)),
    ("bn128_tiny", 64, 128, (1, 1, 1), (1, 1, 4, 4)),
]


@pytest.mark.gpu
@pytest.mark.parametrize("res", [0, 1, 2], ids=["r0", "r_mma", "r_mix"])
@pytest.mark.parametrize("ln_mode", [0, 1, 2], ids=["ln0", "ln1", "ln2"])
@pytest.mark.parametrize("geom", GEOMS, ids=[g[0] for g in GEOMS])
def test_staged_epilogue(geom, ln_mode, res):
    name, Ci, Co, k, shape = geom
    if ln_mode and Co > 256:
        pytest.skip("a fused LayerNorm needs one N tile over Cout")
    v, y, outs = _run(Ci, Co, k, shape, ln_mode=ln_mode, res=res)
    _check(v, y, outs, ln_mode, name)


@pytest.mark.gpu
@pytest.mark.parametrize("case", [("unaligned_out", 128, 256, 2), ("bn32", 64, 96, 0)], ids=lambda c: c[0])
def test_per_thread_stores_where_not_staged(case):
    """outputs that are not 16-byte aligned, and N tiles of 32 channels, keep the per-thread stores"""
    name, Ci, Co, shift = case
    for ln_mode in ((0, 2) if Co == 256 else (0,)):
        v, y, outs = _run(Ci, Co, (1, 3, 3), (1, 2, 20, 24), ln_mode=ln_mode, res=2, out_shift=shift)
        _check(v, y, outs, ln_mode, name)


# vt_workspace_bytes(B = 8) of the benchmark configurations before the staging buffers existed: bf16, exact
WORKSPACES = {
    "kl488": (17448964096, 33555091456),
    "fsq488": (17449127936, 33555255296),
    "v11long": (137322041344, 221476556800),
    "kl41616": (69793878016, 134218387456),
}


@pytest.mark.parametrize("cfg", ["kl488", "fsq488", "v11long", "kl41616"])
def test_workspace_of_benchmark_configurations_unchanged(cfg):
    import os
    import sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import bench
    from vidtok_b200.compat_util import instantiate_from_config
    from vidtok_b200.engine import NativeModel
    c = bench.CONFIGS[cfg]
    nm = NativeModel(instantiate_from_config(bench.model_cfg(c)).spec)
    got = tuple(int(N.lib().vt_workspace_bytes(nm.handle, prec, 8, c["T"], c["H"], c["W"])) for prec in (N.PREC_BF16, N.PREC_EXACT_TC))
    assert min(got) > 0, N.lib().vt_last_error()
    assert got == WORKSPACES[cfg]
