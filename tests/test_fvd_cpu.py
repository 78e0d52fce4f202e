"""FVD without a GPU: the I3D state-dict layout, the library's I3D parameter table and load refusals, the oracle's end-point
shapes and preprocessing, the Frechet distance against scipy, the feature windows of Scorer and the all-reduce of the feature
statistics over two gloo ranks."""
import ctypes as C
import math
import os
import socket

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp
import torch.nn.functional as F

from oracle.i3d_oracle import fvd_fp64, i3d_fp64, preprocess, resized_size, synthetic_i3d_state
from vidtok_b200 import _native as N
from vidtok_b200.metrics import (I3D, I3D_ENDPOINTS, features_to_stats, fvd, fvd_from_stats, fvd_windows, i3d_state,
                                 i3d_state_shapes)


def test_state_layout():
    sd = synthetic_i3d_state(0)
    assert set(sd) == set(i3d_state_shapes())
    assert len([k for k in sd if k.endswith("conv3d.weight")]) == 58      # 57 units and the logits
    assert i3d_state(sd).keys() == sd.keys()
    tracked = dict(sd, **{k.replace("running_var", "num_batches_tracked"): torch.tensor(5) for k in sd if k.endswith("running_var")})
    assert i3d_state(tracked).keys() == sd.keys()
    missing = dict(sd)
    del missing["Mixed_4e.b2b.bn.running_mean"]
    with pytest.raises(KeyError, match="Mixed_4e.b2b.bn.running_mean"):
        i3d_state(missing)
    bad = dict(sd, **{"Mixed_3c.b1b.conv3d.weight": torch.zeros(192, 128, 3, 3, 1)})
    with pytest.raises(ValueError, match="Mixed_3c.b1b.conv3d.weight"):
        i3d_state(bad)


def test_native_manifest_and_load_refusals():
    lib, h = N.lib(), C.c_void_p()
    N.check(lib.vt_i3d_create(0, C.byref(h)))
    try:
        native = {}
        for i in range(lib.vt_i3d_num_params(h)):
            name, shape, nd = C.create_string_buffer(128), (C.c_int64 * 5)(), C.c_int32()
            N.check(lib.vt_i3d_param_info(h, i, name, 128, shape, C.byref(nd)))
            native[name.value.decode()] = tuple(shape[:nd.value])
        assert native == i3d_state_shapes()
        assert lib.vt_i3d_param_info(h, len(native), None, 0, None, None) == -1
        assert lib.vt_last_error() == b"bad parameter index"
        buf = (C.c_float * 64)()
        assert lib.vt_i3d_load_param(h, b"Conv3d_1a_7x7.bn.scale", buf, 64, 0, None) == -1
        assert lib.vt_last_error() == b"unknown I3D parameter Conv3d_1a_7x7.bn.scale"
        assert lib.vt_i3d_load_param(h, b"Conv3d_1a_7x7.bn.bias", buf, 63, 0, None) == -1
        assert lib.vt_last_error() == b"parameter Conv3d_1a_7x7.bn.bias: expected 64 elements, got 63"
        N.check(lib.vt_i3d_load_param(h, b"Conv3d_1a_7x7.bn.bias", buf, 64, 0, None))   # host memory: no device needed
        assert lib.vt_i3d_finalize(h, None) == -3
        assert lib.vt_last_error() == b"I3D parameter Conv3d_1a_7x7.conv3d.weight was never loaded"
    finally:
        lib.vt_i3d_destroy(h)


def test_synthetic_state_is_seeded():
    a, b = synthetic_i3d_state(0), synthetic_i3d_state(0)
    assert all(torch.equal(a[k], b[k]) for k in a)
    assert not torch.equal(a["Conv3d_1a_7x7.conv3d.weight"], synthetic_i3d_state(1)["Conv3d_1a_7x7.conv3d.weight"])
    v = a["Mixed_4c.b1b.bn.running_var"]
    assert 0.8 <= float(v.min()) and float(v.max()) <= 1.2


def _meta_state():
    return {k: v.to("meta") for k, v in synthetic_i3d_state(0).items()}


# Mixed_5c time steps and channels of the table: T = 17 -> 3, 16 -> 2, 9 -> 2, 33 -> 5
@pytest.mark.parametrize("T,t5", [(9, 2), (16, 2), (17, 3), (33, 5)])
@pytest.mark.parametrize("H,W", [(256, 256), (224, 400), (1080, 1920)])
def test_end_point_shapes(T, t5, H, W):
    ep, feats = i3d_fp64(_meta_state(), torch.empty(2, 3, T, H, W, device="meta"))
    t1 = (T + 1) // 2
    t4 = (t1 + 1) // 2
    want = {"Conv3d_1a_7x7": (64, t1, 112), "MaxPool3d_2a_3x3": (64, t1, 56), "Conv3d_2b_1x1": (64, t1, 56),
            "Conv3d_2c_3x3": (192, t1, 56), "MaxPool3d_3a_3x3": (192, t1, 28), "Mixed_3b": (256, t1, 28),
            "Mixed_3c": (480, t1, 28), "MaxPool3d_4a_3x3": (480, t4, 14), "Mixed_4b": (512, t4, 14), "Mixed_4c": (512, t4, 14),
            "Mixed_4d": (512, t4, 14), "Mixed_4e": (528, t4, 14), "Mixed_4f": (832, t4, 14), "MaxPool3d_5a_2x2": (832, t5, 7),
            "Mixed_5b": (832, t5, 7), "Mixed_5c": (1024, t5, 7)}
    assert tuple(ep) == I3D_ENDPOINTS
    for name, (c, t, s) in want.items():
        assert tuple(ep[name].shape) == (2, c, t, s, s), name
    assert tuple(feats.shape) == (2, 400)


def test_short_clips_are_refused():
    with pytest.raises(ValueError, match="9 frames"):
        i3d_fp64(_meta_state(), torch.empty(1, 3, 8, 224, 224, device="meta"))


@pytest.mark.parametrize("H,W", [(256, 256), (224, 400), (1080, 1920), (300, 200), (224, 224)])
def test_preprocessing_is_the_literal_chain(H, W):
    g = torch.Generator().manual_seed(H * W)
    x = torch.rand(1, 3, 2, H, W, generator=g) * 2.4 - 1.2
    h, w = resized_size(H, W)
    assert min(h, w) == 224 and max(h, w) == math.ceil(max(H, W) * 224 / min(H, W))
    frames = ((x.clamp(-1, 1) + 1) / 2)[0].transpose(0, 1)
    r = F.interpolate(frames, size=(h, w), mode="bilinear", align_corners=False)
    r = r[:, :, (h - 224) // 2:(h - 224) // 2 + 224, (w - 224) // 2:(w - 224) // 2 + 224]
    want = ((r - 0.5) * 2).transpose(0, 1)[None]
    assert torch.equal(preprocess(x), want)


def _sqrtm_fvd(fa, fb):
    import scipy.linalg
    a, b = fa.double().numpy(), fb.double().numpy()
    m1, m2 = a.mean(0), b.mean(0)
    s1, s2 = np.cov(a, rowvar=False), np.cov(b, rowvar=False)
    covmean = scipy.linalg.sqrtm(s1 @ s2)
    return float(((m1 - m2) ** 2).sum() + np.trace(s1) + np.trace(s2) - 2 * np.trace(covmean).real)


def _nuclear_fvd(fa, fb):
    """the exact form for n <= 400: tr sqrt(S1 S2) is the sum of the singular values of D1 D2^T / (n - 1), D the centred sets"""
    a, b = fa.double().numpy(), fb.double().numpy()
    m1, m2 = a.mean(0), b.mean(0)
    n = a.shape[0]
    k = (a - m1) @ (b - m2).T / (n - 1)
    s1, s2 = np.cov(a, rowvar=False), np.cov(b, rowvar=False)
    return float(((m1 - m2) ** 2).sum() + np.trace(s1) + np.trace(s2) - 2 * np.linalg.svd(k, compute_uv=False).sum())


# n < 400: the covariances are singular, and the square roots of their zero eigenvalues' rounding noise move scipy's sqrtm by
# up to ~6e-8 of the distance; fvd_from_stats drops the eigenvalues beyond the rank and is checked against the exact form there.
@pytest.mark.parametrize("n,tol", [(600, 1e-9), (300, 1e-7), (64, 1e-7)])
def test_frechet_distance_against_scipy(n, tol):
    g = torch.Generator().manual_seed(n)
    mix = torch.randn(400, 400, generator=g) / 20
    fa = torch.randn(n, 400, generator=g) @ mix + 0.3
    fb = torch.randn(n, 400, generator=g) @ (mix * 1.3) + 0.1 * torch.randn(400, generator=g)
    want = _sqrtm_fvd(fa, fb)
    got = fvd_from_stats(features_to_stats(fa), features_to_stats(fb))
    print(f"n {n}: eigh {got:.12f} sqrtm {want:.12f}")
    assert abs(got - want) <= tol * abs(want)
    if n < 400:
        exact = _nuclear_fvd(fa, fb)
        print(f"exact {exact:.12f}")
        assert abs(got - exact) <= 1e-9 * abs(exact)
    assert abs(fvd(fa, fb) - got) <= 1e-12 * abs(got)
    assert abs(fvd_fp64(fa, fb) - got) <= tol * abs(got)
    assert abs(fvd(fa, fa)) <= 1e-9 * float(torch.cov(fa.double().T).trace())


def test_windows():
    x = torch.arange(2 * 3 * 20 * 2 * 2, dtype=torch.float32).reshape(2, 3, 20, 2, 2)
    w = fvd_windows(x, 9)
    assert w.shape == (4, 3, 9, 2, 2)
    assert torch.equal(w[1], x[0, :, 9:18]) and torch.equal(w[2], x[1, :, 0:9])
    assert fvd_windows(x, None) is x
    with pytest.raises(ValueError):
        fvd_windows(x, 21)


def test_from_files_never_downloads(tmp_path):
    path = str(tmp_path / "nowhere" / "i3d_pretrained_400.pt")
    with pytest.raises(FileNotFoundError, match="nowhere"):
        I3D.from_files(path)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _features(n, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n, 400, generator=g) * 0.7 + 0.2, torch.randn(n, 400, generator=g) * 0.9


def _worker(rank, world, port, q):
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    from vidtok_b200 import dist as vdist
    from vidtok_b200.metrics import Scorer
    vdist.init_from_env("gloo")
    fa, fb = _features(13, 1)
    s, e = vdist.shard_range(13, rank, world)
    # the statistics a Scorer with an I3D model keeps on this rank, then its result() on them
    scorer = Scorer.__new__(Scorer)
    Scorer.__init__(scorer)
    scorer._i3d = object()
    scorer._facc = torch.stack([features_to_stats(fa[s:e]), features_to_stats(fb[s:e])])
    r = scorer._result_fvd(torch.zeros(3, dtype=torch.float64), True)
    q.put((rank, r["fvd"], r["fvd_clips"]))
    vdist.barrier()
    torch.distributed.destroy_process_group()


def test_scorer_statistics_combine_over_two_ranks():
    world, port = 2, _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    [p.start() for p in procs]
    res = sorted(q.get(timeout=120) for _ in range(world))
    [p.join(timeout=60) for p in procs]
    assert all(p.exitcode == 0 for p in procs)
    fa, fb = _features(13, 1)
    want = fvd(fa, fb)
    for _, got, n in res:
        assert n == 13 and abs(got - want) <= 1e-9 * abs(want)
