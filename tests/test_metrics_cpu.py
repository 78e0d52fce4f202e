"""Host side of vidtok_b200.metrics: the pooling rule, argument validation (which comes before any device work), an empty
Scorer, and the identity that lets a running mean over frames replace the evaluation script's groups of 16."""
import math
import os
import socket

import pytest
import torch
import torch.multiprocessing as mp

from vidtok_b200 import metrics
from vidtok_b200.compat_util import compute_psnr, compute_ssim


def test_ssim_pool_factor_is_pythons_round():
    for m in list(range(1, 1200)) + [1440, 2160, 4320]:
        want = max(1, round(m / 256))
        assert metrics.ssim_pool_factor(m, 5000) == want and metrics.ssim_pool_factor(5000, m) == want, m
    assert [metrics.ssim_pool_factor(s, s) for s in (384, 640, 896)] == [2, 2, 4]      # ties go to the even factor
    assert metrics.ssim_pool_factor(1080, 1920) == 4 and metrics.ssim_pool_factor(720, 1280) == 3


def test_frame_scores_validates_before_touching_the_device():
    x = torch.zeros(1, 3, 2, 32, 32)
    with pytest.raises(RuntimeError, match="CUDA tensors"):
        metrics.frame_scores(x, x)
    with pytest.raises(RuntimeError, match="CUDA tensors"):
        metrics.Scorer().update(x, x)
    with pytest.raises(ValueError, match="one shape"):
        metrics.frame_scores(x, torch.zeros(1, 3, 2, 32, 16))
    with pytest.raises(ValueError, match="one shape"):
        metrics.frame_scores(torch.zeros(3, 32, 32), torch.zeros(3, 32, 32))
    with pytest.raises(ValueError, match="float32, bfloat16 or float16"):
        metrics.frame_scores(x.double(), x.double())
    small = torch.zeros(1, 3, 2, 10, 64)
    with pytest.raises(ValueError, match=r"Input size: 10 x 64 \(10 x 64 pooled by 1\)"):
        metrics.frame_scores(small, small)
    with pytest.raises(ValueError, match=r"Input size: 64 x 10 "):
        metrics.Scorer().update(torch.zeros(2, 3, 64, 10), torch.zeros(2, 3, 64, 10))
    with pytest.raises(RuntimeError, match="CUDA tensors"):      # PSNR alone has no minimum size
        metrics.frame_scores(small, small, ssim=False)


def test_fresh_scorer_has_no_frames():
    s = metrics.Scorer()
    r = s.result()
    assert r["frames"] == 0 and math.isnan(r["psnr"]) and math.isnan(r["ssim"])
    s.reset()
    assert s.result(reduce=False)["frames"] == 0


def test_workspace_query_widens_its_products():
    from vidtok_b200 import _native as N
    L = N.lib()
    assert L.vt_frame_scores_workspace_bytes(8, 3, 17, 256, 256) == 8 * 3 * 17 * 4 * 8 * 8
    assert L.vt_frame_scores_workspace_bytes(1, 3, 2, 11, 11) == 1 * 3 * 2 * 8
    assert L.vt_frame_scores_workspace_bytes(1, 3, 2, 1080, 1920) == 6 * 8 * 9 * 8      # pooled 270 x 480, map 260 x 470
    assert L.vt_frame_scores_workspace_bytes(16, 3, 17, 2160, 3840) == 16 * 3 * 17 * 8 * 9 * 8     # 6.8e9 elements
    assert L.vt_frame_scores_workspace_bytes(0, 3, 2, 64, 64) == -1
    assert L.vt_frame_scores_workspace_bytes(1 << 20, 64, 64, 256, 256) == -1 and b"split the batch" in L.vt_last_error()


@pytest.mark.parametrize("frames", [17, 33])
def test_grouping_identity(frames):
    """The script's list -- each group's value once per frame of the group, groups of 16 -- has the mean of the per-frame
    values, because compute_psnr / compute_ssim of a group are means over its frames."""
    g = torch.Generator().manual_seed(frames)
    x = torch.rand(frames, 3, 24, 40, generator=g, dtype=torch.float64)
    y = (x + 0.1 * torch.randn(x.shape, generator=g, dtype=torch.float64)).clamp(0, 1)
    for fn in (compute_psnr, compute_ssim):
        script = []
        for a, b in zip(torch.split(x, 16), torch.split(y, 16)):
            script += [fn(a, b).item()] * a.shape[0]
        per_frame = [fn(x[i:i + 1], y[i:i + 1]).item() for i in range(frames)]
        assert abs(sum(script) / frames - sum(per_frame) / frames) <= 1e-12


def _rank(rank, world, port, q):
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    from vidtok_b200 import dist as vdist
    vdist.init_from_env("gloo")
    part = torch.tensor([[300.0, 9.0, 10.0], [150.5, 4.25, 5.0]], dtype=torch.float64)[rank]
    q.put((rank, vdist.global_scores(part), part.tolist(), metrics.Scorer().result()))
    vdist.barrier()
    torch.distributed.destroy_process_group()


def test_global_scores_sum_the_partials_over_ranks():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_rank, args=(r, 2, port, q)) for r in range(2)]
    [p.start() for p in procs]
    res = sorted(q.get(timeout=120) for _ in range(2))
    [p.join(timeout=60) for p in procs]
    assert all(p.exitcode == 0 for p in procs)
    for rank, got, part, empty in res:
        assert got == {"psnr": 450.5 / 15, "ssim": 13.25 / 15, "frames": 15}
        assert part == [[300.0, 9.0, 10.0], [150.5, 4.25, 5.0]][rank]      # the caller's partial is not overwritten
        assert empty["frames"] == 0                                         # a scorer without frames still joins the all-reduce
