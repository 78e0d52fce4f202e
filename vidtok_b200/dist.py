"""Multi-GPU plumbing for batch-sharded inference (SURVEY.md section 8e).

Clips are independent, so the batch is partitioned contiguously across ranks (one process per GPU, launched by
torchrun), weights are replicated, and encode/decode involve NO communication.  The only collectives are at the
end: an all-reduce of the PSNR partial sums (2 floats per rank) and, optionally, an all-gather of the
reconstructions.  The reference has no inference-time collective at all (its only explicit one,
vidtok/modules/regularizers.py:49-54, sits in the FSQ training loss); this mirrors what a multi-GPU run of
scripts/inference_evaluate.py would need.

Backend: "nccl" on GPUs (NVLink 5 / NVSwitch), "gloo" in the CPU tests.
"""
from __future__ import annotations

import os
from typing import List, Optional, Tuple

import torch
import torch.distributed as dist


def init_from_env(backend: Optional[str] = None) -> Tuple[int, int, int]:
    """(rank, world_size, local_rank) from torchrun's environment; initialises the default process group if
    WORLD_SIZE > 1."""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if world > 1 and not dist.is_initialized():
        if backend is None:
            backend = "nccl" if torch.cuda.is_available() else "gloo"
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29500")
        if backend == "nccl":
            torch.cuda.set_device(local)
            dist.init_process_group(backend, rank=rank, world_size=world, device_id=torch.device("cuda", local))
        else:
            dist.init_process_group(backend, rank=rank, world_size=world)
    return rank, world, local


def shard_range(n_items: int, rank: int, world: int) -> Tuple[int, int]:
    """Contiguous, balanced partition: the first (n % world) ranks get one extra item."""
    base, rem = divmod(n_items, world)
    start = rank * base + min(rank, rem)
    return start, start + base + (1 if rank < rem else 0)


def psnr_partial(x: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
    """Per-frame PSNR partial sums [sum_of_frame_psnr, n_frames] for [B,C,T,H,W] tensors in [-1,1]
    (clamp + (x+1)/2 as scripts/inference_evaluate.py:175-176, metric as vidtok/modules/util.py:146-155)."""
    x01 = (x.clamp(-1, 1) + 1) / 2
    y01 = (y.clamp(-1, 1) + 1) / 2
    mse = ((x01 - y01) ** 2).mean(dim=(1, 3, 4))  # [B,T]
    ps = -10.0 * torch.log10(mse + 1e-8)
    return torch.stack([ps.double().sum(), torch.tensor(float(ps.numel()), dtype=torch.float64, device=ps.device)])


def allreduce_sum(t: torch.Tensor) -> torch.Tensor:
    if dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(t, op=dist.ReduceOp.SUM)
    return t


def allreduce_max(t: torch.Tensor) -> torch.Tensor:
    if dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return t


def global_psnr(partial: torch.Tensor) -> float:
    p = allreduce_sum(partial.clone())
    return float(p[0] / p[1])


def score_partial(x: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
    """This rank's double [sum of frame PSNR, sum of frame SSIM, n_frames] for CUDA tensors [B,C,T,H,W] (or [N,C,H,W]) in
    [-1,1]: the fused kernel of vidtok_b200.metrics (clamp + (x+1)/2 inside it), no host synchronisation."""
    from .metrics import Scorer
    scorer = Scorer()
    scorer.update(x, y)
    return scorer.sums()


def global_scores(partial: torch.Tensor) -> dict:
    """{"psnr", "ssim", "frames"} of the partials of score_partial summed over the ranks (one all-reduce of 3 doubles)."""
    from .metrics import _means
    return _means(allreduce_sum(partial.clone()))


def gather_clips(local: torch.Tensor, counts: List[int]) -> Optional[torch.Tensor]:
    """All-gather of per-rank reconstructions with possibly different clip counts (pads to the max count)."""
    if not (dist.is_initialized() and dist.get_world_size() > 1):
        return local
    world = dist.get_world_size()
    mx = max(counts)
    pad = local
    if local.shape[0] < mx:
        pad = torch.cat([local, local.new_zeros((mx - local.shape[0],) + tuple(local.shape[1:]))], dim=0)
    out = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(out, pad.contiguous())
    return torch.cat([o[:c] for o, c in zip(out, counts)], dim=0)


def barrier():
    if dist.is_initialized() and dist.get_world_size() > 1:
        dist.barrier()
