"""The evaluation protocol's quality numbers on the device (scripts/inference_evaluate.py:175-186): clamp to [-1,1], (v+1)/2,
then compute_psnr / compute_ssim (vidtok/modules/util.py:146-231), as one fused kernel of libvidtok_b200.so that reads the
input clip and the reconstruction once and returns the two scores of every frame.  Nothing here synchronises with the host
until a result is asked for.

The script clamps only the reconstruction; the kernel clamps both clips, which is the identity on an input in [-1,1].

The script scores groups of 16 frames and appends each group's value once per frame of the group; a group's value is the
mean of its frames' values, so the mean of that list is the mean over frames of the per-frame values, whatever the
grouping (tests/test_metrics_cpu.py::test_grouping_identity).  Scorer therefore keeps [sum of PSNR, sum of SSIM, frames]."""
from __future__ import annotations

import ctypes as C
import math

import torch

from . import _native as N

_DTYPES = {torch.float32: N.DTYPE_F32, torch.bfloat16: N.DTYPE_BF16, torch.float16: N.DTYPE_F16}
_WINDOW = 11


def ssim_pool_factor(H: int, W: int) -> int:
    """The factor compute_ssim average-pools a frame by: max(1, round(min(H, W) / 256)), Python's round (half to even:
    384 -> 2, 640 -> 2, 896 -> 4)."""
    return max(1, round(min(H, W) / 256))


def _geometry(x: torch.Tensor, y: torch.Tensor, ssim: bool):
    if x.dim() not in (4, 5) or x.shape != y.shape:
        raise ValueError(f"expected two clips [B,C,T,H,W] or two batches of frames [N,C,H,W] of one shape, got {tuple(x.shape)} and {tuple(y.shape)}")
    if x.dtype not in _DTYPES or y.dtype not in _DTYPES:
        raise ValueError(f"expected float32, bfloat16 or float16 tensors, got {x.dtype} and {y.dtype}")
    if x.numel() == 0:
        raise ValueError(f"empty clip {tuple(x.shape)}")
    B, Cc = x.shape[:2]
    T = x.shape[2] if x.dim() == 5 else 1
    H, W = x.shape[-2:]
    f = ssim_pool_factor(H, W)
    if ssim and (H // f < _WINDOW or W // f < _WINDOW):
        raise ValueError(f"SSIM kernel size can't be greater than actual input size. Input size: {H // f} x {W // f} "
                         f"({H} x {W} pooled by {f}). Kernel size: {_WINDOW} x {_WINDOW}")
    if not (x.is_cuda and y.is_cuda):
        raise RuntimeError("vidtok_b200: inputs must be CUDA tensors; there is no CPU path")
    if x.device != y.device:
        raise ValueError(f"the clips are on different devices: {x.device} and {y.device}")
    return B, Cc, T, H, W


def _workspace_bytes(B, Cc, T, H, W) -> int:
    need = N.lib().vt_frame_scores_workspace_bytes(B, Cc, T, H, W)
    if need < 0:
        raise ValueError(N.lib().vt_last_error().decode(errors="replace"))
    return need


def _launch(x, y, geom, ssim, running, workspace):
    B, Cc, T, H, W = geom
    x, y = x.detach().contiguous(), y.detach().contiguous()
    shape = (B, T) if x.dim() == 5 else (B,)
    with torch.cuda.device(x.device):
        ps = torch.empty(shape, dtype=torch.float32, device=x.device)
        ss = torch.empty(shape, dtype=torch.float32, device=x.device) if ssim else None
        N.check(N.lib().vt_frame_scores(
            C.c_void_p(x.data_ptr()), _DTYPES[x.dtype], C.c_void_p(y.data_ptr()), _DTYPES[y.dtype], B, Cc, T, H, W,
            C.c_void_p(ps.data_ptr()), C.c_void_p(ss.data_ptr()) if ssim else None,
            C.c_void_p(running.data_ptr()) if running is not None else None,
            C.c_void_p(workspace.data_ptr()), workspace.numel(), C.c_void_p(torch.cuda.current_stream(x.device).cuda_stream)))
    return ps, ss


def frame_scores(x: torch.Tensor, y: torch.Tensor, ssim: bool = True):
    """Per-frame PSNR and SSIM of the reconstruction y against the input x, both in [-1,1] before the clamp: clips
    [B,C,T,H,W] -> (psnr[B,T], ssim[B,T]), or frames [N,C,H,W] -> (psnr[N], ssim[N]); fp32 tensors on the clips' device, on
    the current stream, without synchronising.  ssim=False skips the SSIM part and returns (psnr, None).  x and y may each be
    float32, bfloat16 or float16 (the arithmetic is fp32 on the converted values)."""
    geom = _geometry(x, y, ssim)
    ws = torch.empty(max(1, _workspace_bytes(*geom)), dtype=torch.uint8, device=x.device)
    return _launch(x, y, geom, ssim, None, ws)


class Scorer:
    """Running PSNR / SSIM of a video or a dataset scored piece by piece, e.g. push by push of a DecodeStream:

        scorer = Scorer()
        for x, recon in pieces:
            scorer.update(x, recon)            # enqueues one kernel; no host synchronisation
        scorer.result()                        # {"psnr": ..., "ssim": ..., "frames": ...}: the one synchronisation

    The sums live in three doubles on the device, so result() equals the script's np.mean over its per-frame lists (see
    the module docstring for why no grouping by 16 is needed).  The workspace is kept and regrown only for a larger geometry."""

    def __init__(self):
        self._acc = None
        self._ws = None

    def update(self, x: torch.Tensor, y: torch.Tensor):
        """Scores one piece (as frame_scores) and adds its frames to the running sums; returns (psnr, ssim) per frame."""
        geom = _geometry(x, y, True)
        if self._acc is not None and self._acc.device != x.device:
            raise ValueError(f"this Scorer accumulates on {self._acc.device}, got clips on {x.device}")
        need = _workspace_bytes(*geom)
        if self._acc is None:
            self._acc = torch.zeros(3, dtype=torch.float64, device=x.device)
        if self._ws is None or self._ws.numel() < need:
            self._ws = torch.empty(max(1, need), dtype=torch.uint8, device=x.device)
        return _launch(x, y, geom, True, self._acc, self._ws)

    def sums(self) -> torch.Tensor:
        """A copy of the device accumulator, double [sum of PSNR, sum of SSIM, frames] (zeros before the first update)."""
        if self._acc is not None:
            return self._acc.clone()
        return torch.zeros(3, dtype=torch.float64, device="cuda" if torch.cuda.is_available() else "cpu")

    def result(self, reduce: bool = True) -> dict:
        """{"psnr": mean over frames, "ssim": mean over frames, "frames": n}; synchronises once.  With an initialised
        process group and reduce=True the sums are added over the ranks first, so every rank returns the global numbers.
        Before any frame was scored: frames 0 and NaN scores."""
        from .dist import global_scores
        acc = self.sums()
        if not reduce:
            return _means(acc)
        return global_scores(acc)

    def reset(self):
        if self._acc is not None:
            self._acc.zero_()


def _means(sums: torch.Tensor) -> dict:
    p, s, n = sums.tolist()
    n = int(round(n))
    if n == 0:
        return {"psnr": math.nan, "ssim": math.nan, "frames": 0}
    return {"psnr": p / n, "ssim": s / n, "frames": n}
