"""The evaluation protocol's quality numbers on the device (scripts/inference_evaluate.py:175-186): clamp to [-1,1], (v+1)/2,
then compute_psnr / compute_ssim (vidtok/modules/util.py:146-231), as one fused kernel of libvidtok_b200.so that reads the
input clip and the reconstruction once and returns the two scores of every frame.  Nothing here synchronises with the host
until a result is asked for.

The script clamps only the reconstruction; the kernel clamps both clips, which is the identity on an input in [-1,1].

The script scores groups of 16 frames and appends each group's value once per frame of the group; a group's value is the
mean of its frames' values, so the mean of that list is the mean over frames of the per-frame values, whatever the
grouping (tests/test_metrics_cpu.py::test_grouping_identity).  Scorer therefore keeps [sum of PSNR, sum of SSIM, frames], and
with an LPIPS model [sum of LPIPS, frames] next to it.

LPIPS (vidtok/modules/lpips.py, the script's third number) runs VGG16 and the LPIPS head in the library: LPIPS owns the
weights, lpips_scores returns per-frame values."""
from __future__ import annotations

import ctypes as C
import math
import os

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
    """Running PSNR / SSIM (and, given an LPIPS model, LPIPS) of a video or a dataset scored piece by piece, e.g. push by push
    of a DecodeStream:

        scorer = Scorer(lpips=LPIPS.from_files())   # or Scorer() for PSNR / SSIM only
        for x, recon in pieces:
            scorer.update(x, recon)            # enqueues the kernels; no host synchronisation
        scorer.result()                        # {"psnr", "ssim", "frames"[, "lpips"]}: the one synchronisation

    The sums live in doubles on the device, so result() equals the script's np.mean over its per-frame lists (see the module
    docstring for why no grouping by 16 is needed).  The workspaces are kept and regrown only for a larger geometry."""

    def __init__(self, lpips: "LPIPS | None" = None):
        self._acc = None
        self._ws = None
        self._lpips = lpips
        self._lacc = None     # [sum of LPIPS, frames]
        self._lws = None

    def update(self, x: torch.Tensor, y: torch.Tensor):
        """Scores one piece (as frame_scores, and lpips_scores when the Scorer has an LPIPS model) and adds its frames to the
        running sums; returns (psnr, ssim) per frame."""
        geom = _geometry(x, y, True)
        if self._acc is not None and self._acc.device != x.device:
            raise ValueError(f"this Scorer accumulates on {self._acc.device}, got clips on {x.device}")
        need = _workspace_bytes(*geom)
        lneed = self._lpips._workspace_bytes(geom) if self._lpips is not None else 0
        if self._acc is None:
            self._acc = torch.zeros(3, dtype=torch.float64, device=x.device)
        if self._ws is None or self._ws.numel() < need:
            self._ws = torch.empty(max(1, need), dtype=torch.uint8, device=x.device)
        out = _launch(x, y, geom, True, self._acc, self._ws)
        if self._lpips is not None:
            if self._lacc is None:
                self._lacc = torch.zeros(2, dtype=torch.float64, device=x.device)
            if self._lws is None or self._lws.numel() < lneed:
                self._lws = torch.empty(lneed, dtype=torch.uint8, device=x.device)
            self._lpips._launch(x, y, geom, self._lacc, self._lws)
        return out

    def sums(self) -> torch.Tensor:
        """A copy of the device accumulator, double [sum of PSNR, sum of SSIM, frames] (zeros before the first update)."""
        if self._acc is not None:
            return self._acc.clone()
        return torch.zeros(3, dtype=torch.float64, device="cuda" if torch.cuda.is_available() else "cpu")

    def result(self, reduce: bool = True) -> dict:
        """{"psnr": mean over frames, "ssim": mean over frames, "frames": n}; synchronises once.  With an initialised
        process group and reduce=True the sums are added over the ranks first, so every rank returns the global numbers.
        Before any frame was scored: frames 0 and NaN scores."""
        from .dist import allreduce_sum, global_scores
        acc = self.sums()
        if self._lpips is None:
            if not reduce:
                return _means(acc)
            return global_scores(acc)
        lacc = self._lacc.clone() if self._lacc is not None else torch.zeros(2, dtype=torch.float64, device=acc.device)
        both = torch.cat([acc, lacc.to(acc.device)])
        if reduce:
            both = allreduce_sum(both)          # one all-reduce of the five sums
        out = _means(both[:3])
        s, n = both[3:].tolist()
        out["lpips"] = s / n if n > 0 else math.nan
        return out

    def reset(self):
        if self._acc is not None:
            self._acc.zero_()
        if self._lacc is not None:
            self._lacc.zero_()


def _means(sums: torch.Tensor) -> dict:
    p, s, n = sums.tolist()
    n = int(round(n))
    if n == 0:
        return {"psnr": math.nan, "ssim": math.nan, "frames": 0}
    return {"psnr": p / n, "ssim": s / n, "frames": n}


# ---- LPIPS (vidtok/modules/lpips.py; scripts/inference_evaluate.py:175-186) ------------------------------------------------
_LPIPS_PRECISIONS = {"exact": N.PREC_EXACT_TC, "bf16": N.PREC_BF16}
_LPIPS_CONVS = ((1, 0), (1, 2), (2, 5), (2, 7), (3, 10), (3, 12), (3, 14), (4, 17), (4, 19), (4, 21), (5, 24), (5, 26), (5, 28))
_LPIPS_COUT = (64, 64, 128, 128, 256, 256, 256, 512, 512, 512, 512, 512, 512)
_LPIPS_CHNS = (64, 128, 256, 512, 512)
_LPIPS_SHIFT = (-0.030, -0.088, -0.188)
_LPIPS_SCALE = (0.458, 0.448, 0.450)
LPIPS_DEFAULT_PATH = os.path.join("checkpoints", "lpips", "vgg.pth")


def torchvision_vgg16_path() -> str:
    """Where torchvision caches its VGG16 checkpoint: $TORCH_HOME/hub/checkpoints/vgg16-397923af.pth."""
    return os.path.join(torch.hub.get_dir(), "checkpoints", "vgg16-397923af.pth")


def lpips_state_shapes() -> dict:
    """The reference's LPIPS parameter keys and shapes (the ScalingLayer's constant buffers aside)."""
    shapes, ci = {}, 3
    for (s, i), co in zip(_LPIPS_CONVS, _LPIPS_COUT):
        shapes[f"net.slice{s}.{i}.weight"] = (co, ci, 3, 3)
        shapes[f"net.slice{s}.{i}.bias"] = (co,)
        ci = co
    for k, c in enumerate(_LPIPS_CHNS):
        shapes[f"lin{k}.model.1.weight"] = (1, c, 1, 1)
    return shapes


def lpips_state(sd: dict) -> dict:
    """The parameters of an LPIPS state dict under the reference's keys, from the reference's own keys (LPIPS().state_dict())
    or from torchvision's VGG16 keys `features.{i}.*` plus `lin{k}.model.1.weight`.  Raises on a missing or misshaped key, and
    on ScalingLayer buffers that differ from the reference's constants.  Other keys (VGG16's classifier) are ignored."""
    out, missing = {}, []
    for key, shape in lpips_state_shapes().items():
        alt = None
        if key.startswith("net."):
            alt = "features." + key.split(".", 2)[2]
        v = sd.get(key, sd.get(alt) if alt else None)
        if v is None:
            missing.append(key if alt is None else f"{key} (or {alt})")
            continue
        v = torch.as_tensor(v)
        if tuple(v.shape) != shape:
            raise ValueError(f"LPIPS parameter {key}: shape {tuple(v.shape)}, expected {shape}")
        out[key] = v
    if missing:
        raise KeyError("LPIPS state dict lacks " + ", ".join(missing))
    for name, want in (("shift", _LPIPS_SHIFT), ("scale", _LPIPS_SCALE)):
        v = sd.get(f"scaling_layer.{name}")
        if v is not None and not torch.equal(torch.as_tensor(v).float().flatten().cpu(), torch.tensor(want, dtype=torch.float32)):
            raise ValueError(f"scaling_layer.{name} = {torch.as_tensor(v).flatten().tolist()} differs from the reference's {list(want)}")
    return out


def lpips_pass_frames(H: int, W: int) -> int:
    """Frame pairs per pass of the LPIPS executor at H x W: 16, or fewer where relu1_2 of a pass would exceed 2^31 elements."""
    return int(N.lib().vt_lpips_pass_frames(H, W))


class LPIPS:
    """LPIPS with VGG16 on the device (vidtok/modules/lpips.py as scripts/inference_evaluate.py calls it): owns the library's
    weight handle.  precision "exact" (the default: fp32-class results through the split-fp16 tensor-core operands, as the
    script's fp32 run) or "bf16".  Build it with from_state_dict or from_files; score with lpips_scores or Scorer(lpips=...)."""

    def __init__(self, state: dict, device=None, precision: str = "exact"):
        if precision not in _LPIPS_PRECISIONS:
            raise ValueError(f"precision must be one of {sorted(_LPIPS_PRECISIONS)}, got {precision!r}")
        self.precision = precision
        self.device = torch.device(device) if device is not None else torch.device("cuda")
        if self.device.index is None:
            self.device = torch.device(self.device.type, torch.cuda.current_device())
        state = lpips_state(state)
        h = C.c_void_p()
        N.check(N.lib().vt_lpips_create(self.device.index, C.byref(h)))
        self._h = h
        with torch.cuda.device(self.device):
            stream = torch.cuda.current_stream(self.device)
            keep = []
            for key, v in state.items():
                t = v.detach().to(self.device, torch.float32).contiguous()
                keep.append(t)
                N.check(N.lib().vt_lpips_load_param(h, key.encode(), C.c_void_p(t.data_ptr()), t.numel(), 1, C.c_void_p(stream.cuda_stream)))
            N.check(N.lib().vt_lpips_finalize(h, C.c_void_p(stream.cuda_stream)))
            del keep

    @classmethod
    def from_state_dict(cls, sd: dict, device=None, precision: str = "exact") -> "LPIPS":
        return cls(sd, device, precision)

    @classmethod
    def from_files(cls, vgg16_path: str | None = None, lpips_path: str | None = None, device=None, precision: str = "exact") -> "LPIPS":
        """VGG16 from torchvision's checkpoint (default: its cache file, torchvision_vgg16_path()) and the lin weights from
        LPIPS's vgg.pth (default: checkpoints/lpips/vgg.pth, where the reference keeps it).  Nothing is downloaded: a missing
        file raises FileNotFoundError naming the path."""
        vgg16_path = vgg16_path or torchvision_vgg16_path()
        lpips_path = lpips_path or LPIPS_DEFAULT_PATH
        sd = {}
        for path in (vgg16_path, lpips_path):
            if not os.path.isfile(path):
                raise FileNotFoundError(f"LPIPS weights not found: {path}")
            sd.update(torch.load(path, map_location="cpu", weights_only=True))
        return cls(sd, device, precision)

    def close(self):
        if getattr(self, "_h", None):
            N.lib().vt_lpips_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _workspace_bytes(self, geom) -> int:
        need = N.lib().vt_lpips_workspace_bytes(self._h, _LPIPS_PRECISIONS[self.precision], *geom)
        if need < 0:
            raise ValueError(N.lib().vt_last_error().decode(errors="replace"))
        return need

    def _launch(self, x, y, geom, running, workspace, per_layer=False):
        B, Cc, T, H, W = geom
        if x.device != self.device:
            raise ValueError(f"this LPIPS model lives on {self.device}, got clips on {x.device}")
        x, y = x.detach().contiguous(), y.detach().contiguous()
        shape = (B, T) if x.dim() == 5 else (B,)
        with torch.cuda.device(x.device):
            out = torch.empty(shape, dtype=torch.float32, device=x.device)
            layers = torch.empty(shape + (5,), dtype=torch.float32, device=x.device) if per_layer else None
            N.check(N.lib().vt_lpips(
                self._h, _LPIPS_PRECISIONS[self.precision], C.c_void_p(x.data_ptr()), _DTYPES[x.dtype], C.c_void_p(y.data_ptr()),
                _DTYPES[y.dtype], B, Cc, T, H, W, C.c_void_p(out.data_ptr()), C.c_void_p(layers.data_ptr()) if per_layer else None,
                C.c_void_p(running.data_ptr()) if running is not None else None, C.c_void_p(workspace.data_ptr()), workspace.numel(),
                C.c_void_p(torch.cuda.current_stream(x.device).cuda_stream)))
        return (out, layers) if per_layer else out


def lpips_scores(model: LPIPS, x: torch.Tensor, y: torch.Tensor, per_layer: bool = False):
    """Per-frame LPIPS of the reconstruction y against the input x, both in [-1,1] with y not yet clamped: clips [B,3,T,H,W] ->
    fp32 [B,T], or frames [N,3,H,W] -> [N]; with per_layer=True also the five layer terms [..., 5].  On the current stream,
    without synchronising.  x and y may each be float32, bfloat16 or float16."""
    geom = _geometry(x, y, False)
    ws = torch.empty(model._workspace_bytes(geom), dtype=torch.uint8, device=x.device)
    return model._launch(x, y, geom, None, ws, per_layer)
