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

    With an I3D model (Scorer(i3d=I3D.from_files())) each update also adds the input clips' I3D features to the "real"
    statistics and the reconstructions' to the "generated" ones, and result() adds "fvd" and "fvd_clips".  fvd_frames=k cuts
    every clip of an update into consecutive windows of k frames (a shorter tail is dropped); otherwise a clip is one sample.

    The sums live in doubles on the device, so result() equals the script's np.mean over its per-frame lists (see the module
    docstring for why no grouping by 16 is needed).  The workspaces are kept and regrown only for a larger geometry."""

    def __init__(self, lpips: "LPIPS | None" = None, i3d: "I3D | None" = None, fvd_frames: int | None = None):
        self._acc = None
        self._ws = None
        self._lpips = lpips
        self._lacc = None     # [sum of LPIPS, frames]
        self._lws = None
        if fvd_frames is not None and (i3d is None or fvd_frames < I3D_MIN_FRAMES):
            raise ValueError(f"fvd_frames needs an I3D model and at least {I3D_MIN_FRAMES} frames, got {fvd_frames}")
        self._i3d = i3d
        self._fvd_frames = fvd_frames
        self._facc = None     # [2, n + sum f + sum f f^T]: the input clips' features, then the reconstructions'
        self._fws = None

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
        if self._i3d is not None:
            if self._facc is None:
                self._facc = torch.zeros(2, _STATS_LEN, dtype=torch.float64, device=x.device)
            for k, clips in enumerate((x, y)):
                clips = fvd_windows(clips, self._fvd_frames)
                fneed = self._i3d._workspace_bytes(_clip_geometry(clips))
                if self._fws is None or self._fws.numel() < fneed:
                    self._fws = torch.empty(fneed, dtype=torch.uint8, device=x.device)
                self._i3d._launch(clips, self._facc[k], self._fws)
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
        if self._i3d is not None:
            return self._result_fvd(acc, reduce)
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

    def _result_fvd(self, acc: torch.Tensor, reduce: bool) -> dict:
        """result() with FVD: the score sums, the LPIPS sums and both feature accumulators in one all-reduce."""
        from .dist import allreduce_sum
        lacc = self._lacc if self._lacc is not None else torch.zeros(2, dtype=torch.float64, device=acc.device)
        facc = self._facc if self._facc is not None else torch.zeros(2, _STATS_LEN, dtype=torch.float64, device=acc.device)
        both = torch.cat([acc, lacc.to(acc.device), facc.to(acc.device).flatten()])
        if reduce:
            both = allreduce_sum(both)
        out = _means(both[:3])
        if self._lpips is not None:
            s, n = both[3:5].tolist()
            out["lpips"] = s / n if n > 0 else math.nan
        f = both[5:].view(2, _STATS_LEN).cpu()
        n = int(round(float(f[0, 0])))
        out["fvd"] = fvd_from_stats(f[0], f[1]) if n >= 2 else math.nan
        out["fvd_clips"] = n
        return out

    def fvd_sums(self) -> torch.Tensor:
        """A copy of the feature accumulators, float64 [2, n + sum f + sum f f^T] (input clips, reconstructions)."""
        if self._facc is not None:
            return self._facc.clone()
        return torch.zeros(2, _STATS_LEN, dtype=torch.float64)

    def reset(self):
        if self._acc is not None:
            self._acc.zero_()
        if self._lacc is not None:
            self._lacc.zero_()
        if self._facc is not None:
            self._facc.zero_()


def _means(sums: torch.Tensor) -> dict:
    p, s, n = sums.tolist()
    n = int(round(n))
    if n == 0:
        return {"psnr": math.nan, "ssim": math.nan, "frames": 0}
    return {"psnr": p / n, "ssim": s / n, "frames": n}


# ---- LPIPS (vidtok/modules/lpips.py; scripts/inference_evaluate.py:175-186) ------------------------------------------------
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


# The precisions of the evaluation networks (LPIPS, I3D)
_EVAL_PRECISIONS = {"exact": N.PREC_EXACT_TC, "bf16": N.PREC_BF16}


class _EvalNet:
    """The library's weight handle of an evaluation network (the C functions vt_<_net>_*): created on the model's device with
    every parameter of _state(state) loaded and finalized, released by close().  _host_load: the parameters are loaded from
    host tensors rather than from copies on the device."""
    _net: str                # "lpips" or "i3d"
    _state: staticmethod     # the state-dict check of the network (lpips_state, i3d_state)
    _host_load = False

    def __init__(self, state: dict, device=None, precision: str = "exact"):
        if precision not in _EVAL_PRECISIONS:
            raise ValueError(f"precision must be one of {sorted(_EVAL_PRECISIONS)}, got {precision!r}")
        self.precision = precision
        self.device = torch.device(device) if device is not None else torch.device("cuda")
        if self.device.index is None:
            self.device = torch.device(self.device.type, torch.cuda.current_device())
        state = self._state(state)
        h = C.c_void_p()
        N.check(self._fn("create")(self.device.index, C.byref(h)))
        self._h = h
        with torch.cuda.device(self.device):
            stream = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
            keep = []
            for key, v in state.items():
                t = v.detach().to("cpu" if self._host_load else self.device, torch.float32).contiguous()
                keep.append(t)
                N.check(self._fn("load_param")(h, key.encode(), C.c_void_p(t.data_ptr()), t.numel(), int(not self._host_load), stream))
            N.check(self._fn("finalize")(h, stream))
            del keep

    def _fn(self, name: str):
        return getattr(N.lib(), f"vt_{self._net}_{name}")

    @classmethod
    def from_state_dict(cls, sd: dict, device=None, precision: str = "exact"):
        return cls(sd, device, precision)

    def close(self):
        if getattr(self, "_h", None):
            self._fn("destroy")(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _workspace_bytes(self, geom) -> int:
        need = self._fn("workspace_bytes")(self._h, _EVAL_PRECISIONS[self.precision], *geom)
        if need < 0:
            raise ValueError(N.lib().vt_last_error().decode(errors="replace"))
        return need


class LPIPS(_EvalNet):
    """LPIPS with VGG16 on the device (vidtok/modules/lpips.py as scripts/inference_evaluate.py calls it): owns the library's
    weight handle.  precision "exact" (the default: fp32-class results through the split-fp16 tensor-core operands, as the
    script's fp32 run) or "bf16".  Build it with from_state_dict or from_files; score with lpips_scores or Scorer(lpips=...)."""
    _net = "lpips"
    _state = staticmethod(lpips_state)

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
                self._h, _EVAL_PRECISIONS[self.precision], C.c_void_p(x.data_ptr()), _DTYPES[x.dtype], C.c_void_p(y.data_ptr()),
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


# ---- FVD: I3D features and the Frechet distance -------------------------------------------------------------------------------
# The definition (the common one, VideoGPT's fvd module with TF-GAN's Frechet distance; the reference reports FVD but ships no
# code for it): clamp to [-1,1], (v+1)/2, bilinear resize (align_corners=False, no antialias) to short side 224 and long side
# ceil(long * 224 / short), centre crop 224 x 224, (v-0.5)*2; I3D (Inception-v1 inflated, Kinetics-400); the 400 logits averaged
# over time; FVD = |mu1-mu2|^2 + tr S1 + tr S2 - 2 tr((S1^1/2 S2 S1^1/2)^1/2) with unbiased covariances, in float64.
I3D_DEFAULT_PATH = os.path.join("checkpoints", "i3d", "i3d_pretrained_400.pt")
I3D_FEATURES = 400
I3D_MIN_FRAMES = 9
_I3D_MODULES = (("Mixed_3b", (64, 96, 128, 16, 32, 32)), ("Mixed_3c", (128, 128, 192, 32, 96, 64)),
                ("Mixed_4b", (192, 96, 208, 16, 48, 64)), ("Mixed_4c", (160, 112, 224, 24, 64, 64)),
                ("Mixed_4d", (128, 128, 256, 24, 64, 64)), ("Mixed_4e", (112, 144, 288, 32, 64, 64)),
                ("Mixed_4f", (256, 160, 320, 32, 128, 128)), ("Mixed_5b", (256, 160, 320, 32, 128, 128)),
                ("Mixed_5c", (384, 192, 384, 48, 128, 128)))
I3D_ENDPOINTS = ("Conv3d_1a_7x7", "MaxPool3d_2a_3x3", "Conv3d_2b_1x1", "Conv3d_2c_3x3", "MaxPool3d_3a_3x3", "Mixed_3b", "Mixed_3c",
                 "MaxPool3d_4a_3x3", "Mixed_4b", "Mixed_4c", "Mixed_4d", "Mixed_4e", "Mixed_4f", "MaxPool3d_5a_2x2", "Mixed_5b",
                 "Mixed_5c")
_STATS_LEN = 1 + I3D_FEATURES + I3D_FEATURES * I3D_FEATURES


def i3d_units():
    """[(unit key, Cin, Cout, k)] of every conv + BatchNorm + ReLU unit of I3D, in network order."""
    units = [("Conv3d_1a_7x7", 3, 64, 7), ("Conv3d_2b_1x1", 64, 64, 1), ("Conv3d_2c_3x3", 64, 192, 3)]
    cin = 192
    for name, o in _I3D_MODULES:
        units += [(f"{name}.b0", cin, o[0], 1), (f"{name}.b1a", cin, o[1], 1), (f"{name}.b1b", o[1], o[2], 3),
                  (f"{name}.b2a", cin, o[3], 1), (f"{name}.b2b", o[3], o[4], 3), (f"{name}.b3b", cin, o[5], 1)]
        cin = o[0] + o[2] + o[4] + o[5]
    return units


def i3d_state_shapes() -> dict:
    """The PyTorch port's (InceptionI3d, i3d_pretrained_400.pt) parameter keys and shapes."""
    shapes = {}
    for key, ci, co, k in i3d_units():
        shapes[f"{key}.conv3d.weight"] = (co, ci, k, k, k)
        for b in ("weight", "bias", "running_mean", "running_var"):
            shapes[f"{key}.bn.{b}"] = (co,)
    shapes["logits.conv3d.weight"] = (I3D_FEATURES, 1024, 1, 1, 1)
    shapes["logits.conv3d.bias"] = (I3D_FEATURES,)
    return shapes


def i3d_state(sd: dict) -> dict:
    """The I3D parameters of a state dict in the port's layout.  Raises KeyError naming a missing key and ValueError naming a
    misshaped one; other keys (num_batches_tracked) are ignored."""
    out = {}
    missing = [k for k in i3d_state_shapes() if k not in sd]
    if missing:
        raise KeyError("I3D state dict lacks " + ", ".join(missing))
    for key, shape in i3d_state_shapes().items():
        v = torch.as_tensor(sd[key])
        if tuple(v.shape) != shape:
            raise ValueError(f"I3D parameter {key}: shape {tuple(v.shape)}, expected {shape}")
        out[key] = v
    return out


def _clip_geometry(x: torch.Tensor):
    if x.dim() != 5:
        raise ValueError(f"expected clips [B,3,T,H,W], got {tuple(x.shape)}")
    if x.dtype not in _DTYPES:
        raise ValueError(f"expected a float32, bfloat16 or float16 tensor, got {x.dtype}")
    if x.numel() == 0:
        raise ValueError(f"empty clip {tuple(x.shape)}")
    if not x.is_cuda:
        raise RuntimeError("vidtok_b200: inputs must be CUDA tensors; there is no CPU path")
    return tuple(int(d) for d in x.shape)


class I3D(_EvalNet):
    """The FVD feature network on the device: owns the library's I3D weight handle.  precision "exact" (the default:
    fp32-class results through the split-fp16 tensor-core operands) or "bf16".  Build it with from_state_dict or from_files;
    use it with i3d_features or Scorer(i3d=...)."""
    _net = "i3d"
    _state = staticmethod(i3d_state)
    _host_load = True   # finalize folds BatchNorm into the weights on the host

    @classmethod
    def from_files(cls, path: str | None = None, device=None, precision: str = "exact") -> "I3D":
        """The port's Kinetics-400 weights (default: checkpoints/i3d/i3d_pretrained_400.pt).  Nothing is downloaded: a missing
        file raises FileNotFoundError naming the path."""
        path = path or I3D_DEFAULT_PATH
        if not os.path.isfile(path):
            raise FileNotFoundError(f"I3D weights not found: {path}")
        return cls(torch.load(path, map_location="cpu", weights_only=True), device, precision)

    def pass_clips(self, T: int, H: int, W: int) -> int:
        """Clips per pass of the executor: 8, or fewer where an activation of the pass would exceed 2^31 elements."""
        return int(N.lib().vt_i3d_pass_clips(self._h, T, H, W))

    def _launch(self, x, stats, workspace):
        geom = _clip_geometry(x)
        if x.device != self.device:
            raise ValueError(f"this I3D model lives on {self.device}, got clips on {x.device}")
        x = x.detach().contiguous()
        with torch.cuda.device(x.device):
            feats = torch.empty((geom[0], I3D_FEATURES), dtype=torch.float32, device=x.device)
            N.check(N.lib().vt_i3d_features(
                self._h, _EVAL_PRECISIONS[self.precision], C.c_void_p(x.data_ptr()), _DTYPES[x.dtype], *geom,
                C.c_void_p(feats.data_ptr()), C.c_void_p(stats.data_ptr()) if stats is not None else None,
                C.c_void_p(workspace.data_ptr()), workspace.numel(), C.c_void_p(torch.cuda.current_stream(x.device).cuda_stream)))
        return feats

    def endpoint(self, x: torch.Tensor, name: str, workspace: torch.Tensor | None = None) -> torch.Tensor:
        """The activation at end point `name` (I3D_ENDPOINTS) as fp32 [B,C,T,H,W], for the tests: one pass of clips at most."""
        geom = _clip_geometry(x)
        prec = _EVAL_PRECISIONS[self.precision]
        shape = (C.c_int64 * 5)()
        N.check(N.lib().vt_i3d_endpoint(self._h, prec, None, _DTYPES[x.dtype], *geom, name.encode(), None, shape, None, 0, None))
        x = x.detach().contiguous()
        if workspace is None:
            workspace = torch.empty(self._workspace_bytes(geom), dtype=torch.uint8, device=x.device)
        with torch.cuda.device(x.device):
            out = torch.empty(tuple(shape), dtype=torch.float32, device=x.device)
            N.check(N.lib().vt_i3d_endpoint(self._h, prec, C.c_void_p(x.data_ptr()), _DTYPES[x.dtype], *geom, name.encode(),
                                            C.c_void_p(out.data_ptr()), None, C.c_void_p(workspace.data_ptr()), workspace.numel(),
                                            C.c_void_p(torch.cuda.current_stream(x.device).cuda_stream)))
        return out


def i3d_features(model: I3D, clips: torch.Tensor, stats: torch.Tensor | None = None) -> torch.Tensor:
    """fp32 [B,400] I3D features of clips [B,3,T,H,W] in [-1,1] (float32, bfloat16 or float16, T >= 9), on the current stream,
    without synchronising.  stats (optional): a float64 device tensor of i3d_stats_empty()'s shape that receives += this
    call's clips, in clip order."""
    ws = torch.empty(model._workspace_bytes(_clip_geometry(clips)), dtype=torch.uint8, device=clips.device)
    return model._launch(clips, stats, ws)


def i3d_stats_empty(device=None) -> torch.Tensor:
    """A zero accumulator [n, sum f (400), sum f f^T (400 x 400)] in float64."""
    return torch.zeros(_STATS_LEN, dtype=torch.float64, device=device)


def features_to_stats(features: torch.Tensor) -> torch.Tensor:
    """The accumulator of a feature set [n,400], in float64 (host or device)."""
    f = features.to(torch.float64)
    return torch.cat([torch.tensor([f.shape[0]], dtype=torch.float64, device=f.device), f.sum(0), (f.T @ f).flatten()])


def _psd_eigvals(a: torch.Tensor, rank: int):
    """eigh of a symmetric PSD matrix of rank <= rank: eigenvalues clamped at 0, all but the rank largest set to 0 (the
    covariance of n samples has rank n - 1 at most; the square roots of its zero eigenvalues' rounding noise would otherwise
    add ~1e-8 of the distance per sample set below 400 clips)"""
    w, v = torch.linalg.eigh((a + a.T) / 2)
    w = w.clamp(min=0)
    if rank < w.numel():
        w[: w.numel() - rank] = 0
    return w, v


def fvd_from_stats(stats_a: torch.Tensor, stats_b: torch.Tensor) -> float:
    """FVD between the feature sets of two accumulators (each at least two clips), in float64 on the host."""
    out = []
    for s in (stats_a, stats_b):
        s = s.detach().to("cpu", torch.float64)
        n = float(s[0])
        if n < 2:
            raise ValueError(f"FVD needs at least 2 clips per set, got {n:g}")
        mu = s[1:1 + I3D_FEATURES] / n
        cov = (s[1 + I3D_FEATURES:].view(I3D_FEATURES, I3D_FEATURES) - n * torch.outer(mu, mu)) / (n - 1)
        out.append((mu, cov, int(round(n)) - 1))
    (mu1, s1, r1), (mu2, s2, r2) = out
    w, v = _psd_eigvals(s1, r1)
    root = (v * w.sqrt()) @ v.T
    tr = _psd_eigvals(root @ s2 @ root, min(r1, r2))[0].sqrt().sum()
    return float(((mu1 - mu2) ** 2).sum() + torch.trace(s1) + torch.trace(s2) - 2 * tr)


def fvd(features_a: torch.Tensor, features_b: torch.Tensor) -> float:
    """FVD between two feature sets [n,400] (as i3d_features returns them)."""
    return fvd_from_stats(features_to_stats(features_a), features_to_stats(features_b))


def fvd_windows(x: torch.Tensor, k: int | None) -> torch.Tensor:
    """Clips [B,C,T,H,W] cut into consecutive windows of k frames ([B * (T // k), C, k, H, W], a shorter tail dropped), or x
    itself for k None."""
    if k is None:
        return x
    B, Cc, T, H, W = x.shape
    nw = T // k
    if nw == 0:
        raise ValueError(f"clips of {T} frames hold no window of {k} frames")
    return x[:, :, :nw * k].reshape(B, Cc, nw, k, H, W).transpose(1, 2).reshape(B * nw, Cc, k, H, W)
