"""Device-side versions of the conversions the reference's scripts do around the tokenizer
(scripts/inference_reconstruct.py:41-47,71-75: frames.float()/255 -> CenterCrop -> Normalize(.5,.5) -> [C,T,H,W];
:78-82,231-239: tensor_to_uint8 + `t c h w -> t h w c`), and the whole clip transform with the antialiased Resize
(transform_frames).  All run in libvidtok_b200.so; results are bit-identical to the torch / numpy statements
(tests/test_gpu_ops_tc.py::test_video_io_*, tests/test_gpu_video_ingest.py)."""
from __future__ import annotations

import ctypes as C

import torch

from . import _native as N


def _check_cuda(t: torch.Tensor):
    if not t.is_cuda:
        raise RuntimeError("vidtok_b200: inputs must be CUDA tensors; there is no CPU path")


def frames_to_clip(frames: torch.Tensor, height: int, width: int) -> torch.Tensor:
    """uint8 [T,Hs,Ws,C] decoded frames -> fp32 [1,C,T,height,width] clip in [-1,1] (centre crop, as
    torchvision.transforms.CenterCrop rounds it)."""
    _check_cuda(frames)
    if frames.dtype != torch.uint8 or frames.dim() != 4:
        raise ValueError("expected uint8 frames [T,H,W,C]")
    frames = frames.contiguous()
    T, Hs, Ws, Cc = frames.shape
    if height > Hs or width > Ws:
        raise ValueError("crop larger than the frame (the reference would pad; resize first)")
    h0, w0 = int(round((Hs - height) / 2.0)), int(round((Ws - width) / 2.0))
    out = torch.empty((1, Cc, T, height, width), dtype=torch.float32, device=frames.device)
    N.check(N.lib().vt_video_u8_to_clip(C.c_void_p(frames.data_ptr()), C.c_void_p(out.data_ptr()), T, Hs, Ws, Cc, h0, w0, height, width,
                                        C.c_void_p(torch.cuda.current_stream(frames.device).cuda_stream)))
    return out


def resize_crop_geometry(Hs: int, Ws: int, height: int, width: int) -> tuple:
    """(Hr, Wr, h0, w0) of torchvision's Resize(height) + CenterCrop((height, width)) on an Hs x Ws frame: the short side
    becomes `height` and the long side int(height * long / short); the crop starts at round((resized - crop) / 2)."""
    Hr, Wr = (int(height * Hs / Ws), height) if Ws <= Hs else (height, int(height * Ws / Hs))
    if height > Hr or width > Wr:
        raise ValueError("crop larger than the resized frame (the reference would pad)")
    return Hr, Wr, int(round((Hr - height) / 2.0)), int(round((Wr - width) / 2.0))


def transform_frames(frames: torch.Tensor, input_height: int, input_width: int, clip_frames: int | None = None) -> torch.Tensor:
    """uint8 [N,Hs,Ws,C] decoded frames -> fp32 [N/clip_frames,C,clip_frames,input_height,input_width] clips in [-1,1]: the
    reference's per-clip transform (vidtok/data/vidtok.py:51-56,181-185; scripts/inference_reconstruct.py:41-47,73-74)
        Resize(input_height, antialias=True) -> CenterCrop((input_height, input_width)) -> Normalize(.5, .5)
    applied to frames.float() / 255, in one kernel.  Frame n goes to clip n // clip_frames (all N frames form one clip
    when clip_frames is None)."""
    _check_cuda(frames)
    if frames.dtype != torch.uint8 or frames.dim() != 4:
        raise ValueError("expected uint8 frames [N,H,W,C]")
    frames = frames.contiguous()
    n, Hs, Ws, Cc = frames.shape
    tc = n if clip_frames is None else clip_frames
    if tc <= 0 or n % tc != 0:
        raise ValueError(f"{n} frames do not split into clips of {tc}")
    Hr, Wr, h0, w0 = resize_crop_geometry(Hs, Ws, input_height, input_width)
    out = torch.empty((n // tc, Cc, tc, input_height, input_width), dtype=torch.float32, device=frames.device)
    N.check(N.lib().vt_video_u8_to_clip_resized(C.c_void_p(frames.data_ptr()), C.c_void_p(out.data_ptr()), n, Hs, Ws, Cc, Hr, Wr,
                                                h0, w0, input_height, input_width, tc,
                                                C.c_void_p(torch.cuda.current_stream(frames.device).cuda_stream)))
    return out


def clip_to_frames_u8(clip: torch.Tensor) -> torch.Tensor:
    """fp32 [C,T,H,W] (or [1,C,T,H,W]) reconstruction -> uint8 frames [T,H,W,C]."""
    _check_cuda(clip)
    if clip.dim() == 5:
        if clip.shape[0] != 1:
            raise ValueError("one clip at a time")
        clip = clip[0]
    clip = clip.detach().float().contiguous()
    Cc, T, H, W = clip.shape
    out = torch.empty((T, H, W, Cc), dtype=torch.uint8, device=clip.device)
    N.check(N.lib().vt_clip_to_video_u8(C.c_void_p(clip.data_ptr()), C.c_void_p(out.data_ptr()), Cc, T, H, W,
                                        C.c_void_p(torch.cuda.current_stream(clip.device).cuda_stream)))
    return out
