"""Streaming encode / decode of causal tokenizers: a video is pushed a few frames at a time and the memory in use does not
grow with its length.

    enc = EncodeStream(model, batch=B, H=H, W=W)
    for frames in source:                  # [B, C, t, H, W], any t
        z, reg_log = enc.push(frames)      # the latent frames this push completed (possibly none)
    dec = DecodeStream(model, batch=B, Hz=Hz, Wz=Wz)
    x = dec.push(z)                        # decoded frames of these latents

Both streams run on the library's chunk states (vt_encode_chunk / vt_decode_chunk): per-layer caches carry the frames each
causal convolution, time resampling and the fused temporal block need from the previous chunk.

* v1.0 causal models: every norm and attention works within one frame, so a stream computes exactly the whole-clip
  function: in "bf16" and "fma" the concatenated outputs equal `model.encode(whole)` / `model.decode(whole)` bit for bit.
  The split-operand "exact" mode (and "mixed"'s encoder) agrees to fp32 rounding: its tensor-core kernels group the K
  steps of a tile by the taps the tile does not skip, and the tile's depth in frames depends on the clip's length at small
  spatial sizes, so the whole clip's own first frames round differently for different lengths.  The encoder runs the
  first frame together with every complete group of `time_downsample_factor` (tdf) frames that follows it, then complete
  groups; frames that do not yet complete a group wait for the next push.  The first decoded chunk drops tdf-1 frames, as
  the whole clip does.
* v1.1 models: the first frame is a chunk of its own, then complete tdf groups, without overlap look-ahead.  The outputs
  equal `tile_encode` / `tile_decode` with `use_overlap=False` at the same chunking.
* Non-causal models cannot stream (their time padding is symmetric) and are rejected at creation.

Precision is fixed at creation from `model.precision` / the autocast state, as `encode` reads it.  `reg_log` is per push:
`indices` (FSQ) or `kl_loss` (KL, the push's share: the per-push values sum to the whole clip's).  The FSQ `aux_loss`, a
statistic over the whole clip's tokens, is not computed in streams.  KL noise is one CPU `torch.randn` per push over the
push's latent frames unless `noise` is passed.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Tuple

import torch

from . import _native as N
from .engine import ChunkState, _ptr, _stream_ptr


def encode_chunks(avail: int, first: bool, tdf: int, version: int) -> List[int]:
    """Frame counts of the encoder chunks that `avail` buffered frames complete: the first chunk is the first frame plus
    every complete group of tdf frames after it (v1.1: the first frame alone), later chunks all complete groups."""
    out = []
    while avail > 0:
        if first:
            n = 1 if version == 1 else 1 + tdf * ((avail - 1) // tdf)
        else:
            n = tdf * (avail // tdf)
        if n == 0:
            break
        out.append(n)
        avail -= n
        first = False
    return out


class _Stream:
    def __init__(self, model, batch: int, H: int, W: int, is_decoder: bool):
        if not model.is_causal:
            raise ValueError("non-causal models cannot stream: their time padding is symmetric, so a frame depends on later frames")
        rt = model._rt
        self.model = model
        self.native = rt.sync()
        self.spec = model.spec
        self.precision = rt.precision()
        self.out_dtype = rt.out_dtype()
        self.tdf = int(self.spec.time_downsample_factor)
        self.B, self.H, self.W = int(batch), int(H), int(W)
        self.state = ChunkState(self.native, self.precision, self.B, self.H, self.W, is_decoder, False)
        self.first = True

    def reset(self):
        """Start a new video: the next push is its first chunk (the caches are rewritten, not read)."""
        self.first = True

    def close(self):
        self.state.close()

    def _workspace(self, n: int) -> torch.Tensor:
        return self.state.workspace(n)


class EncodeStream(_Stream):
    def __init__(self, model, batch: int, H: int, W: int):
        super().__init__(model, batch, H, W, is_decoder=False)
        self.pending: Optional[torch.Tensor] = None
        self.Hz, self.Wz = self.native.latent_shape(1, H, W)[1:]

    def reset(self):
        super().reset()
        self.pending = None

    def push(self, x: torch.Tensor, noise: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, Dict[str, torch.Tensor]]:
        if not x.is_cuda:
            raise RuntimeError("vidtok_b200: inputs must be CUDA tensors; there is no CPU path")
        if x.dim() != 5 or tuple(x.shape[:2]) != (self.B, self.spec.in_channels) or tuple(x.shape[3:]) != (self.H, self.W):
            raise ValueError(f"expected [{self.B},{self.spec.in_channels},t,{self.H},{self.W}] frames, got {tuple(x.shape)}")
        x = x.detach().to(torch.float32)
        frames = x if self.pending is None else torch.cat([self.pending, x], dim=2)
        chunks = encode_chunks(frames.shape[2], self.first, self.tdf, self.spec.version)
        tzs = [self.native.latent_shape(n, self.H, self.W)[0] if i == 0 and self.first else n // self.tdf
               for i, n in enumerate(chunks)]
        Tz = sum(tzs)
        dev, s = frames.device, self.spec
        kl_noise = s.regularizer == "kl" and s.kl_sample
        if kl_noise:
            shape = (self.B, s.z_channels, Tz, self.Hz, self.Wz)
            if noise is None:
                noise = torch.randn(shape)   # CPU generator, as distributions.py:17
            elif tuple(noise.shape) != shape:
                raise ValueError(f"noise must have shape {shape} (this push's latent frames), got {tuple(noise.shape)}")
            noise = noise.to(device=dev, dtype=torch.float32).contiguous()
        z = torch.empty((self.B, s.z_channels, Tz, self.Hz, self.Wz), dtype=torch.float32, device=dev)
        idx = torch.empty((self.B, Tz, self.Hz, self.Wz), dtype=torch.int32, device=dev) if s.regularizer == "fsq" else None
        kls = torch.zeros((max(len(chunks), 1),), dtype=torch.float32, device=dev)
        t0 = tz0 = 0
        for i, (n, tz) in enumerate(zip(chunks, tzs)):
            xc = frames[:, :, t0:t0 + n].contiguous()
            zc = torch.empty((self.B, s.z_channels, tz, self.Hz, self.Wz), dtype=torch.float32, device=dev)
            ic = torch.empty((self.B, tz, self.Hz, self.Wz), dtype=torch.int32, device=dev) if idx is not None else None
            nc = noise[:, :, tz0:tz0 + tz].contiguous() if kl_noise else None
            ws = self._workspace(n)
            N.check(self.native.lib.vt_encode_chunk(self.state.handle, int(self.first), _ptr(xc), s.in_channels, n, _ptr(nc),
                                                    _ptr(zc), _ptr(ic), _ptr(kls[i:i + 1]) if s.regularizer == "kl" else None,
                                                    _ptr(ws), ws.numel(), _stream_ptr(dev)))
            z[:, :, tz0:tz0 + tz] = zc
            if idx is not None:
                idx[:, tz0:tz0 + tz] = ic
            self.first = False
            t0 += n
            tz0 += tz
        self.pending = frames[:, :, t0:].clone() if t0 < frames.shape[2] else None
        reg_log = {"indices": idx} if s.regularizer == "fsq" else {"kl_loss": kls.sum()}
        return z.to(self.out_dtype), reg_log


class DecodeStream(_Stream):
    def __init__(self, model, batch: int, Hz: int, Wz: int):
        super().__init__(model, batch, Hz, Wz, is_decoder=True)
        self.f = self.native.spatial_factor()

    def push(self, z: torch.Tensor) -> torch.Tensor:
        """z: latents [B,z_channels,tz,Hz,Wz], or FSQ token indices [B,tz,Hz,Wz] (integer tensor)."""
        if not z.is_cuda:
            raise RuntimeError("vidtok_b200: inputs must be CUDA tensors; there is no CPU path")
        s = self.spec
        if z.dim() == 4 and not z.is_floating_point():
            if s.regularizer != "fsq":
                raise ValueError("token indices need an FSQ model")
            z = self.model.indices_to_latent(z)
        if z.dim() != 5 or tuple(z.shape[:2]) != (self.B, s.z_channels) or tuple(z.shape[3:]) != (self.H, self.W):
            raise ValueError(f"expected a [{self.B},{s.z_channels},tz,{self.H},{self.W}] latent, got {tuple(z.shape)}")
        z = z.detach().to(torch.float32).contiguous()
        tz = z.shape[2]
        if tz == 0:
            return torch.empty((self.B, s.out_ch, 0, self.H * self.f, self.W * self.f), dtype=self.out_dtype, device=z.device)
        # v1.1: the first latent frame is a chunk of its own (build_chunk_start_end)
        chunks = [1, tz - 1] if self.first and s.version == 1 and tz > 1 else [tz]
        outs = []
        t0 = 0
        for n in chunks:
            To = self.native.decoded_frames(n) if (self.first or s.version == 1) else n * self.tdf
            out = torch.empty((self.B, s.out_ch, To, self.H * self.f, self.W * self.f), dtype=torch.float32, device=z.device)
            ws = self._workspace(n)
            N.check(self.native.lib.vt_decode_chunk(self.state.handle, int(self.first), _ptr(z[:, :, t0:t0 + n].contiguous()), s.z_channels,
                                                    n, _ptr(out), _ptr(ws), ws.numel(), _stream_ptr(z.device)))
            outs.append(out)
            self.first = False
            t0 += n
        x = outs[0] if len(outs) == 1 else torch.cat(outs, dim=2)
        return x.to(self.out_dtype)
