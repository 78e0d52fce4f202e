"""Streaming encode / decode of causal tokenizers: a video is pushed a few frames at a time and the memory in use does not
grow with its length.

    enc = EncodeStream(model, batch=B, H=H, W=W)
    for frames in source:                  # [B, C, t, H, W], any t
        z, reg_log = enc.push(frames)      # the latent frames this push completed (possibly none)
    dec = DecodeStream(model, batch=B, Hz=Hz, Wz=Wz)
    x = dec.push(z)                        # decoded frames of these latents

The reference's long-video recipe (v1.1 with use_tiling, t_chunk_enc = 16, t_chunk_dec = 16 // tdf, use_overlap) streams as

    enc = EncodeStream(model, B, H, W, t_chunk=16)
    dec = DecodeStream(model, B, Hz, Wz, t_chunk=16 // tdf, use_overlap=True)
    for frames in source:
        z, reg_log = enc.push(frames)
        x = dec.push(z)                    # the frames that are final (possibly none)
    z, reg_log = enc.flush()               # the last, shorter chunk
    x = torch.cat([dec.push(z), dec.flush()], dim=2)

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
* v1.1 models without `t_chunk`: the first frame is a chunk of its own, then complete tdf groups of each push, without
  overlap look-ahead.  The outputs equal `tile_encode` / `tile_decode(use_overlap=False)` when the pushes happen to fall
  on that chunking.
* v1.1 models with `t_chunk` (the chunks of build_chunk_start_end, whatever the push sizes): the encoder runs frame 0
  alone, then chunks of exactly `t_chunk` frames as soon as they are complete, and `flush()` encodes the remainder as the
  last, shorter chunk -- the outputs equal `tile_encode` with t_chunk_enc = t_chunk.  The decoder runs chunks of `t_chunk`
  latent frames; with `use_overlap` a chunk [s, e) is decoded once latent e has arrived, over z[s:e+1] with the look-ahead
  cache rule, and its last tdf frames are dropped (autoencoder_v1_1.py:322-330), and `flush()` decodes the final chunk
  without look-ahead -- the outputs equal `tile_decode` with t_chunk_dec = t_chunk and the same use_overlap.
  Latency: one chunk, plus one latent frame (tdf input frames) with overlap.
* Non-causal models cannot stream (their time padding is symmetric) and are rejected at creation.

Memory: the chunk workspace, the per-layer caches, at most one chunk of buffered input, and O(codebook size) for the FSQ
aux loss -- none of it grows with the video.

Precision is fixed at creation from `model.precision` / the autocast state, as `encode` reads it.  `reg_log` is per push:
`indices` (FSQ) or `kl_loss` (KL).  Without `t_chunk`, `kl_loss` is the push's share (the per-push values sum to the whole
clip's); with `t_chunk` it is tile_encode's value over the chunks encoded so far (the mean of the per-chunk values).  FSQ
streams also return `aux_loss` (a device scalar; zero when both aux weights are zero), the value over everything encoded so
far, with n_steps = global_step // 2 as `encode` uses:
  - v1.0: the whole clip's, all tokens as one segment (token-weighted running sums of the per-chunk partials);
  - v1.1: tile_encode's, the mean over the stream's chunks of each chunk's aux.
Streams use world size 1: ranks need not push in lockstep, so avg_prob is not all-reduced across ranks.  KL noise is one
CPU `torch.randn` per push over the push's latent frames (with `t_chunk`: one per chunk, in chunk order, the draws
tile_encode makes) unless `noise` is passed.  No push synchronises with the host.
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


def recipe_encode_chunks(avail: int, first: bool, t_chunk: int, final: bool) -> List[int]:
    """Frame counts of the build_chunk_start_end chunks (autoencoder_v1_1.py:218-228) that `avail` buffered frames
    complete: the first frame alone, then t_chunk frames each; `final` (the video has ended) adds the remainder as the
    last, shorter chunk."""
    out = []
    while avail > 0:
        n = 1 if first else t_chunk
        if avail < n:
            if final:
                out.append(avail)
            break
        out.append(n)
        avail -= n
        first = False
    return out


def recipe_decode_chunks(avail: int, first: bool, t_chunk: int, use_overlap: bool, tdf: int,
                         final: bool) -> List[Tuple[int, int, int]]:
    """The build_chunk_start_end(decoder_mode=True) chunks that `avail` buffered latent frames let the decoder run, as
    (latent frames decoded, latent frames the chunk covers, decoded frames dropped at its tail).  With use_overlap a chunk
    is decoded together with the next latent frame, its look-ahead, and its last tdf frames are dropped
    (autoencoder_v1_1.py:322-330), so it waits for that frame; `final` decodes the last chunk without look-ahead."""
    out = []
    look = 1 if use_overlap else 0
    while avail > 0:
        n = 1 if first else t_chunk
        if avail >= n + look:
            out.append((n + look, n, tdf * look))
        elif final:
            out.append((avail, avail, 0))   # avail <= n here: the last chunk, min(t, end + step)
            break
        else:
            break
        avail -= n
        first = False
    return out


def check_recipe(version: int, tdf: int, t_chunk: Optional[int], use_overlap: bool, is_decoder: bool):
    """The stream options build_chunk_start_end and the overlap rule accept (ValueError otherwise)."""
    if t_chunk is not None:
        if version != 1:
            raise ValueError("t_chunk needs a v1.1 model: v1.0 streams equal the whole clip for any chunking")
        if int(t_chunk) < 1 or (not is_decoder and int(t_chunk) % tdf != 0):
            raise ValueError(f"t_chunk must be a positive multiple of time_downsample_factor ({tdf}), got {t_chunk}"
                             if not is_decoder else f"t_chunk must be a positive number of latent frames, got {t_chunk}")
    if use_overlap:
        if t_chunk is None or version != 1:
            raise ValueError("use_overlap needs a v1.1 model and t_chunk (the look-ahead follows the tile_decode chunks)")
        if tdf not in (2, 4, 8):
            raise ValueError("use_overlap supports 2x, 4x or 8x temporal downsampling only")


class _Stream:
    def __init__(self, model, batch: int, H: int, W: int, is_decoder: bool, t_chunk: Optional[int] = None,
                 use_overlap: bool = False):
        if not model.is_causal:
            raise ValueError("non-causal models cannot stream: their time padding is symmetric, so a frame depends on later frames")
        self.tdf = int(model.spec.time_downsample_factor)
        check_recipe(model.spec.version, self.tdf, t_chunk, use_overlap, is_decoder)
        self.t_chunk = None if t_chunk is None else int(t_chunk)
        self.use_overlap = bool(use_overlap)
        rt = model._rt
        self.model = model
        self.native = rt.sync()
        self.spec = model.spec
        self.precision = rt.precision()
        self.out_dtype = rt.out_dtype()
        self.B, self.H, self.W = int(batch), int(H), int(W)
        self.state = ChunkState(self.native, self.precision, self.B, self.H, self.W, is_decoder, self.use_overlap)
        self.first = True
        self.finished = False

    def reset(self):
        """Start a new video: the next push is its first chunk (the caches are rewritten, not read)."""
        self.first = True
        self.finished = False

    def close(self):
        self.state.close()

    def _workspace(self, n: int) -> torch.Tensor:
        return self.state.workspace(n)

    def _check_open(self):
        if self.finished:
            raise RuntimeError("the stream was flushed: call reset() to start a new video")


class EncodeStream(_Stream):
    """keep_pre_bound: reg_log also holds "h_pre", the encoder output before the regularizer of this push's latent frames
    ([B, 2z|z, tz, Hz, Wz]), so that a caller can form per-sample losses of a batched stream; the stream's own FSQ aux loss
    is then not formed."""

    def __init__(self, model, batch: int, H: int, W: int, t_chunk: Optional[int] = None, keep_pre_bound: bool = False):
        super().__init__(model, batch, H, W, is_decoder=False, t_chunk=t_chunk)
        self.keep_pre = bool(keep_pre_bound)
        self.pending: Optional[torch.Tensor] = None
        self.Hz, self.Wz = self.native.latent_shape(1, H, W)[1:]
        self.reg = model.regularization
        self.aux = self.spec.regularizer == "fsq" and self.reg.aux_enabled() and not self.keep_pre
        if self.aux:
            dev, J = self.native.device, self.reg.codebook_size
            self.aux_stats = torch.empty((1, 2), dtype=torch.float32, device=dev)   # one chunk's partials
            self.aux_avg = torch.empty((1, J), dtype=torch.float32, device=dev)
        self._reset_losses()

    def _reset_losses(self):
        dev = self.native.device
        self.n_chunks = 0
        self.kl_sum = torch.zeros((), dtype=torch.float32, device=dev)
        self.aux_loss = torch.zeros((), dtype=torch.float32, device=dev)
        if self.aux:
            self.aux_sum = torch.zeros((), dtype=torch.float32, device=dev)        # v1.1: running sum of per-chunk aux
            self.tok_stats = torch.zeros((2,), dtype=torch.float64, device=dev)    # v1.0: token-weighted partials
            self.tok_avg = torch.zeros((self.reg.codebook_size,), dtype=torch.float64, device=dev)
            self.tokens = 0

    def reset(self):
        super().reset()
        self.pending = None
        self._reset_losses()

    def push(self, x: torch.Tensor, noise: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, Dict[str, torch.Tensor]]:
        """x: frames [B,C,t,H,W], any t.  Returns the latent frames of the chunks this push completed (possibly none) and
        reg_log; noise (KL with sampling, optional): [B,z_channels,tz,Hz,Wz] for those latent frames."""
        self._check_open()
        if not x.is_cuda:
            raise RuntimeError("vidtok_b200: inputs must be CUDA tensors; there is no CPU path")
        if x.dim() != 5 or tuple(x.shape[:2]) != (self.B, self.spec.in_channels) or tuple(x.shape[3:]) != (self.H, self.W):
            raise ValueError(f"expected [{self.B},{self.spec.in_channels},t,{self.H},{self.W}] frames, got {tuple(x.shape)}")
        x = x.detach().to(torch.float32)
        frames = x if self.pending is None else torch.cat([self.pending, x], dim=2)
        if self.t_chunk is None:
            chunks = encode_chunks(frames.shape[2], self.first, self.tdf, self.spec.version)
        else:
            chunks = recipe_encode_chunks(frames.shape[2], self.first, self.t_chunk, final=False)
        return self._encode(frames, chunks, noise)

    def flush(self, noise: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, Dict[str, torch.Tensor]]:
        """End of the video: encodes the frames still held back as the last, shorter chunk (v1.1; a v1.0 stream has
        nothing held back when the video has 1 + k * tdf frames, and refuses otherwise).  Pushes are refused afterwards
        until reset()."""
        self._check_open()
        n = 0 if self.pending is None else int(self.pending.shape[2])
        if n and self.spec.version == 0:
            raise ValueError(f"{n} frames do not complete a group of {self.tdf}: a v1.0 stream encodes videos of 1 + k * {self.tdf} frames")
        frames = self.pending if n else torch.empty((self.B, self.spec.in_channels, 0, self.H, self.W), device=self.native.device)
        self.finished = True
        return self._encode(frames, [n] if n else [], noise)

    def _encode(self, frames: torch.Tensor, chunks: List[int], noise: Optional[torch.Tensor]):
        tzs = [self.native.latent_shape(n, self.H, self.W)[0] for n in chunks]
        Tz = sum(tzs)
        dev, s = frames.device, self.spec
        kl_noise = s.regularizer == "kl" and s.kl_sample
        if kl_noise:
            shape = (self.B, s.z_channels, Tz, self.Hz, self.Wz)
            if noise is None:
                # CPU generator, as distributions.py:17: one draw per push, or per chunk in chunk order as tile_encode
                noise = (torch.randn(shape) if self.t_chunk is None or not tzs else
                         torch.cat([torch.randn((self.B, s.z_channels, tz, self.Hz, self.Wz)) for tz in tzs], dim=2))
            elif tuple(noise.shape) != shape:
                raise ValueError(f"noise must have shape {shape} (this push's latent frames), got {tuple(noise.shape)}")
            noise = noise.to(device=dev, dtype=torch.float32).contiguous()
        z = torch.empty((self.B, s.z_channels, Tz, self.Hz, self.Wz), dtype=torch.float32, device=dev)
        idx = torch.empty((self.B, Tz, self.Hz, self.Wz), dtype=torch.int32, device=dev) if s.regularizer == "fsq" else None
        kls = torch.zeros((max(len(chunks), 1),), dtype=torch.float32, device=dev)
        hC = (2 if s.double_z else 1) * s.z_channels
        h = torch.empty((self.B, hC, Tz, self.Hz, self.Wz), dtype=torch.float32, device=dev) if self.keep_pre else None
        lib, stream = self.native.lib, _stream_ptr(dev)
        t0 = tz0 = 0
        for i, (n, tz) in enumerate(zip(chunks, tzs)):
            xc = frames[:, :, t0:t0 + n].contiguous()
            zc = torch.empty((self.B, s.z_channels, tz, self.Hz, self.Wz), dtype=torch.float32, device=dev)
            ic = torch.empty((self.B, tz, self.Hz, self.Wz), dtype=torch.int32, device=dev) if idx is not None else None
            nc = noise[:, :, tz0:tz0 + tz].contiguous() if kl_noise else None
            if self.keep_pre:
                ws = self._workspace(n)
                hc = torch.empty((self.B, hC, tz, self.Hz, self.Wz), dtype=torch.float32, device=dev)
                N.check(lib.vt_encode_chunk_pre(self.state.handle, int(self.first), _ptr(xc), s.in_channels, n, _ptr(nc), _ptr(zc),
                                                _ptr(ic), _ptr(kls[i:i + 1]) if s.regularizer == "kl" else None, _ptr(hc), _ptr(ws),
                                                ws.numel(), stream))
                h[:, :, tz0:tz0 + tz] = hc
            elif self.aux:
                ws = self.state.aux_workspace(n)
                N.check(lib.vt_encode_chunk_fsq_aux(self.state.handle, int(self.first), _ptr(xc), s.in_channels, n, _ptr(zc), _ptr(ic),
                                                    100.0, _ptr(self.aux_stats), _ptr(self.aux_avg), _ptr(ws), ws.numel(), stream))
                self._add_aux_chunk(self.B * tz * self.Hz * self.Wz)
            else:
                ws = self._workspace(n)
                N.check(lib.vt_encode_chunk(self.state.handle, int(self.first), _ptr(xc), s.in_channels, n, _ptr(nc), _ptr(zc),
                                            _ptr(ic), _ptr(kls[i:i + 1]) if s.regularizer == "kl" else None, _ptr(ws), ws.numel(),
                                            stream))
            z[:, :, tz0:tz0 + tz] = zc
            if idx is not None:
                idx[:, tz0:tz0 + tz] = ic
            if self.t_chunk is not None and s.regularizer == "kl":
                self.kl_sum = self.kl_sum + kls[i]   # in chunk order, as tile_encode's mean sums them
            self.first = False
            self.n_chunks += 1
            t0 += n
            tz0 += tz
        self.pending = frames[:, :, t0:].clone() if t0 < frames.shape[2] else None
        if s.regularizer == "fsq":
            if self.aux and chunks and s.version == 0:
                self.aux_loss = self.reg.aux_finalize((self.tok_stats / self.tokens).float().view(1, 2),
                                                      (self.tok_avg / self.tokens).float().view(1, -1),
                                                      n_steps=self.model.global_step // 2, world_size=1)
            log = {"indices": idx, "aux_loss": self.aux_loss}
        else:
            if self.t_chunk is None:
                kl = kls.sum()
            else:
                kl = self._mean(self.kl_sum, self.n_chunks) if self.n_chunks else torch.zeros((), dtype=torch.float32, device=dev)
            log = {"kl_loss": kl}
        if self.keep_pre:
            log["h_pre"] = h
        return z.to(self.out_dtype), log

    @staticmethod
    def _mean(total: torch.Tensor, n: int) -> torch.Tensor:
        """total / n rounded once, as the library's per-chunk means divide (a Python divisor would be applied as a
        multiplication by its reciprocal)"""
        return total / torch.full((), float(n), dtype=torch.float32, device=total.device)

    def _add_aux_chunk(self, tokens: int):
        """Fold the partials one chunk just wrote into the stream's running aux state."""
        if self.spec.version == 0:
            self.tok_stats += tokens * self.aux_stats[0].double()
            self.tok_avg += tokens * self.aux_avg[0].double()
            self.tokens += tokens
        else:
            aux = self.reg.aux_finalize(self.aux_stats, self.aux_avg, n_steps=self.model.global_step // 2, world_size=1)
            self.aux_sum = self.aux_sum + aux
            self.aux_loss = self._mean(self.aux_sum, self.n_chunks + 1)


class DecodeStream(_Stream):
    def __init__(self, model, batch: int, Hz: int, Wz: int, t_chunk: Optional[int] = None, use_overlap: bool = False):
        super().__init__(model, batch, Hz, Wz, is_decoder=True, t_chunk=t_chunk, use_overlap=use_overlap)
        self.f = self.native.spatial_factor()
        self.pending: Optional[torch.Tensor] = None

    def reset(self):
        super().reset()
        self.pending = None

    def _empty(self, device) -> torch.Tensor:
        return torch.empty((self.B, self.spec.out_ch, 0, self.H * self.f, self.W * self.f), dtype=self.out_dtype, device=device)

    def push(self, z: torch.Tensor) -> torch.Tensor:
        """z: latents [B,z_channels,tz,Hz,Wz], or FSQ token indices [B,tz,Hz,Wz] (integer tensor).  Returns the decoded
        frames that are final (with t_chunk possibly none)."""
        self._check_open()
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
        if self.t_chunk is not None:
            z = z if self.pending is None else torch.cat([self.pending, z], dim=2)
            return self._decode(z, recipe_decode_chunks(z.shape[2], self.first, self.t_chunk, self.use_overlap, self.tdf, False))
        tz = z.shape[2]
        if tz == 0:
            return self._empty(z.device)
        # v1.1: the first latent frame is a chunk of its own (build_chunk_start_end)
        chunks = [1, tz - 1] if self.first and s.version == 1 and tz > 1 else [tz]
        return self._decode(z, [(n, n, 0) for n in chunks])

    def flush(self) -> torch.Tensor:
        """End of the video: decodes the latent frames still held back (with t_chunk) as the last chunk, without
        look-ahead.  Pushes are refused afterwards until reset()."""
        self._check_open()
        self.finished = True
        if self.pending is None:
            return self._empty(self.native.device)
        return self._decode(self.pending, recipe_decode_chunks(self.pending.shape[2], self.first, self.t_chunk, self.use_overlap,
                                                               self.tdf, True))

    def _decode(self, z: torch.Tensor, plan: List[Tuple[int, int, int]]) -> torch.Tensor:
        s = self.spec
        outs = []
        t0 = 0
        for n, step, trim in plan:
            To = self.native.decoded_frames(n) if (self.first or s.version == 1) else n * self.tdf
            out = torch.empty((self.B, s.out_ch, To, self.H * self.f, self.W * self.f), dtype=torch.float32, device=z.device)
            ws = self._workspace(n)
            N.check(self.native.lib.vt_decode_chunk(self.state.handle, int(self.first), _ptr(z[:, :, t0:t0 + n].contiguous()), s.z_channels,
                                                    n, _ptr(out), _ptr(ws), ws.numel(), _stream_ptr(z.device)))
            outs.append(out[:, :, :To - trim] if trim else out)
            self.first = False
            t0 += step
        self.pending = z[:, :, t0:].clone() if t0 < z.shape[2] else None
        if not outs:
            return self._empty(z.device)
        x = outs[0].contiguous() if len(outs) == 1 else torch.cat(outs, dim=2)
        return x.to(self.out_dtype)
