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
tile_encode makes) unless `noise` is passed.  No push synchronises with the host.  A stream replays its steady chunks
from CUDA graphs (ChunkGraphs): the same native calls on static buffers, so the outputs are those of the eager chunks.

Pools (EncodePool / DecodePool) carry many videos that start and end independently through one chunk state of batch S
(the capacity), one slot per video.  Every chunk of a video is a chunk of its own recipe stream (PoolSchedule):
  - its first chunk runs on a side state of batch 1 and is then transplanted into its slot
    (vt_chunk_state_copy_slots: every cache of the slot, in one launch);
  - later chunks of exactly t_chunk frames (decoder: t_chunk latent frames, plus the look-ahead frame with use_overlap)
    run as one batched chunk of all S slots per step();
  - close() transplants the slot out to the side state and runs the rest there: v1.1's short last chunk, the decoder's
    last chunk without look-ahead.
A batched chunk advances the caches of every row, so a started video without a full chunk buffered sits the step out:
its slot is copied to a parking state before the batched chunk and back after it (two transplants of that slot's caches
per step it waits; none while every open video keeps up).  Empty slots run on zeros and their outputs are dropped.
Each slot's outputs are therefore its own tile_encode / tile_decode (v1.1) or whole-clip encode / decode (v1.0): bit for
bit in "bf16" and "fma"; in "exact" and "mixed" to fp32 rounding, since the split-operand kernels' tiles (and so their
rounding) may depend on the batch.  Per-slot losses are formed from each video's own slice of the pre-bound latent
(vt_encode_chunk_pre): kl_loss with vt_op_kl per chunk, FSQ aux_loss from vt_fsq_aux_partials / vt_fsq_aux_finalize per
chunk, both over everything the video encoded so far, as the streams report them.  Non-causal models are refused; world
size 1, as the streams.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Tuple

import torch

from . import _native as N
from .engine import ChunkState, _ptr, _refuse_capture, _stream_ptr, chunk_noise


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


def chunk_graph_key(n: int, first: bool, final: bool, entry: str, parity: int) -> Optional[Tuple[int, str, int]]:
    """The CUDA graph a stream chunk replays: None (eager) for a video's first chunk and for the chunk flush() runs, else
    (frames or latent frames in, entry point, cache parity).  A graph reads one buffer of every double-buffered cache and
    writes the other, so it is only valid at the parity it was captured at."""
    if first or final:
        return None
    return (int(n), entry, int(parity))


class ChunkGraphs:
    """The CUDA graphs of one stream's steady chunks.  A key that occurs for the first time runs eagerly (lengths seen once
    never pay for a capture); its second occurrence is captured, after vt_chunk_state_reserve, and runs as the graph's
    first replay; every later occurrence replays.  Each graph owns static input / output buffers: a push copies its chunk in
    and its results out, so the tensors it returns are fresh.  The workspace is one of them, sized eagerly before the
    capture and held there: the graph keeps reading it if the model's workspace grows."""

    def __init__(self):
        self.seen: Dict[Tuple, int] = {}
        self.graphs: Dict[Tuple, Dict] = {}
        self.runs: Dict[Tuple, int] = {}   # per key: chunks run by replaying its graph (the capture's own run included)
        self.replays = 0                    # over all keys
        self.captures = 0

    def action(self, key: Optional[Tuple]) -> str:
        """"eager", "capture" or "replay" for the next chunk of this key (counts the occurrence)."""
        if key is None:
            return "eager"
        if key in self.graphs:
            return "replay"
        self.seen[key] = self.seen.get(key, 0) + 1
        return "eager" if self.seen[key] < 2 else "capture"

    def run(self, key: Tuple, action: str, state: ChunkState, launch, bufs: Dict) -> Dict:
        """Captures (action "capture", launch() being the chunk's native call on the static buffers `bufs`) or looks up the
        graph of key, replays it and advances the state's caches as the chunk call would have.  Returns the static buffers."""
        lib = state.native.lib
        if action == "capture":
            N.check(lib.vt_chunk_state_reserve(state.handle, key[0], _stream_ptr(state.native.device)))
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                launch(bufs)                   # capturing flips the caches' parity, as running the chunk does
            bufs["graph"] = g
            self.graphs[key] = bufs
            self.captures += 1
            g.replay()
        else:
            bufs = self.graphs[key]
            bufs["graph"].replay()
            N.check(lib.vt_chunk_state_advance(state.handle))
        self.runs[key] = self.runs.get(key, 0) + 1
        self.replays += 1
        return bufs


def _check_t_chunk(tdf: int, t_chunk: int, is_decoder: bool):
    if int(t_chunk) < 1 or (not is_decoder and int(t_chunk) % tdf != 0):
        raise ValueError(f"t_chunk must be a positive multiple of time_downsample_factor ({tdf}), got {t_chunk}"
                         if not is_decoder else f"t_chunk must be a positive number of latent frames, got {t_chunk}")


def check_recipe(version: int, tdf: int, t_chunk: Optional[int], use_overlap: bool, is_decoder: bool):
    """The stream options build_chunk_start_end and the overlap rule accept (ValueError otherwise)."""
    if t_chunk is not None:
        if version != 1:
            raise ValueError("t_chunk needs a v1.1 model: v1.0 streams equal the whole clip for any chunking")
        _check_t_chunk(tdf, t_chunk, is_decoder)
    if use_overlap:
        if t_chunk is None or version != 1:
            raise ValueError("use_overlap needs a v1.1 model and t_chunk (the look-ahead follows the tile_decode chunks)")
        if tdf not in (2, 4, 8):
            raise ValueError("use_overlap supports 2x, 4x or 8x temporal downsampling only")


def check_pool_recipe(version: int, tdf: int, t_chunk: Optional[int], use_overlap: bool, is_decoder: bool):
    """The options a pool accepts (ValueError otherwise): every pool has a chunk length, t_chunk frames (encoder, a
    multiple of tdf) or latent frames (decoder); v1.1 pools follow the stream recipe's rules."""
    if t_chunk is None:
        raise ValueError("a pool needs t_chunk: the batched chunks of all its slots have one length")
    # a v1.0 pool's chunks are valid v1.0 stream chunks, which need no t_chunk
    check_recipe(version, tdf, t_chunk if version == 1 else None, use_overlap, is_decoder)
    _check_t_chunk(tdf, t_chunk, is_decoder)


class _Chunked:
    """The set-up and input checks of streams and pools: the options are checked before the model is loaded, and the
    precision is fixed at creation, as encode reads it."""

    def __init__(self, model, H: int, W: int, is_decoder: bool, t_chunk: Optional[int], use_overlap: bool, check):
        if not model.is_causal:
            raise ValueError("non-causal models cannot stream: their time padding is symmetric, so a frame depends on later frames")
        self.tdf = int(model.spec.time_downsample_factor)
        check(model.spec.version, self.tdf, t_chunk, use_overlap, is_decoder)
        self.t_chunk = None if t_chunk is None else int(t_chunk)
        self.use_overlap = bool(use_overlap)
        rt = model._rt
        self.model = model
        self.native = rt.sync()
        self.spec = model.spec
        self.precision = rt.precision()
        self.out_dtype = rt.out_dtype()
        self.H, self.W = int(H), int(W)

    def _frames(self, x: torch.Tensor, B: int) -> torch.Tensor:
        """x checked as frames [B,C,t,H,W], in fp32"""
        if not x.is_cuda:
            raise RuntimeError("vidtok_b200: inputs must be CUDA tensors; there is no CPU path")
        if x.dim() != 5 or tuple(x.shape[:2]) != (B, self.spec.in_channels) or tuple(x.shape[3:]) != (self.H, self.W):
            raise ValueError(f"expected [{B},{self.spec.in_channels},t,{self.H},{self.W}] frames, got {tuple(x.shape)}")
        return x.detach().to(torch.float32)

    def _latents(self, z: torch.Tensor, B: int) -> torch.Tensor:
        """z checked as latents [B,z_channels,tz,Hz,Wz] or FSQ token indices [B,tz,Hz,Wz], as an fp32 latent"""
        if not z.is_cuda:
            raise RuntimeError("vidtok_b200: inputs must be CUDA tensors; there is no CPU path")
        s = self.spec
        if z.dim() == 4 and not z.is_floating_point():
            if s.regularizer != "fsq":
                raise ValueError("token indices need an FSQ model")
            z = self.model.indices_to_latent(z)
        if z.dim() != 5 or tuple(z.shape[:2]) != (B, s.z_channels) or tuple(z.shape[3:]) != (self.H, self.W):
            raise ValueError(f"expected a [{B},{s.z_channels},tz,{self.H},{self.W}] latent, got {tuple(z.shape)}")
        return z.detach().to(torch.float32)


def _mean(total: torch.Tensor, n: int) -> torch.Tensor:
    """total / n rounded once, as the library's per-chunk means divide (a Python divisor would be applied as a
    multiplication by its reciprocal)"""
    return total / torch.full((), float(n), dtype=torch.float32, device=total.device)


class _Losses:
    """One video's running losses over its chunks, as tile_encode (v1.1) or the whole clip (v1.0) forms them.  KL: the
    chunks' values summed in chunk order, reported as their mean (v1.1) or their sum (v1.0).  FSQ aux: v1.1 the mean over
    the chunks of each chunk's aux; v1.0 all of the video's tokens as one segment, from token-weighted fp64 sums of the
    chunks' partials, finalized when reported."""

    def __init__(self, model, device: torch.device, aux: bool):
        self.model = model
        self.n_chunks = 0
        self.kl_sum = torch.zeros((), dtype=torch.float32, device=device)
        self._aux = torch.zeros((), dtype=torch.float32, device=device)
        self._unreported = False   # v1.0: partials folded since _aux was finalized
        if aux:
            self.aux_sum = torch.zeros((), dtype=torch.float32, device=device)
            self.tok_stats = torch.zeros((2,), dtype=torch.float64, device=device)
            self.tok_avg = torch.zeros((model.regularization.codebook_size,), dtype=torch.float64, device=device)
            self.tokens = 0

    def add(self, kl: Optional[torch.Tensor] = None, partials: Optional[Tuple[torch.Tensor, torch.Tensor]] = None,
            tokens: int = 0):
        """One chunk: its KL value, or its FSQ aux partials (stats [1,2], avg [1,J]) over `tokens` tokens."""
        self.n_chunks += 1
        if kl is not None:
            self.kl_sum = self.kl_sum + kl
        if partials is None:
            return
        stats, avg = partials
        if self.model.spec.version == 0:
            self.tok_stats += tokens * stats[0].double()
            self.tok_avg += tokens * avg[0].double()
            self.tokens += tokens
            self._unreported = True
        else:
            self.aux_sum = self.aux_sum + self._finalize(stats, avg)
            self._aux = _mean(self.aux_sum, self.n_chunks)

    def kl_loss(self) -> torch.Tensor:
        if self.model.spec.version == 0:
            return self.kl_sum
        if not self.n_chunks:
            return torch.zeros((), dtype=torch.float32, device=self.kl_sum.device)
        return _mean(self.kl_sum, self.n_chunks)

    def aux_loss(self) -> torch.Tensor:
        if self._unreported:
            self._aux = self._finalize((self.tok_stats / self.tokens).float().view(1, 2),
                                       (self.tok_avg / self.tokens).float().view(1, -1))
            self._unreported = False
        return self._aux

    def _finalize(self, stats: torch.Tensor, avg: torch.Tensor) -> torch.Tensor:
        return self.model.regularization.aux_finalize(stats, avg, n_steps=self.model.global_step // 2, world_size=1)


def _loss_terms(native, reg, h: torch.Tensor, kl: Optional[torch.Tensor] = None):
    """One chunk's loss terms from its own pre-bound latent h [1,2z|z,tz,Hz,Wz] (dense), apart from the batch it ran in: a
    KL model's KL value (vt_op_kl into a scratch z; written to `kl`, else to a new scalar), an FSQ model's aux partials
    (stats, avg)."""
    s, dev = native.spec, native.device
    if s.regularizer != "kl":
        return reg.aux_partials(h)
    zs = torch.empty((1, s.z_channels) + tuple(h.shape[2:]), dtype=torch.float32, device=dev)
    kl = torch.empty((), dtype=torch.float32, device=dev) if kl is None else kl
    N.check(native.lib.vt_op_kl(_ptr(h), None, s.z_channels, h.shape[2] * h.shape[3] * h.shape[4], 1, 0, _ptr(zs), _ptr(kl),
                                _stream_ptr(dev)))
    return kl


class _Stream(_Chunked):
    def __init__(self, model, batch: int, H: int, W: int, is_decoder: bool, t_chunk: Optional[int] = None,
                 use_overlap: bool = False):
        super().__init__(model, H, W, is_decoder, t_chunk, use_overlap, check_recipe)
        self.B = int(batch)
        self.state = ChunkState(self.native, self.precision, self.B, self.H, self.W, is_decoder, self.use_overlap)
        self.first = True
        self.finished = False
        self.graphs = ChunkGraphs()

    def reset(self):
        """Start a new video: the next push is its first chunk (the caches are rewritten, not read)."""
        self.first = True
        self.finished = False

    def close(self):
        self.graphs = ChunkGraphs()
        self.state.close()

    def _graph_action(self, n: int, final: bool, entry: str) -> Tuple[Optional[Tuple], str]:
        key = chunk_graph_key(n, self.first, final, entry, self.native.lib.vt_chunk_state_parity(self.state.handle))
        return key, self.graphs.action(key)

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
            # one chunk's partials, at fixed addresses: a captured graph writes them there
            dev, J = self.native.device, self.reg.codebook_size
            self.aux_stats = torch.empty((1, 2), dtype=torch.float32, device=dev)
            self.aux_avg = torch.empty((1, J), dtype=torch.float32, device=dev)
        self.losses = _Losses(model, self.native.device, self.aux)

    def reset(self):
        super().reset()
        self.pending = None
        self.losses = _Losses(self.model, self.native.device, self.aux)

    def push(self, x: torch.Tensor, noise: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, Dict[str, torch.Tensor]]:
        """x: frames [B,C,t,H,W], any t.  Returns the latent frames of the chunks this push completed (possibly none) and
        reg_log; noise (KL with sampling, optional): [B,z_channels,tz,Hz,Wz] for those latent frames."""
        self._check_open()
        x = self._frames(x, self.B)
        frames = x if self.pending is None else torch.cat([self.pending, x], dim=2)
        if self.t_chunk is None:
            chunks = encode_chunks(frames.shape[2], self.first, self.tdf, self.spec.version)
        else:
            chunks = recipe_encode_chunks(frames.shape[2], self.first, self.t_chunk, final=False)
        return self._encode(frames, chunks, noise, final=False)

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
        return self._encode(frames, [n] if n else [], noise, final=True)

    def _encode(self, frames: torch.Tensor, chunks: List[int], noise: Optional[torch.Tensor], final: bool):
        tzs = [self.native.latent_shape(n, self.H, self.W)[0] for n in chunks]
        Tz = sum(tzs)
        dev, s = frames.device, self.spec
        kl_noise = s.regularizer == "kl" and s.kl_sample
        if kl_noise:
            shape = (self.B, s.z_channels, Tz, self.Hz, self.Wz)
            if noise is None:
                # one draw per push, or per chunk as tile_encode draws them
                noise = chunk_noise(self.B, s.z_channels, tzs if self.t_chunk is not None and tzs else [Tz], self.Hz, self.Wz)
            elif tuple(noise.shape) != shape:
                raise ValueError(f"noise must have shape {shape} (this push's latent frames), got {tuple(noise.shape)}")
            noise = noise.to(device=dev, dtype=torch.float32).contiguous()
        z = torch.empty((self.B, s.z_channels, Tz, self.Hz, self.Wz), dtype=torch.float32, device=dev)
        idx = torch.empty((self.B, Tz, self.Hz, self.Wz), dtype=torch.int32, device=dev) if s.regularizer == "fsq" else None
        kls = torch.zeros((max(len(chunks), 1),), dtype=torch.float32, device=dev)
        hC = (2 if s.double_z else 1) * s.z_channels
        h = torch.empty((self.B, hC, Tz, self.Hz, self.Wz), dtype=torch.float32, device=dev) if self.keep_pre else None
        aux = (self.aux_stats, self.aux_avg) if self.aux else None
        entry = "pre" if self.keep_pre else ("fsq_aux" if self.aux else "plain")
        t0 = tz0 = 0
        for i, (n, tz) in enumerate(zip(chunks, tzs)):
            xc, nc = frames[:, :, t0:t0 + n], noise[:, :, tz0:tz0 + tz] if kl_noise else None
            kl = kls[i:i + 1] if s.regularizer == "kl" else None
            key, action = self._graph_action(n, final, entry)
            if action == "eager":
                b = self.state.encode(xc.contiguous(), self.first, None if nc is None else nc.contiguous(), self.keep_pre, aux,
                                      out={"kl": kl})
            else:
                g = self.graphs.graphs[key] if action == "replay" else self._graph_buffers(n, tz, kl_noise)
                g["x"].copy_(xc)
                if kl_noise:
                    g["noise"].copy_(nc)
                b = self.graphs.run(key, action, self.state, self._launch_encode, g)
                if kl is not None:
                    kl.copy_(b["kl"])
            z[:, :, tz0:tz0 + tz] = b["z"]
            if idx is not None:
                idx[:, tz0:tz0 + tz] = b["idx"]
            if self.keep_pre:
                h[:, :, tz0:tz0 + tz] = b["h"]
            # KL in chunk order for tile_encode's mean; without t_chunk a push reports its own share
            self.losses.add(kl=kls[i] if self.t_chunk is not None and kl is not None else None, partials=aux,
                            tokens=self.B * tz * self.Hz * self.Wz)
            self.first = False
            t0 += n
            tz0 += tz
        self.pending = frames[:, :, t0:].clone() if t0 < frames.shape[2] else None
        if s.regularizer == "fsq":
            log = {"indices": idx, "aux_loss": self.losses.aux_loss()}
        else:
            log = {"kl_loss": kls.sum() if self.t_chunk is None else self.losses.kl_loss()}
        if self.keep_pre:
            log["h_pre"] = h
        return z.to(self.out_dtype), log

    def _graph_buffers(self, n: int, tz: int, kl_noise: bool) -> Dict:
        """New static buffers of a chunk graph: the chunk's frames and noise, and encode_buffers."""
        s, dev = self.spec, self.native.device
        g = self.state.encode_buffers(n, self.keep_pre, self.aux)
        g["x"] = torch.empty((self.B, s.in_channels, n, self.H, self.W), dtype=torch.float32, device=dev)
        g["noise"] = torch.empty((self.B, s.z_channels, tz, self.Hz, self.Wz), dtype=torch.float32, device=dev) if kl_noise else None
        return g

    def _launch_encode(self, g: Dict):
        """The chunk's native call on a graph's static buffers (a later chunk: is_first 0)."""
        self.state.encode(g["x"], False, g["noise"], self.keep_pre, (self.aux_stats, self.aux_avg) if self.aux else None, out=g)


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
        z = self._latents(z, self.B).contiguous()
        if self.t_chunk is not None:
            z = z if self.pending is None else torch.cat([self.pending, z], dim=2)
            return self._decode(z, recipe_decode_chunks(z.shape[2], self.first, self.t_chunk, self.use_overlap, self.tdf, False),
                                final=False)
        tz = z.shape[2]
        if tz == 0:
            return self._empty(z.device)
        # v1.1: the first latent frame is a chunk of its own (build_chunk_start_end)
        chunks = [1, tz - 1] if self.first and self.spec.version == 1 and tz > 1 else [tz]
        return self._decode(z, [(n, n, 0) for n in chunks], final=False)

    def flush(self) -> torch.Tensor:
        """End of the video: decodes the latent frames still held back (with t_chunk) as the last chunk, without
        look-ahead.  Pushes are refused afterwards until reset()."""
        self._check_open()
        self.finished = True
        if self.pending is None:
            return self._empty(self.native.device)
        return self._decode(self.pending, recipe_decode_chunks(self.pending.shape[2], self.first, self.t_chunk, self.use_overlap,
                                                               self.tdf, True), final=True)

    def _decode(self, z: torch.Tensor, plan: List[Tuple[int, int, int]], final: bool) -> torch.Tensor:
        outs = []
        t0 = 0
        for n, step, trim in plan:
            zc = z[:, :, t0:t0 + n]
            key, action = self._graph_action(n, final, "plain")
            if action == "eager":
                out = self.state.decode(zc.contiguous(), self.first)
            else:
                g = self.graphs.graphs[key] if action == "replay" else dict(
                    self.state.decode_buffers(n, first=False),
                    z=torch.empty((self.B, self.spec.z_channels, n, self.H, self.W), dtype=torch.float32, device=z.device))
                g["z"].copy_(zc)
                out = self.graphs.run(key, action, self.state, self._launch_decode, g)["out"].clone()
            outs.append(out[:, :, :out.shape[2] - trim] if trim else out)
            self.first = False
            t0 += step
        self.pending = z[:, :, t0:].clone() if t0 < z.shape[2] else None
        if not outs:
            return self._empty(z.device)
        x = outs[0].contiguous() if len(outs) == 1 else torch.cat(outs, dim=2)
        return x.to(self.out_dtype)

    def _launch_decode(self, g: Dict):
        self.state.decode(g["z"], False, out=g)

# ---------------------------------------------------------------------------------------------------------------------
# Pools: many videos, each starting and ending on its own, through one batched chunk state
# ---------------------------------------------------------------------------------------------------------------------
class PoolSchedule:
    """The host-side plan of a pool, without device work: which slots hold a video, how many frames (encoder) or latent
    frames (decoder) each has buffered, and where each chunk runs.  Chunks are (frames in, frames consumed, decoded frames
    dropped at the tail) as recipe_decode_chunks; an encoder chunk is (n, n, 0).

    A video's chunks are those of the recipe stream run alone: its first chunk (one frame, or one latent plus its look-ahead)
    "joins" on a side state, later chunks of exactly t_chunk (+ look-ahead) run batched, and close() gives the rest -- the
    short last chunk, or the decoder's last chunk without look-ahead -- which runs on the side state again.  For v1.1 these
    are the chunks of build_chunk_start_end; for v1.0 they are valid stream chunks (1 frame, then multiples of tdf), which
    give the whole clip's result."""

    def __init__(self, capacity: int, version: int, tdf: int, t_chunk: int, is_decoder: bool, use_overlap: bool = False):
        if int(capacity) < 1:
            raise ValueError(f"capacity must be positive, got {capacity}")
        self.S, self.version, self.tdf, self.t_chunk = int(capacity), int(version), int(tdf), int(t_chunk)
        self.is_decoder, self.use_overlap = bool(is_decoder), bool(use_overlap)
        self.busy = [False] * self.S     # the slot holds a video
        self.avail = [0] * self.S        # frames buffered and not yet consumed
        self.first = [True] * self.S     # the video's first chunk has not run

    def _chunks(self, slot: int, final: bool) -> List[Tuple[int, int, int]]:
        if self.is_decoder:
            return recipe_decode_chunks(self.avail[slot], self.first[slot], self.t_chunk, self.use_overlap, self.tdf, final)
        return [(n, n, 0) for n in recipe_encode_chunks(self.avail[slot], self.first[slot], self.t_chunk, final)]

    def check(self, slot: int):
        if not (0 <= slot < self.S) or not self.busy[slot]:
            raise RuntimeError(f"slot {slot} holds no open video")

    def open(self) -> int:
        for s in range(self.S):
            if not self.busy[s]:
                self.busy[s], self.avail[s], self.first[s] = True, 0, True
                return s
        raise RuntimeError(f"all {self.S} slots hold a video: close one first")

    def push(self, slot: int, n: int):
        self.check(slot)
        self.avail[slot] += int(n)

    def started(self) -> List[int]:
        """slots whose video has run its first chunk: their caches must survive every batched chunk"""
        return [s for s in range(self.S) if self.busy[s] and not self.first[s]]

    def plan_step(self) -> Tuple[List[Tuple[int, Tuple[int, int, int]]], List[int], Optional[Tuple[int, int, int]]]:
        """(joins, ready, chunk): the first chunks to run on the side state, in slot order; the slots of the batched chunk
        and its (frames in, consumed, dropped), the same for every ready slot (None when no slot is ready)."""
        joins = []
        for s in range(self.S):
            if self.busy[s] and self.first[s]:
                c = self._chunks(s, final=False)
                if c:
                    joins.append((s, c[0]))
                    self.avail[s] -= c[0][1]
                    self.first[s] = False
        ready, chunk = [], None
        for s in self.started():
            c = self._chunks(s, final=False)
            if c:
                ready.append(s)
                chunk = c[0]
        for s in ready:
            self.avail[s] -= chunk[1]
        return joins, ready, chunk

    def close(self, slot: int) -> Tuple[bool, List[Tuple[int, int, int]]]:
        """(started, chunks): the chunks that finish the video (all buffered frames), and whether its first chunk ran
        before (its caches are then in the slot).  Frees the slot."""
        self.check(slot)
        started, chunks = not self.first[slot], self._chunks(slot, final=True)
        if not self.is_decoder and self.version == 0:
            for i, (n, _, _) in enumerate(chunks):
                if (started or i > 0) and n % self.tdf:
                    raise ValueError(f"{n % self.tdf} frames do not complete a group of {self.tdf}: a v1.0 pool encodes "
                                     f"videos of 1 + k * {self.tdf} frames")
        self.busy[slot], self.avail[slot], self.first[slot] = False, 0, True
        return started, chunks


class _Pool(_Chunked):
    def __init__(self, model, capacity: int, H: int, W: int, is_decoder: bool, t_chunk: Optional[int],
                 use_overlap: bool = False):
        super().__init__(model, H, W, is_decoder, t_chunk, use_overlap, check_pool_recipe)
        self.sched = PoolSchedule(capacity, self.spec.version, self.tdf, self.t_chunk, is_decoder, self.use_overlap)
        self.S = self.sched.S
        self.main = ChunkState(self.native, self.precision, self.S, self.H, self.W, is_decoder, self.use_overlap)
        self.side = ChunkState(self.native, self.precision, 1, self.H, self.W, is_decoder, self.use_overlap)
        self.park: Optional[ChunkState] = None   # holds the caches of started slots that sit out a batched chunk
        self.pending: List[Optional[torch.Tensor]] = [None] * self.S
        # batched: batched chunks run; slot_chunks: video chunks they carried; side: chunks on the side state;
        # transplants: slots copied between states
        self.counts = {"batched": 0, "slot_chunks": 0, "side": 0, "transplants": 0}

    def close_pool(self):
        for st in (self.main, self.side, self.park):
            if st is not None:
                st.close()

    def _copy(self, dst: ChunkState, src: ChunkState, dst_slots: List[int], src_slots: List[int]):
        dst.copy_slots(src, dst_slots, src_slots)
        self.counts["transplants"] += len(dst_slots)

    def _open(self) -> int:
        slot = self.sched.open()
        self.pending[slot] = None
        return slot

    def _buffer(self, slot: int, t: torch.Tensor):
        self.sched.push(slot, t.shape[2])
        self.pending[slot] = t if self.pending[slot] is None else torch.cat([self.pending[slot], t], dim=2)

    def _take(self, slot: int, chunk: Tuple[int, int, int]) -> torch.Tensor:
        n, step, _ = chunk
        p = self.pending[slot]
        out = p[:, :, :n].contiguous()
        self.pending[slot] = p[:, :, step:] if step < p.shape[2] else None
        return out

    def _batched(self, ready: List[int], chunk: Tuple[int, int, int], run):
        """run(x_rows) over the main state, every other started slot parked (copied out before and back after, so its
        caches are exactly as they were) and every other row fed zeros; x_rows: {slot: its chunk}"""
        rows = {s: self._take(s, chunk) for s in ready}
        waiting = [s for s in self.sched.started() if s not in rows]
        if waiting:
            if self.park is None:
                self.park = ChunkState(self.native, self.precision, self.S, self.H, self.W, self.sched.is_decoder,
                                       self.use_overlap)
            self._copy(self.park, self.main, waiting, waiting)
        out = run(rows)
        if waiting:
            self._copy(self.main, self.park, waiting, waiting)
        self.counts["batched"] += 1
        self.counts["slot_chunks"] += len(ready)
        return out

    @staticmethod
    def _stack(rows: Dict[int, torch.Tensor], S: int) -> torch.Tensor:
        any_row = next(iter(rows.values()))
        x = torch.zeros((S,) + tuple(any_row.shape[1:]), dtype=any_row.dtype, device=any_row.device)
        for s, r in rows.items():
            x[s] = r[0]
        return x


class EncodePool(_Pool):
    """S slots of one encoder, one (H, W).  Each slot holds one video at a time; videos open, push frames and close
    independently, and each video's outputs equal its own tile_encode (v1.1, t_chunk = t_chunk_enc) or its whole-clip
    encode (v1.0) -- see the module docstring of the pools.

        pool = EncodePool(model, capacity=S, H=H, W=W, t_chunk=16)
        a = pool.open(); pool.push(a, frames)          # frames [1, C, t, H, W], any t
        for slot, (z, reg_log) in pool.step().items(): ...
        z, reg_log = pool.close(a)                      # the rest of the video, its short last chunk included

    generator (open): the CPU generator of the video's KL noise (one torch.randn per chunk, in chunk order, as
    tile_encode draws them); None draws from torch's default generator in the order the pool runs the chunks."""

    def __init__(self, model, capacity: int, H: int, W: int, t_chunk: Optional[int] = None):
        super().__init__(model, capacity, H, W, is_decoder=False, t_chunk=t_chunk)
        self.Hz, self.Wz = self.native.latent_shape(1, H, W)[1:]
        self.reg = model.regularization
        self.aux = self.spec.regularizer == "fsq" and self.reg.aux_enabled()
        self.losses: List[Optional[_Losses]] = [None] * self.S
        self.gens: List[Optional[torch.Generator]] = [None] * self.S

    def open(self, generator: Optional[torch.Generator] = None) -> int:
        slot = self._open()
        self.losses[slot] = _Losses(self.model, self.native.device, self.aux)
        self.gens[slot] = generator
        return slot

    def push(self, slot: int, frames: torch.Tensor):
        """frames: [1, C, t, H, W] CUDA tensor, any t (buffered until they complete a chunk)."""
        self.sched.check(slot)
        self._buffer(slot, self._frames(frames, 1))

    def step(self) -> Dict[int, Tuple[torch.Tensor, Dict[str, torch.Tensor]]]:
        """Runs every first chunk that is buffered (side state, then transplanted into its slot) and one batched chunk of
        every slot with t_chunk frames buffered.  Returns {slot: (z, reg_log)} for the slots that produced latents."""
        _refuse_capture("EncodePool.step (slot transplants upload host tables; KL noise comes from the CPU generator)")
        joins, ready, chunk = self.sched.plan_step()
        parts: Dict[int, List] = {}
        for s, c in joins:
            got = self._run(self.side, {0: self._take(s, c)}, {0: s}, first=True)
            self.counts["side"] += 1
            self._copy(self.main, self.side, [s], [0])
            parts.setdefault(s, []).append(got[0])
        if ready:
            got = self._batched(ready, chunk, lambda rows: self._run(self.main, rows, {s: s for s in rows}, first=False))
            for s in ready:
                parts.setdefault(s, []).append(got[s])
        return {s: self._result(s, p) for s, p in parts.items()}

    def close(self, slot: int) -> Tuple[torch.Tensor, Dict[str, torch.Tensor]]:
        """End of the slot's video: encodes the frames still buffered (v1.1: the last, shorter chunk) on the side state
        and frees the slot.  Returns the latents of those chunks and the video's reg_log (its final losses)."""
        started, chunks = self.sched.close(slot)
        if started and chunks:
            self._copy(self.side, self.main, [0], [slot])
        parts = []
        for i, c in enumerate(chunks):
            parts.append(self._run(self.side, {0: self._take(slot, c)}, {0: slot}, first=not started and i == 0)[0])
            self.counts["side"] += 1
        self.pending[slot] = None
        out = self._result(slot, parts)
        self.losses[slot], self.gens[slot] = None, None
        return out

    def _result(self, slot: int, parts: List) -> Tuple[torch.Tensor, Dict[str, torch.Tensor]]:
        s, dev = self.spec, self.native.device
        if parts:
            z = torch.cat([p[0] for p in parts], dim=2) if len(parts) > 1 else parts[0][0]
        else:
            z = torch.empty((1, s.z_channels, 0, self.Hz, self.Wz), dtype=torch.float32, device=dev)
        L = self.losses[slot]
        if s.regularizer == "fsq":
            if parts:
                idx = torch.cat([p[1] for p in parts], dim=1) if len(parts) > 1 else parts[0][1]
            else:
                idx = torch.empty((1, 0, self.Hz, self.Wz), dtype=torch.int32, device=dev)
            log = {"indices": idx, "aux_loss": L.aux_loss()}
        else:
            log = {"kl_loss": L.kl_loss()}
        return z.to(self.out_dtype), log

    def _run(self, state: ChunkState, rows: Dict[int, torch.Tensor], slot_of: Dict[int, int], first: bool) -> Dict[int, Tuple]:
        """One chunk of `state` over rows {batch row: frames [1,C,n,H,W]} (other rows zeros); per row (z, indices), and
        the row's video's losses updated from its own slice of the pre-bound latent."""
        s, dev = self.spec, self.native.device
        B = self.S if state is self.main else 1
        n = next(iter(rows.values())).shape[2]
        tz = self.native.latent_shape(n, self.H, self.W)[0]
        x = self._stack(rows, B)
        noise = None
        if s.regularizer == "kl" and s.kl_sample:
            noise = torch.zeros((B, s.z_channels, tz, self.Hz, self.Wz), dtype=torch.float32)
            for r in rows:   # row by row, each with its video's generator
                noise[r] = chunk_noise(1, s.z_channels, [tz], self.Hz, self.Wz, self.gens[slot_of[r]])[0]
            noise = noise.to(dev)
        b = state.encode(x, first, noise, want_h=True)
        out = {}
        for r in rows:
            L, h = self.losses[slot_of[r]], b["h"][r:r + 1]
            if s.regularizer == "kl":
                L.add(kl=_loss_terms(self.native, self.reg, h))
            elif self.aux:
                L.add(partials=_loss_terms(self.native, self.reg, h), tokens=tz * self.Hz * self.Wz)
            out[r] = (b["z"][r:r + 1], b["idx"][r:r + 1] if b["idx"] is not None else None)
        return out


class DecodePool(_Pool):
    """S slots of one decoder, one latent (Hz, Wz): the decoding counterpart of EncodePool.  Each video's decoded frames
    equal its own tile_decode (v1.1, t_chunk = t_chunk_dec, the same use_overlap) or its whole-clip decode (v1.0).

        pool = DecodePool(model, capacity=S, Hz=Hz, Wz=Wz, t_chunk=4, use_overlap=True)
        a = pool.open(); pool.push(a, z)                # z [1, z_channels, tz, Hz, Wz], or FSQ indices [1, tz, Hz, Wz]
        for slot, frames in pool.step().items(): ...
        frames = pool.close(a)                          # the last chunk, without look-ahead"""

    def __init__(self, model, capacity: int, Hz: int, Wz: int, t_chunk: Optional[int] = None, use_overlap: bool = False):
        super().__init__(model, capacity, Hz, Wz, is_decoder=True, t_chunk=t_chunk, use_overlap=use_overlap)
        self.f = self.native.spatial_factor()

    def open(self) -> int:
        return self._open()

    def push(self, slot: int, z: torch.Tensor):
        self.sched.check(slot)
        self._buffer(slot, self._latents(z, 1))

    def step(self) -> Dict[int, torch.Tensor]:
        """Runs every first chunk that is buffered (side state, then transplanted into its slot) and one batched chunk of
        every slot with a full chunk (and its look-ahead) buffered.  Returns {slot: decoded frames} of the slots that
        produced frames."""
        _refuse_capture("DecodePool.step (slot transplants upload host tables)")
        joins, ready, chunk = self.sched.plan_step()
        parts: Dict[int, List[torch.Tensor]] = {}
        for s, c in joins:
            parts.setdefault(s, []).append(self._run(self.side, {0: self._take(s, c)}, c, first=True)[0])
            self.counts["side"] += 1
            self._copy(self.main, self.side, [s], [0])
        if ready:
            got = self._batched(ready, chunk, lambda rows: self._run(self.main, rows, chunk, first=False))
            for s in ready:
                parts.setdefault(s, []).append(got[s])
        return {s: self._cat(p) for s, p in parts.items()}

    def close(self, slot: int) -> torch.Tensor:
        """End of the slot's video: decodes the latents still buffered on the side state (the last chunk without
        look-ahead) and frees the slot."""
        started, chunks = self.sched.close(slot)
        if started and chunks:
            self._copy(self.side, self.main, [0], [slot])
        parts = []
        for i, c in enumerate(chunks):
            parts.append(self._run(self.side, {0: self._take(slot, c)}, c, first=not started and i == 0)[0])
            self.counts["side"] += 1
        self.pending[slot] = None
        return self._cat(parts)

    def _cat(self, parts: List[torch.Tensor]) -> torch.Tensor:
        if not parts:
            return torch.empty((1, self.spec.out_ch, 0, self.H * self.f, self.W * self.f), dtype=self.out_dtype,
                               device=self.native.device)
        x = parts[0].contiguous() if len(parts) == 1 else torch.cat(parts, dim=2)
        return x.to(self.out_dtype)

    def _run(self, state: ChunkState, rows: Dict[int, torch.Tensor], chunk: Tuple[int, int, int], first: bool) -> Dict[int, torch.Tensor]:
        B = self.S if state is self.main else 1
        trim = chunk[2]
        out = state.decode(self._stack(rows, B), first)
        To = out.shape[2]
        return {r: out[r:r + 1, :, :To - trim] if trim else out[r:r + 1] for r in rows}
