"""One long video as S shards that run side by side as one batch, with outputs bit-identical to tile_encode / tile_decode.

    z, reg_log = encode_sharded(model, x, shards=4)       # == model.tile_encode(x)[0]
    y = decode_sharded(model, z, shards=4)                 # == model.tile_decode(z) (model.use_overlap as set)

Why it is exact: under the tile_encode / tile_decode chunking an output frame of a causal v1.1 model depends on no input more
than R frames before it (`temporal_reach`, vt_temporal_reach: composed from the executor's layer list).  A shard starts a
fresh chunk state on the global chunk grid (a frame s = m * t_chunk, so that its chunks after the first frame are global
chunks), runs at least R frames (encoder) or latent frames (decoder) of warm-up after that first frame, and keeps only the
chunks it owns.  Those chunks see the same inputs, at the same chunk geometry, through the same kernels as in the sequential
run, and a chunk's result does not depend on the other samples of the batch.  Nothing is blended at the seams.

The S windows have one length, so they run as one batched stream (EncodeStream / DecodeStream with t_chunk) of batch S
(in "exact" and "mixed" one window after another: the split-operand kernels' rounding can depend on the batch).  The
last window ends at the end of the video and is flushed, so its last chunk is the true last chunk; the other windows lie
inside the video, and their chunks that do not match the sequential run (their last chunk, which runs short or without
look-ahead) are computed and dropped.  The windows start (S-1) * step chunks apart; shard 0 owns its warm-up span too, and
the last shard owns what `step` leaves over, so the owned chunks partition the video.

The cost is the warm-up: every window computes `plan.window` frames against the video's T, plan.warmup_fraction of the work.
R is large for the shipped models (e.g. 109 input frames / 46 latent frames for 4x-time 4-level models), so sharding pays
only for videos many times R long.

Losses: the batched chunk state would reduce them over all shards, so each owned chunk's loss terms are formed from its own
pre-bound latent (EncodeStream(keep_pre_bound=True)): the KL loss per chunk (vt_op_kl), then their mean in chunk order as
tile_encode forms it (to fp32 rounding: both sum with double atomics); the FSQ aux partials per chunk
(FSQRegularizer.aux_partials), finalized in global chunk order, bit-identical.  KL noise (kl_sample) is drawn exactly as
tile_encode draws it (one CPU torch.randn per global chunk, in chunk order, so every rank must share the CPU generator's
state) and sliced to the owned chunks.

Ranks: with torch.distributed initialised (world size > 1) the call treats the whole group as working on one video: each
rank runs a contiguous range of the shards on its device, with no collective on the data path.  encode_sharded then
all-reduces the zero-filled latents, indices and per-chunk loss terms so that every rank holds tile_encode's full result;
decode_sharded does not gather frames: each rank gets its owned frames and their global range.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import List, Optional, Tuple

import torch

from . import _native as N
from .engine import chunk_noise, chunk_start_end
from .streaming import DecodeStream, EncodeStream, _loss_terms, _mean


def temporal_reach(native, is_decoder: bool, use_overlap: bool = False) -> int:
    """vt_temporal_reach of a NativeModel: encoder in input frames, decoder in latent frames."""
    r = C.c_int32()
    N.check(native.lib.vt_temporal_reach(native.handle, int(is_decoder), int(use_overlap), C.byref(r)))
    return r.value


@dataclass
class ShardPlan:
    """Shards of one video on the global chunk grid (frames for the encoder, latent frames for the decoder).
    starts[i]: the first frame of shard i's window (a fresh first chunk); every window is `window` long.
    owned[i]: (first, last + 1) global chunk indices shard i keeps; keep[i]: (a, b) the frames of its window those chunks
    cover.  warmup[i]: frames of shard i's window before its first owned frame."""
    T: int
    t_chunk: int
    reach: int
    chunks: List[Tuple[int, int]]
    starts: List[int]
    window: int
    owned: List[Tuple[int, int]]
    keep: List[Tuple[int, int]]
    warmup: List[int]

    @property
    def warmup_fraction(self) -> float:
        """share of the computed frames that no shard keeps"""
        total = len(self.starts) * self.window
        return (total - self.T) / total


def shard_plan(T: int, shards: int, t_chunk: int, reach: int, lookahead: bool = False) -> ShardPlan:
    """Pure host arithmetic.  T: frames (encoder) or latent frames (decoder); t_chunk: t_chunk_enc / t_chunk_dec; reach:
    temporal_reach; lookahead: a decoder with use_overlap (a window's last chunk runs without look-ahead, so it is not kept).
    A window counts the frame it starts on as warm-up: its first chunk treats that frame as a video's first."""
    S, c = int(shards), int(t_chunk)
    if S < 1 or c < 1 or T < 1:
        raise ValueError("shards, t_chunk and T must be positive")
    chunks = chunk_start_end(T, c)
    n = len(chunks) - 1                      # global chunks after the first frame
    warm = -(-int(reach) // c)               # full chunks of warm-up after a window's first frame
    short = chunks[-1][1] - chunks[-1][0] < c if n else False
    drop = 1 if (lookahead or short) else 0  # a non-final window's last chunk does not match the sequential run
    step = (n - warm - drop) // S if S > 1 else n
    if S > 1 and step < 1:
        raise ValueError(f"{S} shards need at least {S + warm + drop} chunks of {c} after the first frame "
                         f"(temporal reach {reach}: {warm} chunks of warm-up per shard); this video has {n}")
    starts = [i * step * c for i in range(S)]
    window = T - starts[-1]
    first = [0] + [i * step + 1 + warm for i in range(1, S)]
    owned = [(first[i], first[i + 1] if i + 1 < S else len(chunks)) for i in range(S)]
    keep = [(chunks[a][0] - starts[i], chunks[b - 1][1] - starts[i]) for i, (a, b) in enumerate(owned)]
    return ShardPlan(T, c, int(reach), chunks, starts, window, owned, keep, [k[0] for k in keep])


def _check_model(model):
    if not getattr(model, "is_causal", False):
        raise ValueError("non-causal models cannot be sharded: their time padding is symmetric, so a frame depends on later frames")
    if model.spec.version != 1:
        raise ValueError("sharding needs a v1.1 model: v1.0 models run whole clips only")


def _group():
    """(rank, world size) of an initialised torch.distributed group, else (0, 1)"""
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


def rank_shards(S: int, rank: int, world: int) -> Tuple[int, int]:
    """the contiguous range of shards rank `rank` of `world` runs"""
    if S < world:
        raise ValueError(f"{S} shards cannot occupy {world} ranks")
    return S * rank // world, S * (rank + 1) // world


def _batches(model, S: int) -> List[List[int]]:
    """The windows one chunk state runs: all S as one batch, but one at a time in the split-operand modes ("exact", and
    "mixed"'s encoder), whose tensor-core tiles can group a tile's K steps differently when the batch changes, so that a
    window's bits would depend on the others."""
    if model._rt.precision() in (N.PREC_EXACT_TC, N.PREC_MIXED):
        return [[i] for i in range(S)]
    return [list(range(S))]


class _Stager:
    """Stages the windows' frames [a, e) to the device: through two pinned buffers for a host video (the copy of one chunk
    overlaps the previous chunk's kernels), directly for a CUDA video."""

    def __init__(self, x: torch.Tensor, starts: List[int], dev):
        self.x, self.starts, self.dev = x, starts, dev
        self.host = not x.is_cuda
        self.bufs, self.events, self.k = {}, [None, None], 0

    def __call__(self, a: int, e: int) -> torch.Tensor:
        x = self.x
        if not self.host:
            return torch.stack([x[0, :, p + a:p + e] for p in self.starts]).float()
        k = self.k & 1
        self.k += 1
        if self.events[k] is not None:
            self.events[k].synchronize()            # the copy that last read this buffer has finished
        shape = (len(self.starts), x.shape[1], e - a, x.shape[3], x.shape[4])
        buf = self.bufs.get((k, shape))
        if buf is None:
            buf = self.bufs[(k, shape)] = torch.empty(shape, dtype=torch.float32).pin_memory()
        torch.stack([x[0, :, p + a:p + e] for p in self.starts], out=buf)
        out = buf.to(self.dev, non_blocking=True)
        self.events[k] = torch.cuda.Event()
        self.events[k].record()
        return out


def encode_sharded(model, x: torch.Tensor, shards: int):
    """model.tile_encode(x) of a causal v1.1 model as `shards` windows in one batch: latents, FSQ indices and FSQ aux_loss
    bit-identical to tile_encode's with t_chunk_enc = model.t_chunk_enc, kl_loss to fp32 rounding.  x: [1,C,T,H,W], CUDA
    or (pinned) host memory; the windows are staged to the device chunk by chunk.  Returns (z, reg_log) as tile_encode
    (fp32 z, whatever the autocast state).  Across ranks every rank gets the full result (see the module docstring)."""
    _check_model(model)
    if x.dim() != 5 or x.shape[0] != 1:
        raise ValueError("expected one video [1,C,T,H,W]")
    nat = model._rt.sync()
    dev, s, reg = nat.device, model.spec, model.regularization
    _, Cin, T, H, W = x.shape
    c, tdf = int(model.t_chunk_enc), s.time_downsample_factor
    plan = shard_plan(T, shards, c, temporal_reach(nat, False))
    rank, world = _group()
    lo, hi = rank_shards(len(plan.starts), rank, world)
    starts, owned = plan.starts[lo:hi], plan.owned[lo:hi]
    S, G = len(starts), len(plan.chunks)
    tz = [nat.latent_shape(e - a, H, W)[0] for a, e in plan.chunks]
    _, Hz, Wz = nat.latent_shape(1, H, W)
    lat0 = [sum(tz[:g]) for g in range(G + 1)]                 # first latent frame of each global chunk
    Tz = lat0[-1]
    kl_noise = s.regularizer == "kl" and s.kl_sample
    if kl_noise:
        draws = chunk_noise(1, s.z_channels, tz, Hz, Wz)   # every global chunk's, as tile_encode draws them
    row = [(a, e, nat.latent_shape(e - a, H, W)[0]) for a, e in chunk_start_end(plan.window, c)]   # a window's chunks
    zlen = sum(t for _, _, t in row)
    row0 = [p // tdf for p in starts]                          # global latent frame of each window's first latent
    noise = None
    if kl_noise:
        noise = torch.zeros((S, s.z_channels, zlen, Hz, Wz))   # warm-up latents are discarded: no draws for them
        for i, (a, b) in enumerate(owned):
            noise[i, :, lat0[a] - row0[i]:lat0[b] - row0[i]] = draws[0, :, lat0[a]:lat0[b]]
    zs, idxs, hs = [], [], []
    for grp in _batches(model, S):   # windows that share one chunk state
        rz, ri, rh = [], [], []
        enc = EncodeStream(model, batch=len(grp), H=H, W=W, t_chunk=c, keep_pre_bound=True)
        enc.out_dtype = torch.float32                          # tile_encode's latents are fp32 under autocast too
        stage, zt = _Stager(x, [starts[i] for i in grp], dev), 0
        try:
            # a short last chunk waits in the stream for flush()
            for k, (a, e, t) in enumerate(row):
                last_short = k == len(row) - 1 and k > 0 and e - a < c
                z, log = enc.push(stage(a, e), None if not kl_noise or last_short else noise[grp, :, zt:zt + t])
                rz.append(z), ri.append(log.get("indices")), rh.append(log["h_pre"])
                zt += z.shape[2]
            z, log = enc.flush(noise[grp, :, zt:] if kl_noise else None)
            rz.append(z), ri.append(log.get("indices")), rh.append(log["h_pre"])
        finally:
            enc.close()
        zs.append(torch.cat(rz, dim=2)), hs.append(torch.cat(rh, dim=2))
        if s.regularizer == "fsq":
            idxs.append(torch.cat(ri, dim=1))
    zr, hr = torch.cat(zs), torch.cat(hs)
    ir = torch.cat(idxs) if s.regularizer == "fsq" else None
    out = torch.zeros((1, s.z_channels, Tz, Hz, Wz), dtype=torch.float32, device=dev)
    idx = torch.zeros((1, Tz, Hz, Wz), dtype=torch.int32, device=dev) if ir is not None else None
    aux = s.regularizer == "fsq" and reg.aux_enabled()
    kls = torch.zeros((G,), dtype=torch.float32, device=dev)
    stats = torch.zeros((G, 2), dtype=torch.float32, device=dev) if aux else None
    avg = torch.zeros((G, reg.codebook_size), dtype=torch.float32, device=dev) if aux else None
    for i, (a, b) in enumerate(owned):
        r0, r1 = lat0[a] - row0[i], lat0[b] - row0[i]
        out[0, :, lat0[a]:lat0[b]] = zr[i, :, r0:r1]
        if idx is not None:
            idx[0, lat0[a]:lat0[b]] = ir[i, r0:r1]
        for g in range(a, b):   # each owned chunk's loss terms, from its own pre-bound latent
            h = hr[i:i + 1, :, lat0[g] - row0[i]:lat0[g + 1] - row0[i]].contiguous()
            if s.regularizer == "kl":
                _loss_terms(nat, reg, h, kls[g:g + 1])
            elif aux:
                st, av = _loss_terms(nat, reg, h)
                stats[g], avg[g] = st[0], av[0]
    if world > 1:
        import torch.distributed as dist
        for t in [out, idx, kls, stats, avg]:
            if t is not None:
                dist.all_reduce(t)   # every entry has exactly one owner; the others add zeros
    if s.regularizer == "kl":
        total = torch.zeros((), dtype=torch.float32, device=dev)
        for g in range(G):
            total = total + kls[g]   # in chunk order, as tile_encode's mean sums them
        return out, {"kl_loss": _mean(total, G)}
    aux_loss = (reg.aux_finalize(stats, avg, n_steps=model.global_step // 2, world_size=1) if aux
                else torch.zeros((), device=dev))
    return out, {"aux_loss": aux_loss, "indices": idx}


def decode_sharded(model, z: torch.Tensor, shards: int, out: Optional[torch.Tensor] = None):
    """model.tile_decode(z) of a causal v1.1 model (t_chunk_dec, use_overlap as set on the model) as `shards` windows in
    one batch: the decoded frames are bit-identical (fp32, whatever the autocast state).  z: CUDA [1,z_channels,Tz,Hz,Wz].
    Windows are decoded chunk by chunk and each chunk's owned frames are copied into `out` (optional: a contiguous fp32
    tensor, CUDA or pinned host memory, of the shape returned).  One process: returns the [1,C,Tz*tdf,H,W] video.  Across
    ranks: returns (frames, (g0, g1)), this rank's owned frames [1,C,g1-g0,H,W], frames g0 .. g1-1 of the video."""
    _check_model(model)
    if z.dim() != 5 or z.shape[0] != 1 or z.shape[1] != model.spec.z_channels:
        raise ValueError(f"expected one latent [1,{model.spec.z_channels},Tz,Hz,Wz], got {tuple(z.shape)}")
    nat = model._rt.sync()
    _, _, Tz, Hz, Wz = z.shape
    ov, tdf, cd = bool(model.use_overlap), model.spec.time_downsample_factor, int(model.t_chunk_dec)
    plan = shard_plan(Tz, shards, cd, temporal_reach(nat, True, ov), lookahead=ov)
    rank, world = _group()
    lo, hi = rank_shards(len(plan.starts), rank, world)
    starts, keep = plan.starts[lo:hi], plan.keep[lo:hi]
    g0, g1 = tdf * (starts[0] + keep[0][0]), tdf * (starts[-1] + keep[-1][1])
    f = nat.spatial_factor()
    shape = (1, model.spec.out_ch, g1 - g0, Hz * f, Wz * f)
    if out is None:
        out = torch.empty(shape, dtype=torch.float32, device=z.device)
    elif tuple(out.shape) != shape or out.dtype != torch.float32 or not out.is_contiguous():
        raise ValueError(f"out must be a contiguous fp32 tensor of shape {shape}")
    for grp in _batches(model, len(starts)):   # windows that share one chunk state
        dec = DecodeStream(model, batch=len(grp), Hz=Hz, Wz=Wz, t_chunk=cd, use_overlap=ov)
        dec.out_dtype = torch.float32
        done = 0   # decoded frames of each window so far: frame k of window i is frame tdf * starts[i] + k of the video

        def take(y):
            nonlocal done
            for r, i in enumerate(grp):
                a, b = keep[i]
                u, v = max(tdf * a, done), min(tdf * b, done + y.shape[2])
                if u < v:
                    g = tdf * starts[i] + u - g0
                    out[0, :, g:g + v - u].copy_(y[r, :, u - done:v - done], non_blocking=True)
            done += y.shape[2]

        try:
            for a, e in chunk_start_end(plan.window, cd):
                take(dec.push(torch.stack([z[0, :, starts[i] + a:starts[i] + e] for i in grp])))
            take(dec.flush())
        finally:
            dec.close()
    if not out.is_cuda:
        torch.cuda.current_stream(z.device).synchronize()
    return out if world == 1 else (out, (g0, g1))
