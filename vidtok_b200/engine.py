"""Host-side mirror of the reference's Python surface for the tokenizer hot path.

Same class names, constructor kwargs, attributes, state-dict keys and return conventions as
  vidtok/models/autoencoder.py:98-229            (AutoencodingEngine, v1.0)
  vidtok/models/autoencoder_v1_1.py:98-342       (AutoencodingEngine with temporal tiling, v1.1)
  vidtok/modules/model_3dcausal[_v1_1].py        (EncoderCausal3DPadding / DecoderCausal3DPadding)
  vidtok/modules/regularizers.py:74-268          (DiagonalGaussianRegularizer / FSQRegularizer)
but every tensor operation runs in libvidtok_b200.so (hand-written sm_90a kernels) through the C ABI of
include/vidtok_b200.h.  There is no PyTorch/CPU fallback: a model that is not on a CUDA device raises.

Precision: the reference scripts run fp32 by default and bf16/fp16 under `--precision autocast`
(scripts/inference_evaluate.py:77-79,137).  Mirroring that, `model.precision = None` (default) selects
  * "exact"  -- fp32-class results on the tensor cores (wgmma) (fp16 hi|lo split operands x 3 MMAs, fp32 LayerNorm/SiLU): the
                parity mode (1e-3 max-abs, FSQ codes equal), unless
  * "bf16"   -- torch.autocast is active (bf16 activations/weights on wgmma, fp32 accumulate: the throughput mode;
                outputs are returned in the autocast dtype like the reference's; an fp16 autocast region also
                computes in bf16).
Explicit settings: "exact", "bf16", "mixed" (encoder exact, decoder bf16: bit-exact FSQ codes / 1e-3 latents with a
bf16 decoder) and "fma" (fp32 FMA kernels without tensor cores, kept as a cross-check).

Threading / streams: one workspace per model handle -- calls on one model must be issued on one CUDA stream at a time
(the reference's modules are not re-entrant either: v1.1 keeps chunk caches on the modules).
"""
from __future__ import annotations

import ctypes as C
import math
import re
import weakref
from dataclasses import dataclass, field
from typing import Any, Dict, List, Optional, Sequence, Tuple

import torch
import torch.nn as nn

from . import _native as N


# --------------------------------------------------------------------------------------------------
# configuration
# --------------------------------------------------------------------------------------------------
@dataclass
class TokenizerSpec:
    version: int = 0
    ch: int = 128
    ch_mult: Tuple[int, ...] = (1, 2, 4, 8)
    num_res_blocks: int = 2
    in_channels: int = 3
    out_ch: int = 3
    z_channels: int = 4
    double_z: bool = True
    norm_type: str = "groupnorm"
    time_downsample_factor: int = 4
    spatial_ds: Optional[Sequence[int]] = None
    tempo_ds: Optional[Sequence[int]] = None
    spatial_us: Optional[Sequence[int]] = None
    tempo_us: Optional[Sequence[int]] = None
    interpolation_mode: str = "nearest"
    regularizer: str = "kl"
    fsq_levels: Tuple[int, ...] = ()
    kl_sample: bool = True
    causal: bool = True   # False: the non-causal family (vidtok/modules/model_3dnoncausal.py)

    @staticmethod
    def from_params(params: Dict[str, Any], version: int, causal: bool = True) -> "TokenizerSpec":
        g = params.get
        if not causal:   # model_3dnoncausal.py:335,515: fixed resampling schedules
            params = {k: v for k, v in params.items() if k not in ("spatial_ds", "tempo_ds", "spatial_us", "tempo_us")}
            g = params.get
        return TokenizerSpec(
            causal=causal,
            version=version, ch=int(params["ch"]), ch_mult=tuple(int(c) for c in g("ch_mult", (1, 2, 4, 8))),
            num_res_blocks=int(params["num_res_blocks"]), in_channels=int(params["in_channels"]),
            out_ch=int(params["out_ch"]), z_channels=int(params["z_channels"]), double_z=bool(g("double_z", True)),
            norm_type=str(g("norm_type", "groupnorm")), time_downsample_factor=int(g("time_downsample_factor", 4)),
            spatial_ds=g("spatial_ds"), tempo_ds=g("tempo_ds"), spatial_us=g("spatial_us"), tempo_us=g("tempo_us"),
            interpolation_mode=str(g("interpolation_mode", "nearest")),
        )

    def to_desc(self) -> N.ModelDesc:
        d = N.ModelDesc()
        d.version = self.version
        d.ch = self.ch
        d.num_levels = len(self.ch_mult)
        for i, c in enumerate(self.ch_mult):
            d.ch_mult[i] = c
        d.num_res_blocks = self.num_res_blocks
        d.in_channels, d.out_ch, d.z_channels = self.in_channels, self.out_ch, self.z_channels
        d.double_z = int(self.double_z)
        if self.norm_type not in ("layernorm", "groupnorm"):
            raise ValueError(f"unknown norm_type {self.norm_type}")
        d.norm_type = 0 if self.norm_type == "layernorm" else 1
        d.time_downsample_factor = self.time_downsample_factor
        for name in ("spatial_ds", "tempo_ds", "spatial_us", "tempo_us"):
            v = getattr(self, name)
            if v is None:
                setattr(d, "n_" + name, -1)
            else:
                setattr(d, "n_" + name, len(v))
                arr = getattr(d, name)
                for i, x in enumerate(v):
                    arr[i] = int(x)
        d.interpolation_mode = 1 if self.interpolation_mode == "trilinear" else 0
        d.regularizer = 1 if self.regularizer == "fsq" else 0
        d.fsq_num_levels = len(self.fsq_levels)
        for i, l in enumerate(self.fsq_levels):
            d.fsq_levels[i] = int(l)
        d.kl_sample = int(self.kl_sample)
        d.noncausal = int(not self.causal)
        return d


def _capturing() -> bool:
    """The current stream is capturing a CUDA graph (torch.cuda.graph, or torch.compile's CUDA graphs)."""
    return torch.cuda.is_available() and torch.cuda.is_current_stream_capturing()


def _stream_ptr(device: torch.device) -> C.c_void_p:
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def _ptr(t: Optional[torch.Tensor]) -> C.c_void_p:
    return C.c_void_p(0 if t is None else t.data_ptr())


def _refuse_capture(what: str):
    """Calls that stage through the library's copy stream, draw CPU noise or move slots with host tables cannot be captured
    in a CUDA graph: refused before anything is enqueued, so the caller's capture stays intact."""
    if _capturing():
        raise RuntimeError(f"vidtok_b200: {what} cannot be captured in a CUDA graph (VT_ERR_CAPTURE): run it eagerly; untiled "
                           "encode / decode / forward and the steady chunks of the streams are the capturable calls")


def chunk_start_end(t: int, step: int) -> List[Tuple[int, int]]:
    """build_chunk_start_end (autoencoder_v1_1.py:218-228): [0,1], then chunks of `step`."""
    out, start, end = [(0, 1)], 1, 1
    while start < t:
        end = min(t, end + step)
        out.append((start, end))
        start = end
    return out


def chunk_noise(B: int, channels: int, tzs: Sequence[int], Hz: int, Wz: int,
                generator: Optional[torch.Generator] = None) -> torch.Tensor:
    """KL noise of consecutive chunks of tzs latent frames: one CPU torch.randn per chunk, in chunk order, concatenated
    along time -- the draws tile_encode makes, as the reference samples each chunk (distributions.py:17)."""
    draws = [torch.randn((B, channels, tz, Hz, Wz), generator=generator) for tz in tzs]
    return draws[0] if len(draws) == 1 else torch.cat(draws, dim=2)


# --------------------------------------------------------------------------------------------------
# native handle
# --------------------------------------------------------------------------------------------------
class NativeModel:
    """Owns one vt_model handle (include/vidtok_b200.h)."""

    def __init__(self, spec: TokenizerSpec, device_index: int = 0):
        self.spec = spec
        self.lib = N.lib()
        self.handle = C.c_void_p()
        desc = spec.to_desc()
        N.check(self.lib.vt_model_create(C.byref(desc), device_index, C.byref(self.handle)))
        self.device_index = device_index
        self._ws: Optional[torch.Tensor] = None
        # workspaces that a captured CUDA graph reads: kept for the model's lifetime once the workspace grows past them, so
        # that the graph never replays into memory torch has handed to someone else
        self._ws_captured = False
        self._ws_kept: List[torch.Tensor] = []
        # handles of the open chunk states: a state returns its caches to the model when destroyed, so any still open go
        # first (the garbage collector finalises a cycle holding both in no particular order)
        self._chunk_handles: Dict[int, C.c_void_p] = {}

    def __del__(self):
        try:
            for h in list(getattr(self, "_chunk_handles", {}).values()):
                if h.value:
                    self.lib.vt_chunk_state_destroy(h)
                    h.value = None
            if getattr(self, "handle", None) and self.handle.value:
                self.lib.vt_model_destroy(self.handle)
                self.handle = C.c_void_p()
        except Exception:
            pass

    def manifest(self) -> List[Tuple[str, Tuple[int, ...]]]:
        out = []
        name = C.create_string_buffer(256)
        shape = (C.c_int64 * 5)()
        ndim = C.c_int32()
        for i in range(self.lib.vt_model_num_params(self.handle)):
            N.check(self.lib.vt_model_param_info(self.handle, i, name, 256, shape, C.byref(ndim)))
            out.append((name.value.decode(), tuple(int(shape[k]) for k in range(ndim.value))))
        return out

    @property
    def device(self) -> torch.device:
        return torch.device("cuda", self.device_index)

    def load(self, name: str, t: torch.Tensor):
        t = t.detach().to(dtype=torch.float32).contiguous()
        N.check(self.lib.vt_model_load_param(self.handle, name.encode(), _ptr(t), t.numel(), int(t.is_cuda),
                                             _stream_ptr(self.device)))
        if not t.is_cuda:
            torch.cuda.current_stream(self.device).synchronize()

    def finalize(self):
        N.check(self.lib.vt_model_finalize(self.handle, _stream_ptr(self.device)))

    def latent_shape(self, T: int, H: int, W: int) -> Tuple[int, int, int]:
        a, b, c = C.c_int32(), C.c_int32(), C.c_int32()
        N.check(self.lib.vt_latent_shape(self.handle, T, H, W, C.byref(a), C.byref(b), C.byref(c)))
        return a.value, b.value, c.value

    def decoded_frames(self, Tz: int) -> int:
        return int(self.lib.vt_decoded_frames(self.handle, Tz))

    def spatial_factor(self) -> int:
        _, hz, _ = self.latent_shape(self.spec.time_downsample_factor, 1 << 10, 1 << 10)
        return (1 << 10) // hz

    def _workspace(self, nbytes: int) -> torch.Tensor:
        if nbytes < 0:
            raise RuntimeError(f"vidtok_b200: {self.lib.vt_last_error().decode()}")
        capturing = _capturing()
        if self._ws is None or self._ws.numel() < nbytes:
            if capturing:
                raise RuntimeError(f"vidtok_b200: the workspace ({0 if self._ws is None else self._ws.numel()} bytes) is smaller than the "
                                   f"{nbytes} bytes this call needs, and it cannot grow while a CUDA graph is being captured: run "
                                   "the call once eagerly with the same geometry and precision before capturing it")
            if self._ws is not None and self._ws_captured:
                self._ws_kept.append(self._ws)
            self._ws = None
            self._ws_captured = False
            self._ws = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        if capturing:
            self._ws_captured = True
        return self._ws

    def workspace_for(self, precision: int, B: int, T: int, H: int, W: int) -> torch.Tensor:
        return self._workspace(int(self.lib.vt_workspace_bytes(self.handle, precision, B, T, H, W)))

    def encode(self, x: torch.Tensor, noise: Optional[torch.Tensor], precision: int, want_h: bool = False):
        B, Cin, T, H, W = x.shape
        if Cin != self.spec.in_channels:
            raise ValueError(f"input has {Cin} channels, the model expects in_channels = {self.spec.in_channels}")
        Tz, Hz, Wz = self.latent_shape(T, H, W)
        s = self.spec
        z = torch.empty((B, s.z_channels, Tz, Hz, Wz), dtype=torch.float32, device=x.device)
        idx = torch.empty((B, Tz, Hz, Wz), dtype=torch.int32, device=x.device) if s.regularizer == "fsq" else None
        kl = torch.empty((), dtype=torch.float32, device=x.device) if s.regularizer == "kl" else None
        h = torch.empty((B, (2 if s.double_z else 1) * s.z_channels, Tz, Hz, Wz), dtype=torch.float32,
                        device=x.device) if want_h else None
        ws = self.workspace_for(precision, B, T, H, W)
        N.check(self.lib.vt_encode(self.handle, precision, _ptr(x), B, Cin, T, H, W, _ptr(noise), _ptr(z), _ptr(idx), _ptr(kl),
                                   _ptr(h), _ptr(ws), ws.numel(), _stream_ptr(x.device)))
        return z, idx, kl, h

    def decode(self, z: torch.Tensor, from_indices: bool, precision: int) -> torch.Tensor:
        if from_indices:
            if z.dim() != 4:
                raise ValueError("expected [B,T,H,W] token indices")
            B, Tz, Hz, Wz = z.shape
            Cz = self.spec.z_channels
        else:
            if z.dim() != 5:
                raise ValueError("expected a [B,C,T,H,W] latent")
            B, Cz, Tz, Hz, Wz = z.shape
            if Cz != self.spec.z_channels:
                raise ValueError(f"latent has {Cz} channels, the model expects z_channels = {self.spec.z_channels}")
        f = self.spatial_factor()
        To = self.decoded_frames(Tz)
        out = torch.empty((B, self.spec.out_ch, To, Hz * f, Wz * f), dtype=torch.float32, device=z.device)
        T_in = max(To, 1)
        ws = self.workspace_for(precision, B, T_in if self.spec.version == 0 else Tz * self.spec.time_downsample_factor,
                                Hz * f, Wz * f)
        N.check(self.lib.vt_decode(self.handle, precision, _ptr(z), int(from_indices), B, Cz, Tz, Hz, Wz, _ptr(out), _ptr(ws),
                                   ws.numel(), _stream_ptr(z.device)))
        return out


class ChunkState:
    """vt_chunk_state: per-video causal caches for v1.1 temporal tiling."""

    def __init__(self, native: NativeModel, precision: int, B: int, H: int, W: int, is_decoder: bool, use_overlap: bool):
        self.native = native
        self.handle = C.c_void_p()
        N.check(native.lib.vt_chunk_state_create(native.handle, precision, B, H, W, int(is_decoder), int(use_overlap),
                                                 C.byref(self.handle)))
        native._chunk_handles[id(self)] = self.handle
        self.B, self.H, self.W = B, H, W

    def close(self):
        self.native._chunk_handles.pop(id(self), None)
        if self.handle and self.handle.value:   # cleared when the model went first
            self.native.lib.vt_chunk_state_destroy(self.handle)
            self.handle = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def workspace(self, Tc: int, fsq_aux: bool = False) -> torch.Tensor:
        """workspace of a chunk of Tc frames (fsq_aux: of vt_encode_chunk_fsq_aux)"""
        lib = self.native.lib
        query = lib.vt_chunk_fsq_aux_workspace_bytes if fsq_aux else lib.vt_chunk_workspace_bytes
        return self.native._workspace(int(query(self.handle, Tc)))

    def encode_buffers(self, n: int, want_h: bool = False, fsq_aux: bool = False,
                       given: Optional[Dict[str, Optional[torch.Tensor]]] = None) -> Dict[str, Optional[torch.Tensor]]:
        """The outputs and workspace of one encoder chunk of n frames, those in `given` kept: z, idx (FSQ), kl (KL),
        h (want_h: the pre-bound latent) and ws, the workspace of the entry point encode() calls."""
        s, dev = self.native.spec, self.native.device
        tz, Hz, Wz = self.native.latent_shape(n, self.H, self.W)
        make = {
            "z": lambda: torch.empty((self.B, s.z_channels, tz, Hz, Wz), dtype=torch.float32, device=dev),
            "idx": lambda: torch.empty((self.B, tz, Hz, Wz), dtype=torch.int32, device=dev) if s.regularizer == "fsq" else None,
            "kl": lambda: torch.empty((1,), dtype=torch.float32, device=dev) if s.regularizer == "kl" else None,
            "h": lambda: (torch.empty((self.B, (2 if s.double_z else 1) * s.z_channels, tz, Hz, Wz), dtype=torch.float32,
                                      device=dev) if want_h else None),
            "ws": lambda: self.workspace(n, fsq_aux),
        }
        given = given or {}
        return {k: given[k] if k in given else f() for k, f in make.items()}

    def encode(self, x: torch.Tensor, first: bool, noise: Optional[torch.Tensor] = None, want_h: bool = False,
               aux: Optional[Tuple[torch.Tensor, torch.Tensor]] = None,
               out: Optional[Dict[str, Optional[torch.Tensor]]] = None) -> Dict[str, Optional[torch.Tensor]]:
        """One encoder chunk of x [B,C,n,H,W] (dense fp32): vt_encode_chunk_pre with want_h, vt_encode_chunk_fsq_aux with
        aux (the caller's stats [1,2] / avg [1,J] buffers of the chunk's FSQ aux partials), else vt_encode_chunk.  out: the
        caller's buffers, as encode_buffers names them (the graph path passes all of its static ones); the others are
        new.  Returns the buffers."""
        n, lib, s = x.shape[2], self.native.lib, self.native.spec
        b = self.encode_buffers(n, want_h, aux is not None, out)
        ws, stream = b["ws"], _stream_ptr(self.native.device)
        if want_h:
            N.check(lib.vt_encode_chunk_pre(self.handle, int(first), _ptr(x), s.in_channels, n, _ptr(noise), _ptr(b["z"]),
                                            _ptr(b["idx"]), _ptr(b["kl"]), _ptr(b["h"]), _ptr(ws), ws.numel(), stream))
        elif aux is not None:
            N.check(lib.vt_encode_chunk_fsq_aux(self.handle, int(first), _ptr(x), s.in_channels, n, _ptr(b["z"]), _ptr(b["idx"]),
                                                100.0, _ptr(aux[0]), _ptr(aux[1]), _ptr(ws), ws.numel(), stream))
        else:
            N.check(lib.vt_encode_chunk(self.handle, int(first), _ptr(x), s.in_channels, n, _ptr(noise), _ptr(b["z"]),
                                        _ptr(b["idx"]), _ptr(b["kl"]), _ptr(ws), ws.numel(), stream))
        return b

    def decode_buffers(self, n: int, first: bool) -> Dict[str, torch.Tensor]:
        """The output (every frame the chunk decodes) and workspace of one decoder chunk of n latent frames.  v1.0 drops
        tdf-1 frames of a video's first chunk only; v1.1 decodes every chunk as a video of its own."""
        s, nat = self.native.spec, self.native
        To = nat.decoded_frames(n) if (first or s.version == 1) else n * s.time_downsample_factor
        f = nat.spatial_factor()
        return {"out": torch.empty((self.B, s.out_ch, To, self.H * f, self.W * f), dtype=torch.float32, device=nat.device),
                "ws": self.workspace(n)}

    def decode(self, z: torch.Tensor, first: bool, out: Optional[Dict[str, torch.Tensor]] = None) -> torch.Tensor:
        """One decoder chunk of z [B,Cz,n,Hz,Wz] (dense fp32, the look-ahead frame included): vt_decode_chunk into
        out["out"] with workspace out["ws"] (the graph path's static buffers), or new ones.  Returns the decoded frames."""
        n, nat = z.shape[2], self.native
        b = self.decode_buffers(n, first) if out is None else out
        ws = b["ws"]
        N.check(nat.lib.vt_decode_chunk(self.handle, int(first), _ptr(z), nat.spec.z_channels, n, _ptr(b["out"]), _ptr(ws),
                                        ws.numel(), _stream_ptr(nat.device)))
        return b["out"]

    def copy_slots(self, src: "ChunkState", dst_slots: Sequence[int], src_slots: Sequence[int]):
        """vt_chunk_state_copy_slots: slot dst_slots[i] of this state becomes the state slot src_slots[i] of src would
        have had (every cache copied, in one launch on the current stream)."""
        n = len(dst_slots)
        if len(src_slots) != n:
            raise ValueError("dst_slots and src_slots must have the same length")
        d, s = (C.c_int32 * max(n, 1))(*dst_slots), (C.c_int32 * max(n, 1))(*src_slots)
        N.check(self.native.lib.vt_chunk_state_copy_slots(self.handle, src.handle, n, d, s, _stream_ptr(self.native.device)))


# --------------------------------------------------------------------------------------------------
# parameter trees with the reference's checkpoint keys
# --------------------------------------------------------------------------------------------------
_TEMPORAL_CONV2 = re.compile(r"^(down_temporal|up_temporal)\.\d+\.block\.\d+\.conv2\.conv\.(weight|bias)$")


def _init_like_reference(rel: str, shape: Tuple[int, ...]) -> torch.Tensor:
    """PyTorch-default style initialisation (kaiming-uniform convs, unit norms), mix_factor = 2.0
    (model_3dcausal.py:238,260) and zero-initialised temporal conv2 (:460-462)."""
    leaf = rel.rsplit(".", 1)[-1]
    if leaf == "mix_factor":
        return torch.full(shape, 2.0)
    if _TEMPORAL_CONV2.match(rel):
        return torch.zeros(shape)
    if len(shape) >= 2:
        fan_in = int(math.prod(shape[1:]))
        bound = 1.0 / math.sqrt(fan_in)
        return torch.empty(shape).uniform_(-bound, bound)
    if ".norm" in rel or rel.startswith("norm_out"):
        return torch.ones(shape) if leaf == "weight" else torch.zeros(shape)
    return torch.empty(shape).uniform_(-0.05, 0.05)


class _Indexed(nn.Module):
    """Stands in for the reference's nn.ModuleList containers (`down`, `up`, `block`, ...): children are named
    "0", "1", ... so the checkpoint keys are identical, and `model.decoder.up_temporal[2]` style indexing works
    (autoencoder_v1_1.py:311-319 uses it)."""

    def __getitem__(self, i: int) -> nn.Module:
        return self._modules[str(i if i >= 0 else len(self._modules) + i)]

    def __len__(self) -> int:
        return len(self._modules)

    def __iter__(self):
        return iter(self._modules[str(i)] for i in range(len(self._modules)))


def _attach(root: nn.Module, rel: str, value: torch.Tensor):
    parts = rel.split(".")
    mod = root
    for i, p in enumerate(parts[:-1]):
        if p not in mod._modules:
            mod.add_module(p, _Indexed() if parts[i + 1].isdigit() else nn.Module())
        mod = mod._modules[p]
    mod.register_parameter(parts[-1], nn.Parameter(value))


class _Stack(nn.Module):
    """Common part of the encoder / decoder mirrors: owns the parameters of one stack."""

    _prefix = ""
    _causal = True

    def __init__(self, version: int, **params):
        super().__init__()
        self.spec = TokenizerSpec.from_params(params, version, causal=self._causal)
        self.norm_type = self.spec.norm_type
        self.ch = self.spec.ch
        self.num_resolutions = len(self.spec.ch_mult)
        self.num_res_blocks = self.spec.num_res_blocks
        self.in_channels = self.spec.in_channels
        self.time_downsample_factor = params.get("time_downsample_factor", 4)
        self.fix_encoder = params.get("fix_encoder", False)
        self.fix_decoder = params.get("fix_decoder", False)
        if not self.spec.double_z:  # the parameter manifest does not depend on the regularizer
            self.spec.regularizer, self.spec.fsq_levels = "fsq", (8,) * self.spec.z_channels
        probe = NativeModel(self.spec)  # manifest only; no CUDA work
        for name, shape in probe.manifest():
            if name.startswith(self._prefix):
                rel = name[len(self._prefix):]
                _attach(self, rel, _init_like_reference(rel, shape))
        del probe
        self._engine = None  # weakref to the owning AutoencodingEngine
        self._solo: Optional["_Runtime"] = None

    def _runtime(self) -> "_Runtime":
        eng = self._engine() if self._engine is not None else None
        if eng is not None:
            return eng._rt
        if self._solo is None:
            self._solo = _Runtime(self.spec, {self._prefix: self})
        return self._solo


class EncoderCausal3DPadding(_Stack):
    """vidtok.modules.model_3dcausal.EncoderCausal3DPadding (model_3dcausal.py:674-689)."""

    _prefix = "encoder."
    _version = 0

    def __init__(self, *args, **params):
        assert not args, "keyword arguments only (as instantiate_from_config passes them)"
        super().__init__(self._version, **params)
        self.is_causal = True
        self.init_pad_mode = params.get("init_pad_mode", "replicate")
        if self.init_pad_mode != "replicate":
            raise NotImplementedError("only init_pad_mode='replicate' (every shipped config) is on the path")
        if self.fix_encoder:
            for p in self.parameters():
                p.requires_grad = False

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        rt = self._runtime()
        _, _, _, h = rt.encode_raw(x, want_h=True, noise=None, need_reg=False)
        return h


class DecoderCausal3DPadding(_Stack):
    """vidtok.modules.model_3dcausal.DecoderCausal3DPadding (model_3dcausal.py:873-885)."""

    _prefix = "decoder."
    _version = 0

    def __init__(self, *args, **params):
        assert not args
        super().__init__(self._version, **params)
        if self.fix_decoder:
            for p in self.parameters():
                p.requires_grad = False

    def get_last_layer(self, **kwargs):
        return self.conv_out.conv.weight

    def forward(self, z: torch.Tensor) -> torch.Tensor:
        return self._runtime().decode_raw(z, from_indices=False)


class Encoder3D(_Stack):
    """vidtok.modules.model_3dnoncausal.Encoder3D (model_3dnoncausal.py:314-482)."""

    _prefix = "encoder."
    _causal = False

    def __init__(self, *args, **params):
        assert not args, "keyword arguments only (as instantiate_from_config passes them)"
        if params.get("norm_type", "groupnorm") != "layernorm":
            raise NotImplementedError("non-causal models with GroupNorm are not on the path (every shipped config uses layernorm)")
        super().__init__(0, **params)
        self.is_causal = False
        self.tempo_ds = [self.num_resolutions - 2, self.num_resolutions - 3]
        if self.fix_encoder:
            for p in self.parameters():
                p.requires_grad = False

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        _, _, _, h = self._runtime().encode_raw(x, want_h=True, noise=None, need_reg=False)
        return h


class Decoder3D(_Stack):
    """vidtok.modules.model_3dnoncausal.Decoder3D (model_3dnoncausal.py:485-651)."""

    _prefix = "decoder."
    _causal = False

    def __init__(self, *args, **params):
        assert not args
        if params.get("norm_type", "groupnorm") != "layernorm":
            raise NotImplementedError("non-causal models with GroupNorm are not on the path (every shipped config uses layernorm)")
        if params.get("give_pre_end") or params.get("tanh_out"):
            raise NotImplementedError("give_pre_end / tanh_out are not used by any shipped config")
        super().__init__(0, **params)
        self.tempo_us = [1, 2]
        if self.fix_decoder:
            for p in self.parameters():
                p.requires_grad = False

    def get_last_layer(self, **kwargs):
        return self.conv_out.weight

    def forward(self, z: torch.Tensor, **kwargs) -> torch.Tensor:
        return self._runtime().decode_raw(z, from_indices=False)


class EncoderCausal3DPaddingV11(EncoderCausal3DPadding):
    _version = 1


class DecoderCausal3DPaddingV11(DecoderCausal3DPadding):
    _version = 1


# --------------------------------------------------------------------------------------------------
# regularizers
# --------------------------------------------------------------------------------------------------
class DiagonalGaussianRegularizer(nn.Module):
    """vidtok.modules.regularizers.DiagonalGaussianRegularizer (regularizers.py:74-92)."""

    def __init__(self, sample: bool = True):
        super().__init__()
        self.sample = sample

    def get_trainable_parameters(self):
        yield from ()

    def forward(self, z: torch.Tensor, n_steps=None):
        if not z.is_cuda:
            raise RuntimeError("vidtok_b200 runs on CUDA devices only")
        lib = N.lib()
        B, C2 = z.shape[0], z.shape[1]
        zc = C2 // 2
        P = z[0, 0].numel()
        zf = z.detach().float().contiguous()
        noise = None
        if self.sample:
            noise = torch.randn((B, zc, *z.shape[2:])).to(device=z.device)  # distributions.py:17
        out = torch.empty((B, zc, *z.shape[2:]), dtype=torch.float32, device=z.device)
        kl = torch.empty((), dtype=torch.float32, device=z.device)
        N.check(lib.vt_op_kl(_ptr(zf), _ptr(noise), zc, P, B, int(self.sample), _ptr(out), _ptr(kl), _stream_ptr(z.device)))
        return out, {"kl_loss": kl}


def _world_size() -> int:
    """regularizers.py:49-64: avg_prob is all-reduced when torch.distributed runs with more than one rank."""
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        return dist.get_world_size()
    return 1


class FSQRegularizer(nn.Module):
    """vidtok.modules.regularizers.FSQRegularizer (regularizers.py:95-268): `z` (codes), `reg_log['indices']` and
    `reg_log['aux_loss']`.  The auxiliary loss (:232-245: clamped per-sample entropy, codebook entropy of the batch-mean
    code distribution, commitment MSE) is computed on the device from one small softmax per latent channel
    (csrc/fsq_aux.cu) instead of the tokens x codebook matrix; it is a device scalar (no host synchronisation).  As in the
    reference it is computed whenever entropy_loss_weight or commitment_loss_weight is positive, in eval too, and avg_prob
    is all-reduced over the ranks of an initialised torch.distributed group.  No gradient flows through it."""

    def __init__(self, levels: List[int], dim: Optional[int] = None, num_codebooks=1,
                 keep_num_codebooks_dim: Optional[bool] = None, scale: Optional[float] = None,
                 entropy_loss_weight: float = 0.0, entropy_loss_annealing_steps: int = 0,
                 entropy_loss_annealing_factor: float = 1.0, commitment_loss_weight: float = 0.0,
                 diversity_gamma: float = 1.0):
        super().__init__()
        if num_codebooks != 1 or (dim is not None and dim != len(levels)):
            raise NotImplementedError("FSQ with projections / multiple codebooks is not used by any shipped config")
        self.levels = [int(l) for l in levels]
        self.register_buffer("_levels", torch.tensor(self.levels, dtype=torch.int32), persistent=False)
        self.register_buffer("_basis", torch.cumprod(torch.tensor([1] + self.levels[:-1]), dim=0, dtype=torch.int32),
                             persistent=False)
        self.codebook_dim = len(levels)
        self.num_codebooks = 1
        self.effective_codebook_dim = self.codebook_dim
        self.keep_num_codebooks_dim = False
        self.dim = len(levels)
        self.has_projections = False
        self.project_in = nn.Identity()
        self.project_out = nn.Identity()
        self.codebook_size = int(math.prod(self.levels))
        self.scale = scale
        self.entropy_loss_weight = entropy_loss_weight
        self.entropy_loss_annealing_steps = entropy_loss_annealing_steps
        self.entropy_loss_annealing_factor = entropy_loss_annealing_factor
        self.commitment_loss_weight = commitment_loss_weight
        self.diversity_gamma = diversity_gamma

    def get_trainable_parameters(self):
        return self.parameters()

    def _levels_c(self):
        return (C.c_int32 * len(self.levels))(*self.levels)

    def calculate_entropy_loss_weight(self, n_steps):
        """regularizers.py:200-204"""
        if n_steps >= self.entropy_loss_annealing_steps:
            return self.entropy_loss_weight
        start = self.entropy_loss_annealing_factor * self.entropy_loss_weight
        return start - (n_steps / self.entropy_loss_annealing_steps) * (start - self.entropy_loss_weight)

    def aux_enabled(self) -> bool:
        """regularizers.py:232: the auxiliary branch runs iff one of its weights is positive."""
        return self.entropy_loss_weight > 0 or self.commitment_loss_weight > 0

    def aux_partials(self, h: torch.Tensor, inv_temperature: float = 100.0) -> Tuple[torch.Tensor, torch.Tensor]:
        """Per-segment partials of the auxiliary loss of one pre-bound latent h [B,d,...]: stats [1,2] = (per-sample
        entropy, commitment MSE) and avg_prob [1,codebook_size]."""
        hf = h.detach().float().contiguous()
        B, P = hf.shape[0], hf[0, 0].numel()
        lib = N.lib()
        nbytes = int(lib.vt_fsq_aux_workspace_bytes(self.dim, self._levels_c(), B * P))
        if nbytes < 0:
            raise RuntimeError(f"vidtok_b200: {lib.vt_last_error().decode()}")
        ws = torch.empty(nbytes, dtype=torch.uint8, device=hf.device)
        stats = torch.empty((1, 2), dtype=torch.float32, device=hf.device)
        avg = torch.empty((1, self.codebook_size), dtype=torch.float32, device=hf.device)
        N.check(lib.vt_fsq_aux_partials(_ptr(hf), self.dim, self._levels_c(), P, B, float(inv_temperature), _ptr(stats), _ptr(avg),
                                        _ptr(ws), nbytes, _stream_ptr(hf.device)))
        return stats, avg

    def aux_finalize(self, stats: torch.Tensor, avg_prob: torch.Tensor, n_steps: int = 0, world_size: Optional[int] = None,
                     components: Optional[torch.Tensor] = None) -> torch.Tensor:
        """aux_loss (a device scalar) from the partials of n segments (stats [n,2], avg_prob [n,codebook_size]): the mean
        over the segments of (per_sample_entropy - diversity_gamma * codebook_entropy) * w(n_steps) + commit *
        commitment_loss_weight.  world_size None: all-reduce avg_prob over the torch.distributed group when there is
        one (in place, regularizers.py:49-59); an explicit world_size means avg_prob already holds the sum over the ranks.
        components (optional, fp32 [n,4] on the device) receives each segment's (per_sample_entropy, codebook_entropy,
        commit_loss, aux)."""
        if world_size is None:
            import torch.distributed as dist
            if _capturing() and dist.is_available() and dist.is_initialized():
                raise RuntimeError("vidtok_b200: the FSQ aux_loss all-reduces avg_prob over the process group, which is not "
                                   "captured in a CUDA graph: capture without return_reg_log, or pass world_size")
            world_size = _world_size()
            if world_size > 1:
                import torch.distributed as dist
                dist.all_reduce(avg_prob)
        aux = torch.empty((), dtype=torch.float32, device=avg_prob.device)
        N.check(N.lib().vt_fsq_aux_finalize(_ptr(stats), _ptr(avg_prob), int(stats.shape[0]), self.dim, self._levels_c(),
                                            int(world_size), float(self.calculate_entropy_loss_weight(n_steps)),
                                            float(self.diversity_gamma), float(self.commitment_loss_weight), _ptr(aux),
                                            _ptr(components), _stream_ptr(avg_prob.device)))
        return aux

    def aux_loss(self, h: torch.Tensor, inv_temperature: float = 100.0, n_steps: int = 0) -> torch.Tensor:
        """reg_log['aux_loss'] of one regularizer call on the pre-bound latent h (0 when both weights are 0)."""
        if not self.aux_enabled():
            return torch.zeros((), device=h.device)
        stats, avg = self.aux_partials(h, inv_temperature)
        return self.aux_finalize(stats, avg, n_steps)

    def indices_to_codes(self, indices: torch.Tensor, project_out=True) -> torch.Tensor:
        """regularizers.py:180-198: [B, ...] int -> [B, d, ...] for image/video shaped input, [..., d] otherwise."""
        if not indices.is_cuda:
            raise RuntimeError("vidtok_b200 runs on CUDA devices only")
        idx = indices.detach().to(torch.int32).contiguous()
        is_img_or_video = idx.ndim >= 3
        B = idx.shape[0] if is_img_or_video else 1
        P = idx.numel() // B
        out = torch.empty((B, self.dim, P), dtype=torch.float32, device=idx.device)
        N.check(N.lib().vt_op_fsq_indices_to_codes(_ptr(idx), self.dim, self._levels_c(), P, B, _ptr(out),
                                                   _stream_ptr(idx.device)))
        if is_img_or_video:
            return out.reshape(B, self.dim, *idx.shape[1:])
        return out.reshape(self.dim, P).t().reshape(*idx.shape, self.dim)

    def forward(self, z: torch.Tensor, inv_temperature: float = 100.0, n_steps: int = 0):
        if not z.is_cuda:
            raise RuntimeError("vidtok_b200 runs on CUDA devices only")
        assert z.shape[1] == self.dim, f"expected dimension of {self.dim} but found dimension of {z.shape[1]}"
        zf = z.detach().float().contiguous()
        B = z.shape[0]
        P = zf[0, 0].numel()
        codes = torch.empty_like(zf)
        idx = torch.empty((B, *z.shape[2:]), dtype=torch.int32, device=z.device)
        N.check(N.lib().vt_op_fsq(_ptr(zf), self.dim, self._levels_c(), P, B, _ptr(codes), _ptr(idx), _stream_ptr(z.device)))
        return codes.to(z.dtype), {"indices": idx, "aux_loss": self.aux_loss(zf, inv_temperature, n_steps)}


# --------------------------------------------------------------------------------------------------
# runtime shared by an engine (or a stand-alone stack)
# --------------------------------------------------------------------------------------------------
class _Runtime:
    def __init__(self, spec: TokenizerSpec, stacks: Dict[str, nn.Module]):
        self.spec = spec
        self.stacks = stacks  # prefix -> module
        self.native: Optional[NativeModel] = None
        self._sig = None
        self.precision_override: Optional[str] = None

    _MODES = {"exact": N.PREC_EXACT_TC, "bf16": N.PREC_BF16, "mixed": N.PREC_MIXED, "fma": N.PREC_FMA32}

    def precision(self) -> int:
        p = self.precision_override
        if p is None:
            return N.PREC_BF16 if torch.is_autocast_enabled() else N.PREC_EXACT_TC
        if p not in self._MODES:
            raise ValueError("precision must be None, 'exact', 'bf16', 'mixed' or 'fma'")
        return self._MODES[p]

    def out_dtype(self) -> torch.dtype:
        """Reference semantics: fp32 tensors, or the autocast dtype inside a torch.autocast region."""
        if self.precision_override is None and torch.is_autocast_enabled():
            return torch.get_autocast_dtype("cuda")
        return torch.float32

    def _params(self):
        for prefix, mod in self.stacks.items():
            for n, p in mod.named_parameters():
                yield prefix + n, p

    def sync(self) -> NativeModel:
        plist = list(self._params())
        if not plist:
            raise RuntimeError("no parameters")
        dev = plist[0][1].device
        if dev.type != "cuda":
            raise RuntimeError("vidtok_b200: the model must live on a CUDA device (model.to('cuda')); there is no CPU path")
        sig = (dev.index, tuple((p.data_ptr(), p._version) for _, p in plist))
        if _capturing():   # loading and finalizing copy and synchronise: a capture needs the weights the last call used
            if self.native is None or sig != self._sig:
                raise RuntimeError("vidtok_b200: the weights changed (or were never loaded) since the last call, and they cannot be "
                                   "repacked while a CUDA graph is being captured: run one eager call after changing them")
            return self.native
        if self.native is None or self.native.device_index != (dev.index or 0):
            self.native = NativeModel(self.spec, dev.index or 0)
            self._sig = None
        if sig != self._sig:
            have = set()
            for name, p in plist:
                self.native.load(name, p.data)
                have.add(name)
            for name, shape in self.native.manifest():  # stand-alone stack: the other half is unused
                if name not in have:
                    self.native.load(name, torch.zeros(shape, device=dev))
            self.native.finalize()
            self._sig = sig
        return self.native

    @staticmethod
    def _as_input(x: torch.Tensor) -> torch.Tensor:
        if not x.is_cuda:
            raise RuntimeError("vidtok_b200: inputs must be CUDA tensors; there is no CPU path")
        if x.dim() != 5:
            raise ValueError("expected a [B,C,T,H,W] tensor")
        return x.detach().to(torch.float32).contiguous()

    def draw_noise(self, shape, device) -> Optional[torch.Tensor]:
        if self.spec.regularizer == "kl" and self.spec.kl_sample:
            return torch.randn(shape).to(device=device)  # CPU generator, as distributions.py:17
        return None

    def encode_raw(self, x, want_h=False, noise=None, need_reg=True):
        nat = self.sync()
        x = self._as_input(x)
        if x.device.index != nat.device_index:
            raise RuntimeError("input and model are on different devices")
        B, _, T, H, W = x.shape
        sampled = self.spec.regularizer == "kl" and self.spec.kl_sample
        if need_reg and noise is not None:
            if not sampled:
                raise ValueError("noise= is the KL regularizer's sample: this model does not sample")
            shape = (B, self.spec.z_channels) + nat.latent_shape(T, H, W)
            if tuple(noise.shape) != shape or not noise.is_cuda or noise.device.index != nat.device_index:
                raise ValueError(f"noise must be a CUDA tensor of shape {shape} on the model's device, got {tuple(noise.shape)}")
            noise = noise.detach().to(torch.float32).contiguous()
        elif need_reg and sampled and _capturing():
            raise RuntimeError("vidtok_b200: the KL sample draws its noise on the CPU generator, which a CUDA graph cannot "
                               "capture: pass noise= (a static device tensor you refill before each replay), or build the "
                               "regularizer with sample=False")
        if need_reg and noise is None:
            Tz, Hz, Wz = nat.latent_shape(T, H, W)
            noise = self.draw_noise((B, self.spec.z_channels, Tz, Hz, Wz), x.device)
        elif not need_reg and self.spec.regularizer == "kl" and self.spec.kl_sample:
            Tz, Hz, Wz = nat.latent_shape(T, H, W)
            noise = torch.zeros((B, self.spec.z_channels, Tz, Hz, Wz), device=x.device)
        return nat.encode(x, noise, self.precision(), want_h=want_h)

    def decode_raw(self, z, from_indices: bool):
        nat = self.sync()
        if not z.is_cuda:
            raise RuntimeError("vidtok_b200: inputs must be CUDA tensors; there is no CPU path")
        z = z.detach().to(torch.int32 if from_indices else torch.float32).contiguous()
        return nat.decode(z, from_indices, self.precision())


# --------------------------------------------------------------------------------------------------
# AutoencodingEngine
# --------------------------------------------------------------------------------------------------
def _instantiate(cfg):
    from .compat_util import instantiate_from_config
    return instantiate_from_config(cfg)


class _EngineBase(nn.Module):
    _version = 0
    global_step = 0

    def __init__(self, *args, encoder_config: Dict, decoder_config: Dict, loss_config: Optional[Dict] = None,
                 regularizer_config: Dict = None, optimizer_config: Optional[Dict] = None, lr_g_factor: float = 1.0,
                 compile_model: bool = False, ckpt_path: Optional[str] = None, ignore_keys=(), verbose: bool = True,
                 ema_decay=None, monitor=None, mode=None, input_key: str = "jpg", **kwargs):
        super().__init__()
        if kwargs:
            raise TypeError(f"unexpected arguments {sorted(kwargs)}")
        self.input_key = input_key
        self.use_ema = ema_decay is not None
        if monitor is not None:
            self.monitor = monitor
        if mode is not None:
            self.mode = mode
        self.encoder = _instantiate(encoder_config)
        self.decoder = _instantiate(decoder_config)
        # The loss (LPIPS + discriminator, vidtok/modules/losses.py) is training-only and downloads VGG weights;
        # it is accepted and skipped here.  Checkpoint keys under `loss.` are ignored like strict=False does.
        self.loss = nn.Identity()
        self.regularization = _instantiate(regularizer_config)
        self.optimizer_config = optimizer_config
        self.lr_g_factor = lr_g_factor
        self.is_causal = self.encoder.is_causal

        spec = TokenizerSpec.from_params(dict(encoder_config.get("params", {})), self._version, causal=self.encoder.spec.causal)
        if self.encoder.spec.causal != self.decoder.spec.causal:
            raise ValueError("encoder and decoder must both be causal or both be non-causal")
        if isinstance(self.regularization, FSQRegularizer):
            spec.regularizer, spec.fsq_levels = "fsq", tuple(self.regularization.levels)
        elif isinstance(self.regularization, DiagonalGaussianRegularizer):
            spec.regularizer, spec.kl_sample = "kl", bool(self.regularization.sample)
        else:
            raise NotImplementedError(f"regularizer {type(self.regularization).__name__} is not on the path")
        if self.encoder.spec.version != self._version or self.decoder.spec.version != self._version:
            raise ValueError("encoder/decoder classes do not match the engine version")
        self.spec = spec
        self._rt = _Runtime(spec, {"encoder.": self.encoder, "decoder.": self.decoder})
        self.encoder._engine = weakref.ref(self)
        self.decoder._engine = weakref.ref(self)
        if ckpt_path is not None:
            self.init_from_ckpt(ckpt_path, ignore_keys=ignore_keys, verbose=verbose)

    # precision selector (extension; see module docstring)
    @property
    def precision(self) -> Optional[str]:
        return self._rt.precision_override

    @precision.setter
    def precision(self, v: Optional[str]):
        self._rt.precision_override = v

    def init_from_ckpt(self, path: str, ignore_keys=tuple(), verbose: bool = True) -> None:
        """autoencoder.py:146-176"""
        if path.endswith("ckpt"):
            ckpt = torch.load(path, map_location="cpu")
            weights = ckpt["state_dict"] if "state_dict" in ckpt else ckpt
        elif path.endswith("safetensors"):
            from safetensors.torch import load_file
            weights = load_file(path)
        else:
            raise NotImplementedError(f"Unknown checkpoint: {path}")
        for k in list(weights.keys()):
            for ik in ignore_keys:
                if re.match(ik, k):
                    del weights[k]
                    break
        missing, unexpected = self.load_state_dict(weights, strict=False)
        if verbose:
            print(f"[vidtok_b200] restored from {path}: {len(missing)} missing, {len(unexpected)} unexpected keys")

    def get_input(self, batch: Dict) -> torch.Tensor:
        return batch[self.input_key]

    def get_last_layer(self):
        return self.decoder.get_last_layer()

    def _wants_aux(self, return_reg_log: bool) -> bool:
        return return_reg_log and self.spec.regularizer == "fsq" and self.regularization.aux_enabled()

    def _reg_log(self, idx, kl, h=None):
        if self.spec.regularizer == "fsq":
            # autoencoder.py:199 / autoencoder_v1_1.py:238: regularization(z, n_steps=self.global_step // 2)
            aux = (self.regularization.aux_loss(h, n_steps=self.global_step // 2) if h is not None
                   else torch.zeros((), device=idx.device))
            return {"indices": idx, "aux_loss": aux}
        return {"kl_loss": kl}

    def indices_to_latent(self, token_indices: torch.Tensor) -> torch.Tensor:
        """autoencoder.py:205-213"""
        return self.regularization.indices_to_codes(token_indices)


class AutoencodingEngine(_EngineBase):
    """vidtok.models.autoencoder.AutoencodingEngine (autoencoder.py:98-229), inference methods."""

    _version = 0

    def encode(self, x: Any, return_reg_log: bool = False, *, noise: Optional[torch.Tensor] = None) -> Any:
        """noise (extension, KL with sampling): the sample's standard normal draws [B,z,Tz,Hz,Wz] on the device instead of
        the CPU generator's; required inside a CUDA graph capture."""
        z, idx, kl, h = self._rt.encode_raw(x, want_h=self._wants_aux(return_reg_log), noise=noise)
        z = z.to(self._rt.out_dtype())
        if return_reg_log:
            return z, self._reg_log(idx, kl, h)
        return z

    def decode(self, z: Any, decode_from_indices: bool = False) -> torch.Tensor:
        return self._rt.decode_raw(z, decode_from_indices).to(self._rt.out_dtype())

    def forward(self, x: Any, *, noise: Optional[torch.Tensor] = None):
        z, reg_log = self.encode(x, return_reg_log=True, noise=noise)
        dec = self.decode(z)
        return z, dec, reg_log


class AutoencodingEngineV11(_EngineBase):
    """vidtok.models.autoencoder_v1_1.AutoencodingEngine (autoencoder_v1_1.py:98-342): adds temporal tiling."""

    _version = 1

    def __init__(self, *args, **kwargs):
        self.__dict__["use_tiling"] = kwargs.pop("use_tiling", False)
        self.__dict__["t_chunk_enc"] = kwargs.pop("t_chunk_enc", 16)
        super().__init__(*args, **kwargs)
        self.t_chunk_dec = self.t_chunk_enc // self.encoder.time_downsample_factor
        self.use_overlap = False

    def build_chunk_start_end(self, t, decoder_mode=False):
        """autoencoder_v1_1.py:218-228: a list of [start, end] lists"""
        return [list(c) for c in chunk_start_end(t, self.t_chunk_dec if decoder_mode else self.t_chunk_enc)]

    def encode(self, x: Any, return_reg_log: bool = False, *, noise: Optional[torch.Tensor] = None) -> Any:
        """noise: as AutoencodingEngine.encode (untiled calls only)."""
        if self.use_tiling:
            if noise is not None:
                raise ValueError("noise= applies to untiled calls: tile_encode draws one sample per chunk")
            z, reg_log = self.tile_encode(x)
        else:
            z, idx, kl, h = self._rt.encode_raw(x, want_h=self._wants_aux(return_reg_log), noise=noise)
            reg_log = self._reg_log(idx, kl, h)
        z = z.to(self._rt.out_dtype())
        if return_reg_log:
            return z, reg_log
        return z

    def tile_encode(self, x: Any) -> Any:
        """autoencoder_v1_1.py:244-264: first frame alone, then chunks of t_chunk_enc, causal caches carried over.  One
        native call per video (vt_encode_video): the chunk loop, the caches and the double-buffered chunk staging live in
        the library.  `x` may be a CUDA tensor or a (pinned) host tensor -- then the chunks are staged host -> device on the
        library's copy stream while the previous chunk computes.  Not capturable in a CUDA graph (the copy stream and the
        host staging): refused under capture."""
        _refuse_capture("tile_encode")
        rt = self._rt
        nat = rt.sync()
        if x.dim() != 5:
            raise ValueError("expected a [B,C,T,H,W] tensor")
        on_host = not x.is_cuda
        x = x.detach().to(torch.float32).contiguous()
        dev = nat.device
        B, Cin, T, H, W = x.shape
        if Cin != self.spec.in_channels:
            raise ValueError(f"input has {Cin} channels, the model expects in_channels = {self.spec.in_channels}")
        prec = rt.precision()
        lib = nat.lib
        chunks = self.build_chunk_start_end(T)
        shapes = [nat.latent_shape(e - s, H, W) for s, e in chunks]
        Hz, Wz = shapes[0][1], shapes[0][2]
        Tz = sum(sh[0] for sh in shapes)
        noise = None
        if self.spec.regularizer == "kl" and self.spec.kl_sample:
            noise = chunk_noise(B, self.spec.z_channels, [sh[0] for sh in shapes], Hz, Wz).to(dev)
        z = torch.empty((B, self.spec.z_channels, Tz, Hz, Wz), dtype=torch.float32, device=dev)
        idx = torch.empty((B, Tz, Hz, Wz), dtype=torch.int32, device=dev) if self.spec.regularizer == "fsq" else None
        kl = torch.empty((), dtype=torch.float32, device=dev) if self.spec.regularizer == "kl" else None
        reg = self.regularization
        if self.spec.regularizer == "fsq" and reg.aux_enabled():
            # one regularizer call per chunk (autoencoder_v1_1.py:253): the chunk loop writes each chunk's aux partials
            stats = torch.empty((len(chunks), 2), dtype=torch.float32, device=dev)
            avg = torch.empty((len(chunks), reg.codebook_size), dtype=torch.float32, device=dev)
            ws = nat._workspace(int(lib.vt_encode_video_fsq_aux_workspace_bytes(nat.handle, prec, B, T, H, W, int(self.t_chunk_enc))))
            N.check(lib.vt_encode_video_fsq_aux(nat.handle, prec, _ptr(x), int(on_host), B, Cin, T, H, W, int(self.t_chunk_enc), _ptr(z),
                                                _ptr(idx), 100.0, _ptr(stats), _ptr(avg), _ptr(ws), ws.numel(), _stream_ptr(dev)))
            if on_host:
                torch.cuda.current_stream(dev).synchronize()
            # per-chunk all-reduce of the reference = one all-reduce of all chunks' avg_prob; mean over the chunks (:261-264)
            return z, {"aux_loss": reg.aux_finalize(stats, avg, n_steps=self.global_step // 2), "indices": idx}
        ws = nat._workspace(int(lib.vt_encode_video_workspace_bytes(nat.handle, prec, B, T, H, W, int(self.t_chunk_enc))))
        N.check(lib.vt_encode_video(nat.handle, prec, _ptr(x), int(on_host), B, Cin, T, H, W, int(self.t_chunk_enc), _ptr(noise), _ptr(z),
                                    _ptr(idx), _ptr(kl), _ptr(ws), ws.numel(), _stream_ptr(dev)))
        if on_host:
            torch.cuda.current_stream(dev).synchronize()   # the host tensor must outlive the staged copies
        if self.spec.regularizer == "kl":
            return z, {"kl_loss": kl}
        return z, {"aux_loss": torch.zeros((), device=dev), "indices": idx}

    def tile_indices_to_latent(self, token_indices: torch.Tensor) -> torch.Tensor:
        return self.indices_to_latent(token_indices)

    def decode(self, z: Any, decode_from_indices: bool = False) -> torch.Tensor:
        if decode_from_indices:
            z = self.indices_to_latent(z)
        if self.use_tiling:
            return self.tile_decode(z).to(self._rt.out_dtype())
        return self._rt.decode_raw(z, False).to(self._rt.out_dtype())

    def tile_decode(self, z: Any, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """autoencoder_v1_1.py:302-331: one look-ahead latent frame per chunk when use_overlap, tail frames dropped.  One
        native call per video (vt_decode_video).  `out` (optional): a pre-allocated fp32 [B,C,T',H,W] tensor, CUDA or pinned
        host memory -- decoded chunks are then copied out on the library's copy stream while the next chunk computes.  Not
        capturable in a CUDA graph, as tile_encode."""
        _refuse_capture("tile_decode")
        rt = self._rt
        nat = rt.sync()
        if not z.is_cuda:
            raise RuntimeError("vidtok_b200: inputs must be CUDA tensors; there is no CPU path")
        if z.dim() != 5 or z.shape[1] != self.spec.z_channels:
            raise ValueError(f"expected a [B,{self.spec.z_channels},T,H,W] latent, got {tuple(z.shape)}")
        z = z.detach().float().contiguous()
        B, Cz, nf, Hz, Wz = z.shape
        tdf = self.encoder.time_downsample_factor
        if self.use_overlap:
            assert tdf in [2, 4, 8], "Only support 2x, 4x or 8x temporal downsampling now."
        prec = rt.precision()
        f = nat.spatial_factor()
        lib = nat.lib
        tcd, ov = int(self.t_chunk_dec), int(bool(self.use_overlap))
        T_out = int(lib.vt_decode_video_frames(nat.handle, nf, tcd, ov))
        shape = (B, self.spec.out_ch, T_out, Hz * f, Wz * f)
        if out is None:
            out = torch.empty(shape, dtype=torch.float32, device=z.device)
        elif tuple(out.shape) != shape or out.dtype != torch.float32 or not out.is_contiguous():
            raise ValueError(f"out must be a contiguous fp32 tensor of shape {shape}")
        ws = nat._workspace(int(lib.vt_decode_video_workspace_bytes(nat.handle, prec, B, nf, Hz, Wz, tcd, ov)))
        N.check(lib.vt_decode_video(nat.handle, prec, _ptr(z), B, Cz, nf, Hz, Wz, tcd, ov, _ptr(out), int(not out.is_cuda), _ptr(ws),
                                    ws.numel(), _stream_ptr(z.device)))
        if not out.is_cuda:
            torch.cuda.current_stream(z.device).synchronize()
        return out

    def forward(self, x: Any, *, noise: Optional[torch.Tensor] = None):
        z, reg_log = self.encode(x, return_reg_log=True, noise=noise)
        dec = self.decode(z)
        if dec.shape[2] != x.shape[2]:  # autoencoder_v1_1.py:340-341
            dec = dec[:, :, -x.shape[2]:, ...]
        return z, dec, reg_log
