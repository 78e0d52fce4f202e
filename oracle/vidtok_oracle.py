"""TEST INFRASTRUCTURE ONLY.

CPU restatement (plain PyTorch fp32/fp64 functional code, NCDHW like the reference) of the VidTok causal
tokenizer hot path: encode -> KL/FSQ regularize -> decode, for the v1.0 and v1.1 model families.
Only tests/, __graft_entry__.smoke() and bench.py's CPU-baseline / `--impl reference` legs may import
this file; the product path (vidtok_b200/) never does and fails loudly without its CUDA library.

Parity pin: the reference ships no tests or golden vectors (SURVEY.md section 4), so this restatement
is pinned against the UNMODIFIED reference modules imported from /root/reference in the authoring
container: oracle/make_golden.py runs both on identical seeded weights/inputs, asserts agreement, and
writes tests/golden/*.npz; tests/test_oracle_golden.py re-checks this file against those fixtures on
any machine (the GPU box has no /root/reference).

Every function cites the reference file:line it restates (paths relative to /root/reference).
State dict keys are the reference's checkpoint keys (SURVEY.md section 8b).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import torch
import torch.nn.functional as F

Tensor = torch.Tensor


# --------------------------------------------------------------------------------------------------
# configuration (mirrors the encoder `params:` block of configs/*.yaml)
# --------------------------------------------------------------------------------------------------
@dataclass
class OracleCfg:
    ch: int = 128
    ch_mult: Tuple[int, ...] = (1, 2, 4, 4)
    num_res_blocks: int = 2
    in_channels: int = 3
    out_ch: int = 3
    z_channels: int = 4
    double_z: bool = True
    norm_type: str = "layernorm"
    time_downsample_factor: int = 4
    spatial_ds: Optional[List[int]] = None
    tempo_ds: Optional[List[int]] = None
    spatial_us: Optional[List[int]] = None
    tempo_us: Optional[List[int]] = None
    version: str = "v1_0"  # "v1_0" | "v1_1"
    interpolation_mode: str = "nearest"  # v1.1 only (model_3dcausal_v1_1.py:794)
    regularizer: str = "kl"  # "kl" | "fsq"
    fsq_levels: Tuple[int, ...] = (8, 8, 8, 8, 8)
    kl_sample: bool = True
    causal: bool = True  # False: vidtok.modules.model_3dnoncausal.Encoder3D / Decoder3D (v1.0 only)

    @property
    def nres(self) -> int:
        return len(self.ch_mult)

    def enc_spatial_ds(self):  # model_3dcausal.py:539
        return list(range(0, self.nres - 1)) if self.spatial_ds is None else list(self.spatial_ds)

    def enc_tempo_ds(self):  # model_3dcausal.py:540
        return [self.nres - 2, self.nres - 3] if self.tempo_ds is None else list(self.tempo_ds)

    def dec_spatial_us(self):  # model_3dcausal.py:756
        return list(range(1, self.nres)) if self.spatial_us is None else list(self.spatial_us)

    def dec_tempo_us(self):  # model_3dcausal.py:757
        return [1, 2] if self.tempo_us is None else list(self.tempo_us)


def cfg_from_model_yaml(model_cfg: dict) -> OracleCfg:
    """model_cfg = `model:` section of a reference YAML."""
    ep = model_cfg["params"]["encoder_config"]["params"]
    tgt = model_cfg["target"]
    reg = model_cfg["params"]["regularizer_config"]
    kw = dict(
        ch=ep["ch"], ch_mult=tuple(ep["ch_mult"]), num_res_blocks=ep["num_res_blocks"],
        in_channels=ep["in_channels"], out_ch=ep["out_ch"], z_channels=ep["z_channels"],
        double_z=ep.get("double_z", True), norm_type=ep.get("norm_type", "groupnorm"),
        time_downsample_factor=ep.get("time_downsample_factor", 4),
        spatial_ds=ep.get("spatial_ds"), tempo_ds=ep.get("tempo_ds"),
        spatial_us=ep.get("spatial_us"), tempo_us=ep.get("tempo_us"),
        version="v1_1" if "v1_1" in tgt else "v1_0",
        interpolation_mode=ep.get("interpolation_mode", "nearest"),
        causal="noncausal" not in model_cfg["params"]["encoder_config"]["target"],
    )
    if not kw["causal"]:   # model_3dnoncausal.py:335,515: fixed schedules, no overrides
        kw["spatial_ds"] = kw["tempo_ds"] = kw["spatial_us"] = kw["tempo_us"] = None
    if reg["target"].endswith("FSQRegularizer"):
        kw["regularizer"] = "fsq"
        kw["fsq_levels"] = tuple(reg["params"]["levels"])
    else:
        kw["regularizer"] = "kl"
        kw["kl_sample"] = reg.get("params", {}).get("sample", True)
    return OracleCfg(**kw)


# --------------------------------------------------------------------------------------------------
# chunk state for v1.1 (the reference keeps these as attributes on the modules:
# model_3dcausal_v1_1.py:155-157,212-214,286-287,321-323)
# --------------------------------------------------------------------------------------------------
@dataclass
class ChunkState:
    first: bool = True
    cache: Dict[str, Tensor] = field(default_factory=dict)
    cache_offset: Dict[str, int] = field(default_factory=dict)  # key prefix -> offset

    def offset_for(self, key: str) -> int:
        best, val = -1, 0
        for p, v in self.cache_offset.items():
            if key.startswith(p) and len(p) > best:
                best, val = len(p), v
        return val


# --------------------------------------------------------------------------------------------------
# primitives
# --------------------------------------------------------------------------------------------------
def silu(x: Tensor) -> Tensor:
    """model_3dcausal.py:26-27 -- x * sigmoid(x)."""
    return x * torch.sigmoid(x)


def norm(sd, key: str, x: Tensor, cfg: OracleCfg, per_position: bool = False) -> Tensor:
    """Normalize() applied the way every call site applies it: per frame.

    layernorm: model_3dcausal.py:62-80 -- nn.LayerNorm(C, eps=1e-6) over the channel axis at every
    (b,t,h,w); checkpoint keys `<key>.norm.{weight,bias}`.
    groupnorm: model_3dcausal.py:30-32 -- GroupNorm(32, C, eps=1e-6) on `(b t) c h w`
    (model_3dcausal.py:403-406,477-480,665-668 rearrange before the norm, so statistics are per frame);
    keys `<key>.{weight,bias}`.
    per_position=True restates the temporal 1D blocks: ResnetCausalBlock1D._forward takes
    `B = x.shape[0]` of the `(b h w) c t` tensor (model_3dcausal.py:474), so its
    "(b s) c t -> (b t) c s" rearrange (:477,486) yields s == 1 and GroupNorm statistics run over the
    C/32 channels of ONE position (LayerNorm is per-position either way).
    x: [B,C,T,H,W].
    """
    B, C, T, H, W = x.shape
    if cfg.norm_type == "layernorm":
        y = F.layer_norm(x.permute(0, 2, 3, 4, 1), (C,), sd[key + ".norm.weight"], sd[key + ".norm.bias"], eps=1e-6)
        return y.permute(0, 4, 1, 2, 3)
    if per_position:
        y = x.permute(0, 2, 3, 4, 1).reshape(-1, C, 1)
        y = F.group_norm(y, 32, sd[key + ".weight"], sd[key + ".bias"], eps=1e-6)
        return y.reshape(B, T, H, W, C).permute(0, 4, 1, 2, 3)
    y = x.permute(0, 2, 1, 3, 4).reshape(B * T, C, H, W)
    y = F.group_norm(y, 32, sd[key + ".weight"], sd[key + ".bias"], eps=1e-6)
    return y.reshape(B, T, C, H, W).permute(0, 2, 1, 3, 4)


def _time_front(x: Tensor, time_pad: int, key: str, cfg: OracleCfg, st: Optional[ChunkState]) -> Tensor:
    """Front padding in time for a causal conv.

    v1.0: zeros (model_3dcausal.py:157-158,194-196; pad_mode is always "constant").
    v1.1: first frame replicated on the first chunk, else the tail of the cached padded input of the
    previous chunk; then cache := padded input minus `cache_offset` tail frames
    (model_3dcausal_v1_1.py:159-176,216-233).
    """
    if cfg.version == "v1_0":
        return F.pad(x, (0, 0, 0, 0, time_pad, 0))
    if st.first:
        pad = x[:, :, :1].repeat(1, 1, time_pad, 1, 1)
    else:
        c = st.cache[key]
        pad = c[:, :, -time_pad:] if time_pad != 0 else c[:, :, 0:0]
    x = torch.cat((pad, x), dim=2)
    off = st.offset_for(key)
    st.cache[key] = x.clone() if off == 0 else x[:, :, :-off].clone()
    return x


def causal_conv3d(sd, key: str, x: Tensor, cfg: OracleCfg, st, stride=(1, 1, 1)) -> Tensor:
    """CausalConv3d: model_3dcausal.py:162-197 (v1.0) / model_3dcausal_v1_1.py:181-236 (v1.1).
    keys `<key>.conv.{weight,bias}`; spatial zero padding (k-1)+(1-stride) split floor/ceil."""
    w, b = sd[key + ".conv.weight"], sd[key + ".conv.bias"]
    kt, kh, kw = w.shape[2:]
    time_pad = (kt - 1) + (1 - stride[0])
    hp = (kh - 1) + (1 - stride[1])
    wp = (kw - 1) + (1 - stride[2])
    x = _time_front(x, time_pad, key, cfg, st)
    x = F.pad(x, (wp // 2, wp - wp // 2, hp // 2, hp - hp // 2, 0, 0))
    return F.conv3d(x, w, b, stride=stride)


def causal_conv1d(sd, key: str, x: Tensor, cfg: OracleCfg, st) -> Tensor:
    """CausalConv1d on `(b h w) c t`: model_3dcausal.py:144-159 / model_3dcausal_v1_1.py:144-178.
    x: [B,C,T,H,W] (the rearranges of model_3dcausal.py:20,22 are done here)."""
    w, b = sd[key + ".conv.weight"], sd[key + ".conv.bias"]
    B, C, T, H, W = x.shape
    k = w.shape[2]
    x = _time_front(x, k - 1, key, cfg, st)
    Tp = x.shape[2]
    y = x.permute(0, 3, 4, 1, 2).reshape(B * H * W, C, Tp)
    y = F.conv1d(y, w, b)
    return y.reshape(B, H, W, -1, y.shape[-1]).permute(0, 3, 4, 1, 2)


def conv2d_frames(x: Tensor, w: Tensor, b: Tensor, stride=1, padding=0) -> Tensor:
    """nn.Conv2d applied on `(b t) c h w` (model_3dcausal.py:17-19)."""
    B, C, T, H, W = x.shape
    y = x.permute(0, 2, 1, 3, 4).reshape(B * T, C, H, W)
    y = F.conv2d(y, w, b, stride=stride, padding=padding)
    return y.reshape(B, T, y.shape[1], y.shape[2], y.shape[3]).permute(0, 2, 1, 3, 4)


def resnet_block_2d(sd, key: str, x: Tensor, cfg: OracleCfg) -> Tensor:
    """ResnetBlock._forward: model_3dcausal.py:317-337 (temb is None, dropout p=0)."""
    h = silu(norm(sd, key + ".norm1", x, cfg))
    h = conv2d_frames(h, sd[key + ".conv1.weight"], sd[key + ".conv1.bias"], padding=1)
    h = silu(norm(sd, key + ".norm2", h, cfg))
    h = conv2d_frames(h, sd[key + ".conv2.weight"], sd[key + ".conv2.bias"], padding=1)
    if key + ".nin_shortcut.weight" in sd:
        x = conv2d_frames(x, sd[key + ".nin_shortcut.weight"], sd[key + ".nin_shortcut.bias"])
    return x + h


def resnet_block_1d(sd, key: str, x: Tensor, cfg: OracleCfg, st) -> Tensor:
    """ResnetCausalBlock1D._forward: model_3dcausal.py:473-499 (in==out channels always)."""
    h = silu(norm(sd, key + ".norm1", x, cfg, per_position=True))
    h = causal_conv1d(sd, key + ".conv1", h, cfg, st)
    h = silu(norm(sd, key + ".norm2", h, cfg, per_position=True))
    h = causal_conv1d(sd, key + ".conv2", h, cfg, st)
    return x + h


def resnet_block_3d(sd, key: str, x: Tensor, cfg: OracleCfg, st) -> Tensor:
    """ResnetCausalBlock._forward: model_3dcausal.py:400-424 (mid blocks, in==out)."""
    h = silu(norm(sd, key + ".norm1", x, cfg))
    h = causal_conv3d(sd, key + ".conv1", h, cfg, st)
    h = silu(norm(sd, key + ".norm2", h, cfg))
    h = causal_conv3d(sd, key + ".conv2", h, cfg, st)
    return x + h


def attn_block(sd, key: str, x: Tensor, cfg: OracleCfg, st) -> Tensor:
    """AttnBlockWrapper: model_3dcausal.py:114-141 -- per-frame single-head attention, D=C,
    scale C**-0.5 (SDPA default), q/k/v/proj are 1x1x1 causal convs."""
    B, C, T, H, W = x.shape
    h = norm(sd, key + ".norm", x, cfg)
    q = causal_conv3d(sd, key + ".q", h, cfg, st)
    k = causal_conv3d(sd, key + ".k", h, cfg, st)
    v = causal_conv3d(sd, key + ".v", h, cfg, st)
    q, k, v = (t.permute(0, 2, 3, 4, 1).reshape(B, T, H * W, C) for t in (q, k, v))
    o = F.scaled_dot_product_attention(q, k, v)
    o = o.reshape(B, T, H, W, C).permute(0, 4, 1, 2, 3)
    o = causal_conv3d(sd, key + ".proj_out", o, cfg, st)
    return x + o


def downsample(sd, key: str, x: Tensor) -> Tensor:
    """Downsample: model_3dcausal.py:223-230 -- zero pad (0,1,0,1) then conv3x3 stride 2."""
    B, C, T, H, W = x.shape
    y = x.permute(0, 2, 1, 3, 4).reshape(B * T, C, H, W)
    y = F.pad(y, (0, 1, 0, 1))
    y = F.conv2d(y, sd[key + ".conv.weight"], sd[key + ".conv.bias"], stride=2)
    return y.reshape(B, T, C, y.shape[2], y.shape[3]).permute(0, 2, 1, 3, 4)


def upsample(sd, key: str, x: Tensor) -> Tensor:
    """Upsample: model_3dcausal.py:208-212 -- nearest 2x (H,W) then conv3x3 pad 1."""
    B, C, T, H, W = x.shape
    y = x.permute(0, 2, 1, 3, 4).reshape(B * T, C, H, W)
    y = F.interpolate(y.float(), scale_factor=2.0, mode="nearest").to(x.dtype)
    y = F.conv2d(y, sd[key + ".conv.weight"], sd[key + ".conv.bias"], padding=1)
    return y.reshape(B, T, C, 2 * H, 2 * W).permute(0, 2, 1, 3, 4)


def time_downsample(sd, key: str, x: Tensor, cfg: OracleCfg, st) -> Tensor:
    """TimeDownsampleResCausal2x: model_3dcausal.py:247-252 / model_3dcausal_v1_1.py:289-302.
    alpha*avgpool3d((3,1,1),s=(2,1,1))(front-pad-1(x)) + (1-alpha)*cconv3d(k3,s=(2,1,1))(x)."""
    alpha = torch.sigmoid(sd[key + ".mix_factor"])
    if cfg.version == "v1_0":
        xp = F.pad(x, (0, 0, 0, 0, 1, 0))
    else:
        if st.first:
            xp = F.pad(x, (0, 0, 0, 0, 1, 0), mode="replicate")
        else:
            xp = torch.cat((st.cache[key + "#pool"], x), dim=2)
        st.cache[key + "#pool"] = xp[:, :, -1:].clone()
    x1 = F.avg_pool3d(xp, (3, 1, 1), stride=(2, 1, 1))
    x2 = causal_conv3d(sd, key + ".conv", x, cfg, st, stride=(2, 1, 1))
    return alpha * x1 + (1 - alpha) * x2


def time_upsample(sd, key: str, x: Tensor, cfg: OracleCfg, st, num_temp_upsample: int) -> Tensor:
    """TimeUpsampleResCausal2x: model_3dcausal.py:267-273 / model_3dcausal_v1_1.py:325-343."""
    alpha = torch.sigmoid(sd[key + ".mix_factor"])
    mode = "nearest" if cfg.version == "v1_0" else cfg.interpolation_mode

    def interp(t):
        return F.interpolate(t.float(), scale_factor=[2.0, 1.0, 1.0], mode=mode).to(t.dtype)

    if mode != "trilinear":
        x = interp(x)
    elif not st.first:
        n = num_temp_upsample
        x = torch.cat([st.cache[key + "#up"], x], dim=2)
        st.cache[key + "#up"] = x[:, :, -2 * n:-n].clone()
        x = interp(x)[:, :, 2 * n:]
    else:
        n = num_temp_upsample
        st.cache[key + "#up"] = x[:, :, -n:].clone()
        a, b = x[:, :, :n], x[:, :, n:]
        a = interp(a)
        x = torch.cat([a, interp(b)], dim=2) if b.shape[2] > 0 else a
    x_ = causal_conv3d(sd, key + ".conv", x, cfg, st)
    return alpha * x + (1 - alpha) * x_


# --------------------------------------------------------------------------------------------------
# non-causal family (vidtok/modules/model_3dnoncausal.py): same stacks, symmetric zero padding in time, plain
# nn.Conv3d / nn.Conv1d (checkpoint keys without the inner `.conv`), no front padding / frame dropping
# --------------------------------------------------------------------------------------------------
def nc_conv3d(sd, key: str, x: Tensor, stride=(1, 1, 1), padding=None) -> Tensor:
    """nn.Conv3d(k, padding=(k-1)/2): model_3dnoncausal.py:20-23,271,276,348,430,522,600."""
    w, b = sd[key + ".weight"], sd[key + ".bias"]
    if padding is None:
        padding = tuple((k - 1) // 2 for k in w.shape[2:])
    return F.conv3d(x, w, b, stride=stride, padding=padding)


def nc_conv1d(sd, key: str, x: Tensor) -> Tensor:
    """nn.Conv1d(k=3, padding=1) on `(b h w) c t` (model_3dnoncausal.py:203,208; rearranges of model_3dcausal.py:20,22)."""
    w, b = sd[key + ".weight"], sd[key + ".bias"]
    B, C, T, H, W = x.shape
    y = x.permute(0, 3, 4, 1, 2).reshape(B * H * W, C, T)
    y = F.conv1d(y, w, b, padding=1)
    return y.reshape(B, H, W, -1, T).permute(0, 3, 4, 1, 2)


def nc_norm(sd, key: str, x: Tensor, cfg: OracleCfg, mode: str) -> Tensor:
    """Normalize() as the non-causal call sites apply it.  layernorm: per position over C everywhere
    (model_3dcausal.py:62-80).  groupnorm (no shipped config): statistics over whatever tensor the call site passes --
    `frames`: `(b t) c h w` (ResnetBlock, via spatial_temporal_resblk), `seq`: `(b h w) c t` (ResnetBlock1D,
    model_3dnoncausal.py:221-235), `volume`: the 5-D tensor (ResnetNoncausalBlock :284-300, AttnBlockWrapper :25-26)."""
    B, C, T, H, W = x.shape
    if cfg.norm_type == "layernorm":
        y = F.layer_norm(x.permute(0, 2, 3, 4, 1), (C,), sd[key + ".norm.weight"], sd[key + ".norm.bias"], eps=1e-6)
        return y.permute(0, 4, 1, 2, 3)
    g, b = sd[key + ".weight"], sd[key + ".bias"]
    if mode == "frames":
        y = F.group_norm(x.permute(0, 2, 1, 3, 4).reshape(B * T, C, H, W), 32, g, b, eps=1e-6)
        return y.reshape(B, T, C, H, W).permute(0, 2, 1, 3, 4)
    if mode == "seq":
        y = F.group_norm(x.permute(0, 3, 4, 1, 2).reshape(B * H * W, C, T), 32, g, b, eps=1e-6)
        return y.reshape(B, H, W, C, T).permute(0, 3, 4, 1, 2)
    return F.group_norm(x, 32, g, b, eps=1e-6)


def nc_resblock(sd, key: str, x: Tensor, cfg: OracleCfg, kind: str) -> Tensor:
    """ResnetBlock (2D, frames) / ResnetBlock1D (seq) / ResnetNoncausalBlock (volume): model_3dnoncausal.py:152-179,
    221-248,284-311 -- norm, SiLU, conv, norm, SiLU, conv, + skip (1x1 nin_shortcut when channels change)."""
    def conv(k, t):
        if kind == "frames":
            return conv2d_frames(t, sd[k + ".weight"], sd[k + ".bias"], padding=(sd[k + ".weight"].shape[-1] - 1) // 2)
        if kind == "seq":
            return nc_conv1d(sd, k, t)
        return nc_conv3d(sd, k, t)
    h = conv(key + ".conv1", silu(nc_norm(sd, key + ".norm1", x, cfg, kind)))
    h = conv(key + ".conv2", silu(nc_norm(sd, key + ".norm2", h, cfg, kind)))
    if key + ".nin_shortcut.weight" in sd:
        x = conv(key + ".nin_shortcut", x)
    return x + h


def nc_attn_block(sd, key: str, x: Tensor, cfg: OracleCfg) -> Tensor:
    """AttnBlockWrapper: model_3dnoncausal.py:17-34 (per-frame single-head SDPA, 1x1x1 nn.Conv3d projections)."""
    B, C, T, H, W = x.shape
    h = nc_norm(sd, key + ".norm", x, cfg, "volume")
    q, k, v = (nc_conv3d(sd, f"{key}.{n}", h).permute(0, 2, 3, 4, 1).reshape(B, T, H * W, C) for n in ("q", "k", "v"))
    o = F.scaled_dot_product_attention(q, k, v).reshape(B, T, H, W, C).permute(0, 4, 1, 2, 3)
    return x + nc_conv3d(sd, key + ".proj_out", o)


def nc_time_downsample(sd, key: str, x: Tensor) -> Tensor:
    """TimeDownsampleRes2x: model_3dnoncausal.py:84-90 -- one zero frame appended, then
    alpha*avgpool3d((3,1,1),s=(2,1,1)) + (1-alpha)*conv3d(k3, s=(2,1,1), padding=(0,1,1))."""
    alpha = torch.sigmoid(sd[key + ".mix_factor"])
    xp = F.pad(x, (0, 0, 0, 0, 0, 1))
    return alpha * F.avg_pool3d(xp, (3, 1, 1), stride=(2, 1, 1)) + (1 - alpha) * nc_conv3d(sd, key + ".conv", xp, stride=(2, 1, 1), padding=(0, 1, 1))


def nc_time_upsample(sd, key: str, x: Tensor) -> Tensor:
    """TimeUpsampleRes2x: model_3dnoncausal.py:105-115 -- nearest 2x in T, alpha*x' + (1-alpha)*conv3d(k3, pad 1)(x')."""
    alpha = torch.sigmoid(sd[key + ".mix_factor"])
    x = F.interpolate(x.float(), scale_factor=[2.0, 1.0, 1.0], mode="nearest").to(x.dtype)
    return alpha * x + (1 - alpha) * nc_conv3d(sd, key + ".conv", x)


def nc_encoder_forward(sd, x: Tensor, cfg: OracleCfg) -> Tensor:
    """Encoder3D.forward: model_3dnoncausal.py:446-482 (tempo_ds = [L-2, L-3], :335)."""
    P = "encoder."
    L = cfg.nres
    h = nc_conv3d(sd, P + "conv_in", x)
    for lvl in range(L):
        for blk in range(cfg.num_res_blocks):
            h = nc_resblock(sd, f"{P}down.{lvl}.block.{blk}", h, cfg, "frames")
            h = nc_resblock(sd, f"{P}down_temporal.{lvl}.block.{blk}", h, cfg, "seq")
        if lvl != L - 1:
            h = downsample(sd, f"{P}down.{lvl}.downsample", h)
            if lvl in (L - 2, L - 3):
                h = nc_time_downsample(sd, f"{P}down_temporal.{lvl}.downsample", h)
    h = nc_resblock(sd, P + "mid.block_1", h, cfg, "volume")
    h = nc_attn_block(sd, P + "mid.attn_1", h, cfg)
    h = nc_resblock(sd, P + "mid.block_2", h, cfg, "volume")
    return nc_conv3d(sd, P + "conv_out", silu(nc_norm(sd, P + "norm_out", h, cfg, "volume")))


def nc_decoder_forward(sd, z: Tensor, cfg: OracleCfg) -> Tensor:
    """Decoder3D.forward: model_3dnoncausal.py:618-651 (tempo_us = [1, 2], :515)."""
    P = "decoder."
    h = nc_conv3d(sd, P + "conv_in", z)
    h = nc_resblock(sd, P + "mid.block_1", h, cfg, "volume")
    h = nc_attn_block(sd, P + "mid.attn_1", h, cfg)
    h = nc_resblock(sd, P + "mid.block_2", h, cfg, "volume")
    for lvl in reversed(range(cfg.nres)):
        for blk in range(cfg.num_res_blocks + 1):
            h = nc_resblock(sd, f"{P}up.{lvl}.block.{blk}", h, cfg, "frames")
            h = nc_resblock(sd, f"{P}up_temporal.{lvl}.block.{blk}", h, cfg, "seq")
        if lvl != 0:
            h = upsample(sd, f"{P}up.{lvl}.upsample", h)
            if lvl in (1, 2):
                h = nc_time_upsample(sd, f"{P}up_temporal.{lvl}.upsample", h)
    return nc_conv3d(sd, P + "conv_out", silu(nc_norm(sd, P + "norm_out", h, cfg, "volume")))


# --------------------------------------------------------------------------------------------------
# encoder / decoder stacks
# --------------------------------------------------------------------------------------------------
def encoder_forward(sd, x: Tensor, cfg: OracleCfg, st: Optional[ChunkState] = None) -> Tensor:
    """EncoderCausal3DPadding.forward -> EncoderCausal3D.forward: model_3dcausal.py:685-689,631-671
    (v1.1: model_3dcausal_v1_1.py:755-760).  Keys under `encoder.`."""
    tdf = cfg.time_downsample_factor
    T = x.shape[2]
    if T % tdf != 0:
        tp = (tdf - 1) if cfg.version == "v1_0" else (tdf - T % tdf)
        x = torch.cat([x[:, :, :1].repeat(1, 1, tp, 1, 1), x], dim=2)  # init_pad_mode "replicate"
    P = "encoder."
    h = causal_conv3d(sd, P + "conv_in", x, cfg, st)
    sds, tds = cfg.enc_spatial_ds(), cfg.enc_tempo_ds()
    for lvl in range(cfg.nres):
        for blk in range(cfg.num_res_blocks):
            h = resnet_block_2d(sd, f"{P}down.{lvl}.block.{blk}", h, cfg)
            h = resnet_block_1d(sd, f"{P}down_temporal.{lvl}.block.{blk}", h, cfg, st)
        if lvl in sds:
            h = downsample(sd, f"{P}down.{lvl}.downsample", h)
            if lvl in tds:
                h = time_downsample(sd, f"{P}down_temporal.{lvl}.downsample", h, cfg, st)
    h = resnet_block_3d(sd, P + "mid.block_1", h, cfg, st)
    h = attn_block(sd, P + "mid.attn_1", h, cfg, st)
    h = resnet_block_3d(sd, P + "mid.block_2", h, cfg, st)
    h = silu(norm(sd, P + "norm_out", h, cfg))
    return causal_conv3d(sd, P + "conv_out", h, cfg, st)


def decoder_forward(sd, z: Tensor, cfg: OracleCfg, st: Optional[ChunkState] = None) -> Tensor:
    """DecoderCausal3DPadding.forward -> DecoderCausal3D.forward: model_3dcausal.py:883-885,828-870.
    v1.0 drops the first tdf-1 frames (:885); v1.1 returns everything (model_3dcausal_v1_1.py:959)."""
    P = "decoder."
    h = causal_conv3d(sd, P + "conv_in", z, cfg, st)
    h = resnet_block_3d(sd, P + "mid.block_1", h, cfg, st)
    h = attn_block(sd, P + "mid.attn_1", h, cfg, st)
    h = resnet_block_3d(sd, P + "mid.block_2", h, cfg, st)
    sus, tus = cfg.dec_spatial_us(), cfg.dec_tempo_us()
    # num_temp_upsample doubles in construction order (levels visited high->low):
    # model_3dcausal_v1_1.py:856,880-882
    ntu, n = {}, 1
    for lvl in reversed(range(cfg.nres)):
        if lvl in tus:
            ntu[lvl] = n
            n *= 2
    for lvl in reversed(range(cfg.nres)):
        for blk in range(cfg.num_res_blocks + 1):
            h = resnet_block_2d(sd, f"{P}up.{lvl}.block.{blk}", h, cfg)
            h = resnet_block_1d(sd, f"{P}up_temporal.{lvl}.block.{blk}", h, cfg, st)
        if lvl in sus:
            h = upsample(sd, f"{P}up.{lvl}.upsample", h)
            if lvl in tus:
                h = time_upsample(sd, f"{P}up_temporal.{lvl}.upsample", h, cfg, st, ntu[lvl])
    h = silu(norm(sd, P + "norm_out", h, cfg))
    h = causal_conv3d(sd, P + "conv_out", h, cfg, st)
    if cfg.version == "v1_0":
        h = h[:, :, cfg.time_downsample_factor - 1:]
    return h


# --------------------------------------------------------------------------------------------------
# regularizers
# --------------------------------------------------------------------------------------------------
def kl_regularize(h: Tensor, noise: Optional[Tensor], sample: bool = True):
    """DiagonalGaussianRegularizer.forward + DiagonalGaussianDistribution:
    regularizers.py:82-92, distributions.py:5-28.  `noise` stands for the reference's
    torch.randn(mean.shape) drawn on the CPU generator (distributions.py:17); the caller draws it at
    the same point so both paths consume the same numbers."""
    mean, logvar = torch.chunk(h, 2, dim=1)
    logvar = torch.clamp(logvar, -30.0, 20.0)
    std = torch.exp(0.5 * logvar)
    var = torch.exp(logvar)
    z = mean + std * noise.to(h.dtype) if sample else mean
    kl = 0.5 * torch.sum(mean.pow(2) + var - 1.0 - logvar, dim=[1, 2, 3])
    return z, {"kl_loss": torch.sum(kl) / kl.shape[0]}


def fsq_constants(levels, dtype=torch.float32, device="cpu"):
    """regularizers.py:111-115,153-158: levels, basis=cumprod([1]+levels[:-1]), half_l, offset, shift (computed on the
    CPU, then placed on `device`)."""
    lv = torch.tensor(levels, dtype=torch.int32)
    basis = torch.cumprod(torch.tensor([1] + list(levels[:-1])), dim=0, dtype=torch.int32)
    half_l = (lv - 1) * (1 + 1e-3) / 2
    offset = torch.where(lv % 2 == 0, 0.5, 0.0)
    shift = (offset / half_l).atanh()
    return tuple(t.to(device) for t in (lv, basis, half_l.to(dtype), offset.to(dtype), shift.to(dtype)))


def fsq_regularize(h: Tensor, levels):
    """FSQRegularizer.forward, inference outputs only: regularizers.py:206-268 (project_in/out are
    Identity because dim == len(levels), :135-140).  Returns codes [B,d,T,H,W] (fp32 math as in
    :225-227, cast back to the input dtype :249) and int32 indices [B,T,H,W].
    aux_loss (the 32768-way entropy branch, :232-245) is NOT restated: no inference consumer reads it
    (SURVEY.md section 0.7); reported as 0."""
    lv, basis, half_l, offset, shift = fsq_constants(levels, device=h.device)
    z = h.permute(0, 2, 3, 4, 1).float()  # b t h w d
    bounded = torch.tanh(z + shift) * half_l - offset  # bound(): :153-158
    q = bounded.round()  # round_ste: :35-38 (half-to-even)
    half_w = lv // 2
    codes = q / half_w  # quantize(): :160-164
    idx = ((codes * half_w + half_w) * basis).sum(dim=-1).to(torch.int32)  # :166-178
    codes = codes.to(h.dtype).permute(0, 4, 1, 2, 3)
    return codes, {"indices": idx, "aux_loss": torch.zeros((), dtype=h.dtype, device=h.device), "pre_round": bounded}


def fsq_indices_to_codes(idx: Tensor, levels, dtype=torch.float32) -> Tensor:
    """indices_to_codes + AutoencodingEngine.indices_to_latent: regularizers.py:180-198,
    autoencoder.py:205-213.  idx [B,T,H,W] int -> codes [B,d,T,H,W]."""
    lv, basis, *_ = fsq_constants(levels, device=idx.device)
    d = (idx.unsqueeze(-1) // basis) % lv
    half_w = lv // 2
    codes = (d - half_w) / half_w
    return codes.to(dtype).permute(0, 4, 1, 2, 3)


# --------------------------------------------------------------------------------------------------
# wrapper: AutoencodingEngine.encode / decode / forward
# --------------------------------------------------------------------------------------------------
def build_chunk_start_end(t: int, chunk: int):
    """autoencoder_v1_1.py:218-228 -- [[0,1],[1,1+chunk],...]."""
    out = [[0, 1]]
    start = end = 1
    while start < t:
        end = min(t, end + chunk)
        out.append([start, end])
        start = end
    return out


class OracleModel:
    """Functional stand-in for vidtok.models.autoencoder[_v1_1].AutoencodingEngine (inference methods
    only: autoencoder.py:197-229, autoencoder_v1_1.py:230-342)."""

    def __init__(self, cfg: OracleCfg, state_dict: Dict[str, Tensor], dtype=torch.float32):
        self.cfg = cfg
        self.sd = {k: v.to(dtype) for k, v in state_dict.items() if k.startswith(("encoder.", "decoder."))}
        self.dtype = dtype
        self.use_tiling = False
        self.t_chunk_enc = 16
        self.t_chunk_dec = self.t_chunk_enc // cfg.time_downsample_factor
        self.use_overlap = False

    # noise_fn() must return torch.randn(shape) exactly where the reference would call it
    def _regularize(self, h: Tensor, noise_fn):
        if self.cfg.regularizer == "fsq":
            z, log = fsq_regularize(h, self.cfg.fsq_levels)
            return z, log
        shape = (h.shape[0], h.shape[1] // 2, *h.shape[2:])
        noise = noise_fn(shape) if self.cfg.kl_sample else None
        return kl_regularize(h, noise, self.cfg.kl_sample)

    @torch.no_grad()
    def encode(self, x: Tensor, noise_fn=torch.randn, return_pre: bool = False):
        cfg = self.cfg
        x = x.to(self.dtype)
        if not cfg.causal:
            h = nc_encoder_forward(self.sd, x, cfg)
            z, log = self._regularize(h, noise_fn)
            return (z, log, h) if return_pre else (z, log)
        if cfg.version == "v1_0":
            h = encoder_forward(self.sd, x, cfg, None)
            z, log = self._regularize(h, noise_fn)
            return (z, log, h) if return_pre else (z, log)
        st = ChunkState(first=True)
        if not self.use_tiling:
            h = encoder_forward(self.sd, x, cfg, st)
            z, log = self._regularize(h, noise_fn)
            return (z, log, h) if return_pre else (z, log)
        zs, logs, hs = [], [], []
        for i, (s, e) in enumerate(build_chunk_start_end(x.shape[2], self.t_chunk_enc)):
            st.first = i == 0
            h = encoder_forward(self.sd, x[:, :, s:e], cfg, st)
            z, log = self._regularize(h, noise_fn)
            zs.append(z), logs.append(log), hs.append(h)
        z = torch.cat(zs, dim=2)
        if "kl_loss" in logs[0]:  # autoencoder_v1_1.py:256-259
            log = {"kl_loss": torch.mean(torch.stack([d["kl_loss"] for d in logs]))}
        else:  # :261-264
            log = {"aux_loss": torch.mean(torch.stack([d["aux_loss"] for d in logs])),
                   "indices": torch.cat([d["indices"] for d in logs], dim=1),
                   "pre_round": torch.cat([d["pre_round"] for d in logs], dim=1)}
        return (z, log, torch.cat(hs, dim=2)) if return_pre else (z, log)

    @torch.no_grad()
    def decode(self, z: Tensor, decode_from_indices: bool = False):
        cfg = self.cfg
        if decode_from_indices:
            z = fsq_indices_to_codes(z, cfg.fsq_levels, self.dtype)
        z = z.to(self.dtype)
        if not cfg.causal:
            return nc_decoder_forward(self.sd, z, cfg)
        if cfg.version == "v1_0":
            return decoder_forward(self.sd, z, cfg, None)
        st = ChunkState(first=True)
        if not self.use_tiling:
            return decoder_forward(self.sd, z, cfg, st)
        tdf = cfg.time_downsample_factor
        if self.use_overlap:  # autoencoder_v1_1.py:307-320
            assert tdf in (2, 4, 8)
            D = "decoder."
            st.cache_offset[D] = 1
            if tdf == 4:
                for k in ("up_temporal.2.upsample", "up_temporal.1."):
                    st.cache_offset[D + k] = 2
                for k in ("up_temporal.1.upsample", "up_temporal.0.", "conv_out"):
                    st.cache_offset[D + k] = 4
            elif tdf == 2:
                for k in ("up_temporal.2.upsample", "up_temporal.1.", "up_temporal.0.", "conv_out"):
                    st.cache_offset[D + k] = 2
            else:
                for k in ("up_temporal.3.upsample", "up_temporal.2."):
                    st.cache_offset[D + k] = 2
                for k in ("up_temporal.2.upsample", "up_temporal.1."):
                    st.cache_offset[D + k] = 4
                for k in ("up_temporal.1.upsample", "up_temporal.0.", "conv_out"):
                    st.cache_offset[D + k] = 8
        nf = z.shape[2]
        outs = []
        for i, (s, e) in enumerate(build_chunk_start_end(nf, self.t_chunk_dec)):
            st.first = i == 0
            look = self.use_overlap and e + 1 <= nf
            c = decoder_forward(self.sd, z[:, :, s:e + 1] if look else z[:, :, s:e], cfg, st)
            if look:
                c = c[:, :, :-tdf]
            outs.append(c)
        return torch.cat(outs, dim=2)

    @torch.no_grad()
    def forward(self, x: Tensor, noise_fn=torch.randn):
        z, log = self.encode(x, noise_fn)
        dec = self.decode(z)
        if dec.shape[2] != x.shape[2]:  # autoencoder_v1_1.py:340-341
            dec = dec[:, :, -x.shape[2]:]
        return z, dec, log


# --------------------------------------------------------------------------------------------------
# metric (vidtok/modules/util.py:146-155)
# --------------------------------------------------------------------------------------------------
def compute_psnr(x: Tensor, y: Tensor) -> Tensor:
    if x.dim() == 5:
        x = x.permute(0, 2, 1, 3, 4).reshape(-1, x.shape[1], x.shape[3], x.shape[4])
        y = y.permute(0, 2, 1, 3, 4).reshape(-1, y.shape[1], y.shape[3], y.shape[4])
    mse = torch.mean((x - y) ** 2, dim=[1, 2, 3])
    return (-10 * torch.log10(mse + 1e-8)).mean(dim=0)


# --------------------------------------------------------------------------------------------------
# parameter table: the checkpoint keys / shapes the reference modules register
# (EncoderCausal3D.__init__ model_3dcausal.py:535-620, DecoderCausal3D.__init__ :724-811; v1.1 identical keys)
# --------------------------------------------------------------------------------------------------
def reference_param_shapes(cfg: OracleCfg) -> Dict[str, Tuple[int, ...]]:
    """{state_dict key: shape} of the reference model for `cfg` -- lets the CPU-only legs (bench.py reference arm,
    tests) build synthetic weights without touching the CUDA library."""
    out: Dict[str, Tuple[int, ...]] = {}
    ln = cfg.norm_type == "layernorm"

    def norm(key, c):
        k = key + ".norm" if ln else key
        out[k + ".weight"], out[k + ".bias"] = (c,), (c,)

    inner = ".conv" if cfg.causal else ""   # CausalConv3d / CausalConv1d wrap an nn.Conv; the non-causal family uses it directly

    def conv3d(key, co, ci, k=3):
        out[key + inner + ".weight"], out[key + inner + ".bias"] = (co, ci, k, k, k), (co,)

    def conv1d(key, co, ci):
        out[key + inner + ".weight"], out[key + inner + ".bias"] = (co, ci, 3), (co,)

    def tconv(key, c):   # Time{Down,Up}sampleRes[Causal]2x.conv
        out[key + ".conv" + inner + ".weight"], out[key + ".conv" + inner + ".bias"] = (c, c, 3, 3, 3), (c,)

    def conv2d(key, co, ci, k):
        out[key + ".weight"], out[key + ".bias"] = (co, ci, k, k), (co,)

    def res2d(key, ci, co):
        norm(key + ".norm1", ci); conv2d(key + ".conv1", co, ci, 3); norm(key + ".norm2", co); conv2d(key + ".conv2", co, co, 3)
        if ci != co:
            conv2d(key + ".nin_shortcut", co, ci, 1)

    def res1d(key, c):
        norm(key + ".norm1", c); conv1d(key + ".conv1", c, c); norm(key + ".norm2", c); conv1d(key + ".conv2", c, c)

    def res3d(key, c):
        norm(key + ".norm1", c); conv3d(key + ".conv1", c, c); norm(key + ".norm2", c); conv3d(key + ".conv2", c, c)

    def attn(key, c):
        norm(key + ".norm", c)
        for n in ("q", "k", "v", "proj_out"):
            conv3d(f"{key}.{n}", c, c, 1)

    L = cfg.nres
    conv3d("encoder.conv_in", cfg.ch, cfg.in_channels)
    block_in = cfg.ch
    for l in range(L):
        block_out = cfg.ch * cfg.ch_mult[l]
        for b in range(cfg.num_res_blocks):
            res2d(f"encoder.down.{l}.block.{b}", block_in, block_out)
            res1d(f"encoder.down_temporal.{l}.block.{b}", block_out)
            block_in = block_out
        if l in cfg.enc_spatial_ds():
            conv2d(f"encoder.down.{l}.downsample.conv", block_in, block_in, 3)
            if l in cfg.enc_tempo_ds():
                out[f"encoder.down_temporal.{l}.downsample.mix_factor"] = (1,)
                tconv(f"encoder.down_temporal.{l}.downsample", block_in)
    res3d("encoder.mid.block_1", block_in); attn("encoder.mid.attn_1", block_in); res3d("encoder.mid.block_2", block_in)
    norm("encoder.norm_out", block_in)
    conv3d("encoder.conv_out", (2 if cfg.double_z else 1) * cfg.z_channels, block_in)

    block_in = cfg.ch * cfg.ch_mult[L - 1]
    conv3d("decoder.conv_in", block_in, cfg.z_channels)
    res3d("decoder.mid.block_1", block_in); attn("decoder.mid.attn_1", block_in); res3d("decoder.mid.block_2", block_in)
    for l in reversed(range(L)):
        block_out = cfg.ch * cfg.ch_mult[l]
        for b in range(cfg.num_res_blocks + 1):
            res2d(f"decoder.up.{l}.block.{b}", block_in, block_out)
            res1d(f"decoder.up_temporal.{l}.block.{b}", block_out)
            block_in = block_out
        if l in cfg.dec_spatial_us():
            conv2d(f"decoder.up.{l}.upsample.conv", block_in, block_in, 3)
        if l in cfg.dec_tempo_us():
            out[f"decoder.up_temporal.{l}.upsample.mix_factor"] = (1,)
            tconv(f"decoder.up_temporal.{l}.upsample", block_in)
    norm("decoder.norm_out", block_in)
    conv3d("decoder.conv_out", cfg.out_ch, block_in)
    return out
