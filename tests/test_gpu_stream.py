"""-m gpu: streaming encode / decode (vidtok_b200.streaming) and the cached fused temporal block.

A causal v1.0 stream computes exactly the whole-clip function (every norm and attention works within one frame, the caches
carry what each causal convolution, time resampling and fused temporal block needs from the previous chunk), so the
checks here are bitwise: streamed latents, FSQ indices and reconstructions are torch.equal to the whole-clip calls.

One exception, in the split-operand modes ("exact", and "mixed"'s encoder) at small spatial sizes: conv_tc sums a tile's K steps
in kparts groups sized from the taps the tile does not skip, and when a level's H x W does not fill 128 rows the tile is
several frames deep, a depth chosen from the clip length.  The whole clip's own first frames then round differently for
different clip lengths (the latents of the first 5 frames of a 17-frame clip are not bitwise those of a 5-frame clip), so no
chunking can match every length bit for bit.  The split-operand encoder also differs from the whole clip by fp32 rounding
(measured 7e-6 on kl488 latents) at production geometry, where the cause is not yet pinned down.  Those cases are held to
fp32 rounding here; bf16 and fma streams are bitwise everywhere."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from conftest import load_golden, resolved_model_cfg, synth_weights  # noqa: E402
from vidtok_b200 import _native as N  # noqa: E402

V10_CASES = ["tiny_kl_v10", "tiny_fsq_v10", "tiny_kl_gn_v10", "tiny_kl_444_v10", "tiny_kl_288_v10", "tiny_kl_v10_t8",
             "mid_kl_v10", "mid_fsq_v10"]
SCHEDULES = {"1+4x4": [1, 4, 4, 4, 4], "1+16": [1, 16], "17": [17], "ragged": [3, 2, 7, 5]}


def _model(cfg, sd):
    from vidtok_b200.compat_util import instantiate_from_config
    model = instantiate_from_config(cfg)
    missing, unexpected = model.load_state_dict(sd, strict=False)
    assert not missing and not unexpected
    return model.to("cuda").eval()


def _latents_after(frames, tdf):
    """latent frames a v1.0 encode stream has produced once `frames` frames were pushed"""
    return 0 if frames < 1 else 1 + (frames - 1) // tdf


def _stream_encode(model, x, schedule, noise=None):
    from vidtok_b200.streaming import EncodeStream
    B, _, T, H, W = x.shape
    tdf = model.encoder.time_downsample_factor
    enc = EncodeStream(model, B, H, W)
    zs, logs, t0 = [], [], 0
    for n in schedule:
        a, b = _latents_after(t0, tdf), _latents_after(t0 + n, tdf)
        z, log = enc.push(x[:, :, t0:t0 + n], noise=None if noise is None else noise[:, :, a:b])
        assert z.shape[2] == b - a
        zs.append(z)
        logs.append(log)
        t0 += n
    enc.close()
    return torch.cat(zs, dim=2), logs


def _stream_decode(model, z, schedule):
    from vidtok_b200.streaming import DecodeStream
    dec = DecodeStream(model, z.shape[0], z.shape[3], z.shape[4])
    outs, t0 = [], 0
    for n in schedule:
        outs.append(dec.push(z[:, :, t0:t0 + n]))
        t0 += n
    dec.close()
    return torch.cat(outs, dim=2)


def _same(got, want, bitwise, what):
    if bitwise:
        assert torch.equal(got, want), (what, float((got - want).abs().max()))
    else:
        err = float((got - want).abs().max())
        assert got.shape == want.shape and err <= 1e-4 * (1.0 + float(want.abs().max())), (what, err)


def _whole_and_noise(model, x, seed=1234):
    """whole-clip encode, and the noise tensor it drew (KL with sampling), for slicing into the pushes"""
    torch.manual_seed(seed)
    z, log = model.encode(x, return_reg_log=True)
    noise = None
    s = model.spec
    if s.regularizer == "kl" and s.kl_sample:
        torch.manual_seed(seed)
        noise = torch.randn(tuple(z.shape))
    return z, log, noise


@pytest.mark.parametrize("mode", ["exact", "bf16", "mixed", "fma"])
@pytest.mark.parametrize("case", V10_CASES)
def test_v10_stream_equals_whole_clip(case, mode):
    from vidtok_b200.synth import synth_clip
    d, meta = load_golden(case)
    model = _model(resolved_model_cfg(meta), synth_weights(meta, d))
    model.precision = mode
    B, _, _, H, W = meta["input"]
    x = synth_clip(B, 17, H, W, seed=meta["input_seed"]).cuda()
    enc_bitwise = mode in ("bf16", "fma")   # see the module docstring for the split-operand modes
    dec_bitwise = mode in ("bf16", "fma", "mixed")
    with torch.no_grad():
        z_w, log_w, noise = _whole_and_noise(model, x)
        for name, sched in SCHEDULES.items():
            z, logs = _stream_encode(model, x, sched, noise)
            _same(z, z_w, enc_bitwise or len(sched) == 1, name)
            if model.spec.regularizer == "fsq":
                idx = torch.cat([l["indices"] for l in logs], dim=1)
                mism = int((idx != log_w["indices"]).sum())
                assert mism == 0 or (not enc_bitwise and mism <= 1e-3 * idx.numel()), (name, mism)
            else:
                kl = sum(float(l["kl_loss"]) for l in logs)
                assert abs(kl - float(log_w["kl_loss"])) <= 1e-6 * abs(float(log_w["kl_loss"])), (name, kl, float(log_w["kl_loss"]))
        x_w = model.decode(z_w)
        tz = z_w.shape[2]
        for name, sched in {"ones": [1] * tz, "all": [tz], "2+rest": [2, tz - 2]}.items():
            xs = _stream_decode(model, z_w, sched)
            _same(xs, x_w, dec_bitwise or len(sched) == 1, name)
        if model.spec.regularizer == "fsq":   # token indices decode like their codes
            from vidtok_b200.streaming import DecodeStream
            dec = DecodeStream(model, B, z_w.shape[3], z_w.shape[4])
            assert torch.equal(dec.push(log_w["indices"]), model.decode(model.indices_to_latent(log_w["indices"])))
            dec.close()


def _kl488(seed=0):
    import os
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
    from oracle.make_golden import model_yaml
    from vidtok_b200.compat_util import instantiate_from_config
    from vidtok_b200.synth import synth_state_dict
    cfg = model_yaml(version="v1_0", reg="kl", ch=128, ch_mult=(1, 2, 4, 4), z=4, interp=None)
    cfg["params"]["decoder_config"]["params"] = dict(cfg["params"]["encoder_config"]["params"])
    cfg["params"]["regularizer_config"]["params"] = {"sample": False}   # z = the mode: no noise
    model = instantiate_from_config(cfg)
    model.load_state_dict(synth_state_dict({k: tuple(v.shape) for k, v in model.state_dict().items()}, seed=seed))
    return model.cuda().eval()


def _launches(fn):
    import ctypes as C
    import json
    lib = N.lib()
    lib.vt_profile_start()
    out = fn()
    torch.cuda.synchronize()
    buf = C.create_string_buffer(1 << 16)
    n = lib.vt_profile_stop(buf, len(buf))
    prof = json.loads(buf.value.decode()) if n > 0 else {}
    return out, {k: v["launches"] for k, v in prof.items()}


@pytest.mark.parametrize("mode", ["bf16", "exact"])
def test_kl488_production_geometry_stream(mode):
    """kl_causal_488_4chn with synthetic weights, 1x3x33x256x256: streamed (1 + 16 + 16 frames) equals the whole clip (bf16
    bit for bit, exact to fp32 rounding: see the module docstring), and the streamed bf16 run launches the fused temporal block per chunk exactly as the whole clip does (no fallback
    to two conv_tc launches)."""
    from vidtok_b200.synth import synth_clip
    model = _kl488()
    model.precision = mode
    x = synth_clip(1, 33, 256, 256, seed=7).cuda()
    with torch.no_grad():
        z_w, lw = _launches(lambda: model.encode(x))
        z_s, ls = _launches(lambda: _stream_encode(model, x, [1, 16, 16])[0])
        _same(z_s, z_w, mode == "bf16", "encode")
        x_w = model.decode(z_w)
        x_s = _stream_decode(model, z_w, [1, 4, 4])
        _same(x_s, x_w, mode == "bf16", "decode")
    if mode == "bf16":
        assert lw.get("tblock_tc", 0) > 0 and ls.get("tblock_tc", 0) == 3 * lw["tblock_tc"], (lw, ls)
        assert ls.get("conv_tc", 0) == 3 * lw.get("conv_tc", 0), (lw, ls)


def test_high_resolution_streams():
    """720x1280 bf16: a 17-frame stream equals the whole-clip encode and decode bitwise.  1080x1920 exact (the whole clip
    does not fit on an 80 GB card): a 17-frame stream runs, and by causality its first two latent frames equal the
    whole-clip encode of the first 5 frames (to fp32 rounding, see the module docstring)."""
    from vidtok_b200.synth import synth_clip
    model = _kl488()
    with torch.no_grad():
        model.precision = "bf16"
        x = synth_clip(1, 17, 720, 1280, seed=3).cuda()
        z_w = model.encode(x)
        z_s = _stream_encode(model, x, [1, 4, 4, 4, 4])[0]
        assert torch.equal(z_s, z_w)
        x_w = model.decode(z_w)
        x_s = _stream_decode(model, z_w, [1, 2, 2])
        assert torch.equal(x_s, x_w)
        del x, x_w, x_s
        torch.cuda.empty_cache()
        model.precision = "exact"
        x = synth_clip(1, 17, 1080, 1920, seed=5).cuda()
        z_s = _stream_encode(model, x, [1, 4, 4, 4, 4])[0]
        assert z_s.shape == (1, 4, 5, 135, 240)
        model._rt.native._ws = None
        torch.cuda.empty_cache()
        z5 = model.encode(x[:, :, :5].contiguous())
        _same(z_s[:, :, :2], z5, False, "1080p exact")


@pytest.mark.parametrize("case", ["tiny_kl_v11_tiled", "tiny_fsq_v11_tiled"])
def test_v11_stream_equals_tile_encode_without_overlap(case):
    from vidtok_b200.synth import synth_clip
    d, meta = load_golden(case)
    model = _model(resolved_model_cfg(meta), synth_weights(meta, d))
    model.precision = "exact"
    model.use_tiling, model.t_chunk_enc, model.t_chunk_dec, model.use_overlap = True, 16, 4, False
    B, _, _, H, W = meta["input"]
    x = synth_clip(B, 33, H, W, seed=meta["input_seed"]).cuda()
    with torch.no_grad():
        torch.manual_seed(5)
        z_t, log_t = model.tile_encode(x)
        noise = None
        if model.spec.regularizer == "kl" and model.spec.kl_sample:
            torch.manual_seed(5)
            noise = torch.cat([torch.randn((B, model.spec.z_channels, n, z_t.shape[3], z_t.shape[4])) for n in (1, 4, 4)], dim=2)
        from vidtok_b200.streaming import EncodeStream
        enc = EncodeStream(model, B, H, W)
        zs, t0, l0 = [], 0, 0
        for n, nl in ((1, 1), (16, 4), (16, 4)):
            z, log = enc.push(x[:, :, t0:t0 + n], noise=None if noise is None else noise[:, :, l0:l0 + nl])
            zs.append(z)
            t0, l0 = t0 + n, l0 + nl
        enc.close()
        assert torch.equal(torch.cat(zs, dim=2), z_t)
        x_t = model.tile_decode(z_t)
        x_s = _stream_decode(model, z_t, [1, 4, 4])
        assert torch.equal(x_s, x_t)


@pytest.mark.parametrize("case", ["tiny_kl_v10", "tiny_fsq_v11_tiled"])
def test_fresh_chunk_state_refuses_a_later_chunk(case):
    """A chunk state that has not run a first chunk holds no cached frames: a later chunk is refused with VT_ERR_NOT_READY
    (-3), naming the cache, before anything reads it; the same state then takes a first chunk as a fresh stream does."""
    from vidtok_b200.engine import _ptr, _stream_ptr
    from vidtok_b200.streaming import DecodeStream, EncodeStream
    from vidtok_b200.synth import synth_clip
    d, meta = load_golden(case)
    model = _model(resolved_model_cfg(meta), synth_weights(meta, d))
    model.precision = "bf16"
    s = model.spec
    tdf = int(s.time_downsample_factor)
    B, _, _, H, W = meta["input"]
    x = synth_clip(B, 1 + tdf, H, W, seed=meta["input_seed"]).cuda()
    dev = x.device
    with torch.no_grad():
        enc = EncodeStream(model, B, H, W)
        lib = enc.native.lib
        Hz, Wz = enc.Hz, enc.Wz
        noise = torch.randn((B, s.z_channels, 2, Hz, Wz))   # 1 + tdf frames: two latent frames
        xc = x[:, :, 1:].contiguous()                        # tdf frames: a later chunk
        nc = noise[:, :, 1:].contiguous().to(dev)
        z = torch.empty((B, s.z_channels, 1, Hz, Wz), device=dev)
        idx = torch.empty((B, 1, Hz, Wz), dtype=torch.int32, device=dev)
        kl = torch.zeros((1,), device=dev)
        ws = enc.state.workspace(tdf)
        rc = lib.vt_encode_chunk(enc.state.handle, 0, _ptr(xc), s.in_channels, tdf, _ptr(nc), _ptr(z), _ptr(idx), _ptr(kl),
                                 _ptr(ws), ws.numel(), _stream_ptr(dev))
        msg = lib.vt_last_error().decode()
        assert rc == -3 and msg.startswith("cache encoder.") and "empty" in msg, (rc, msg)
        z_s, _ = enc.push(x, noise=noise)
        enc.close()
        z_f, _ = _stream_encode(model, x, [1 + tdf], noise)
        assert torch.equal(z_s, z_f)

        dec = DecodeStream(model, B, Hz, Wz)
        zc = z_f[:, :, 1:].float().contiguous()
        To = dec.native.decoded_frames(1) if s.version == 1 else tdf
        out = torch.empty((B, s.out_ch, To, H, W), device=dev)
        ws = dec.state.workspace(1)
        rc = lib.vt_decode_chunk(dec.state.handle, 0, _ptr(zc), s.z_channels, 1, _ptr(out), _ptr(ws), ws.numel(), _stream_ptr(dev))
        msg = lib.vt_last_error().decode()
        assert rc == -3 and msg.startswith("cache decoder.") and "empty" in msg, (rc, msg)
        x_s = dec.push(z_f)
        dec.close()
        assert torch.equal(x_s, _stream_decode(model, z_f, [z_f.shape[2]]))


# ---------------------------------------------------------------------------------------------------------------
# op level: the cached fused temporal block
# ---------------------------------------------------------------------------------------------------------------
def _tblock_operands(B, T, H, W, seed=0):
    g = torch.Generator().manual_seed(seed)
    C_ = 128
    r = lambda *s, sc=1.0: torch.randn(*s, generator=g) * sc  # noqa: E731
    n1 = r(B, T, H, W, C_).to(torch.bfloat16)
    x = r(B, T, H, W, C_).to(torch.bfloat16)
    w1 = (r(C_, C_, 3, sc=1 / math.sqrt(3 * C_))).to(torch.bfloat16).float()
    w2 = (r(C_, C_, 3, sc=1 / math.sqrt(3 * C_))).to(torch.bfloat16).float()
    vec = [r(C_) * 0.3 for _ in range(6)]
    vec[1], vec[4] = 1.0 + vec[1], 1.0 + vec[4]   # b1, g2, be2, b2, g3, be3
    return n1, x, w1, w2, vec


def _tblock(n1, x, w1, w2, vec, caches=None):
    from gpu_util import _p, stream
    B, T, H, W, C_ = n1.shape
    dev = [t.contiguous().cuda() for t in (n1, x, w1, w2, *vec)]
    n1d, xd, w1d, w2d, b1, g2, be2, b2, g3, be3 = dev
    o, o2 = torch.empty_like(xd), torch.empty_like(xd)
    if caches is None:
        N.check(N.lib().vt_op_tblock(_p(n1d), _p(xd), _p(w1d), _p(b1), _p(g2), _p(be2), _p(w2d), _p(b2), _p(g3), _p(be3), 1,
                                     _p(o), _p(o2), B, T, H, W, C_, stream()))
    else:
        cn1, ch, cn1_out, ch_out = caches
        N.check(N.lib().vt_op_tblock_cached(_p(n1d), _p(xd), _p(w1d), _p(b1), _p(g2), _p(be2), _p(w2d), _p(b2), _p(g3), _p(be3), 1,
                                            _p(o), _p(o2), _p(cn1), _p(ch), _p(cn1_out), _p(ch_out), B, T, H, W, C_, stream()))
    torch.cuda.synchronize()
    return o, o2


@pytest.mark.parametrize("chunk", [1, 2, 4])
def test_cached_tblock_chunks_equal_one_launch(chunk):
    """A T-frame block run as chunks of 1, 2 or 4 frames through the cached kernel equals one uncached launch bitwise."""
    B, T, H, W = 2, 8, 16, 64
    n1, x, w1, w2, vec = _tblock_operands(B, T, H, W, seed=3)
    o_ref, o2_ref = _tblock(n1, x, w1, w2, vec)
    shape = (B, 2, H, W, 128)
    bufs = [torch.full(shape, float("nan"), dtype=torch.bfloat16, device="cuda") for _ in range(4)]
    cur = None
    outs, outs2 = [], []
    for t0 in range(0, T, chunk):
        nxt = (bufs[0], bufs[1]) if cur is None or cur[0] is bufs[2] else (bufs[2], bufs[3])
        o, o2 = _tblock(n1[:, t0:t0 + chunk], x[:, t0:t0 + chunk], w1, w2, vec,
                        caches=(None, None, *nxt) if cur is None else (*cur, *nxt))
        outs.append(o)
        outs2.append(o2)
        cur = nxt
    assert torch.equal(torch.cat(outs, dim=1), o_ref)
    assert torch.equal(torch.cat(outs2, dim=1), o2_ref)
    # the n1 cache after the last chunk holds the block input's last two frames
    assert torch.equal(cur[0].cpu(), n1[:, T - 2:])


def test_cached_tblock_against_fp64_with_cache_frames_prepended():
    """out = x + conv2(silu(LN2(conv1([n1 cache | n1])))) with h's cache frames in front of conv2's input, in fp64 on the
    bf16 operands; h is bf16 inside the kernel, hence the slack."""
    import torch.nn.functional as F
    from test_gpu_ops_tc import check, ln_ref
    B, T, H, W, C_ = 1, 3, 8, 128, 128
    n1, x, w1, w2, (b1, g2, be2, b2, g3, be3) = _tblock_operands(B, T, H, W, seed=9)
    g = torch.Generator().manual_seed(10)
    cn1 = torch.randn((B, 2, H, W, C_), generator=g).to(torch.bfloat16)
    ch = torch.randn((B, 2, H, W, C_), generator=g).to(torch.bfloat16)
    outs = [torch.empty((B, 2, H, W, C_), dtype=torch.bfloat16, device="cuda") for _ in range(2)]
    o, o2 = _tblock(n1, x, w1, w2, [b1, g2, be2, b2, g3, be3], caches=(cn1.cuda(), ch.cuda(), *outs))

    def tconv(a, w, b):   # [B,T',H,W,C] fp64, valid causal conv over T' -> T'-2 frames
        Tp = a.shape[1]
        a = a.permute(0, 2, 3, 4, 1).reshape(-1, C_, Tp)
        return F.conv1d(a, w.double(), b.double()).reshape(B, H, W, C_, Tp - 2).permute(0, 4, 1, 2, 3)
    h = tconv(torch.cat([cn1, n1], dim=1).double(), w1, b1)
    hn = ln_ref(h.permute(0, 4, 1, 2, 3), g2, be2, True).permute(0, 2, 3, 4, 1).to(torch.bfloat16)
    ref = x.double() + tconv(torch.cat([ch, hn], dim=1).double(), w2, b2)
    ref2 = ln_ref(ref.permute(0, 4, 1, 2, 3), g3, be3, True).permute(0, 2, 3, 4, 1)
    check(o.float().cpu(), ref, N.PREC_BF16, "cached tblock out", slack=2.0)
    check(o2.float().cpu(), ref2, N.PREC_BF16, "cached tblock out2", slack=2.5)
    assert torch.equal(outs[0].cpu(), n1[:, 1:])
    check(outs[1].float().cpu()[:, 0], hn[:, 1].double(), N.PREC_BF16, "h cache", slack=2.0)
    check(outs[1].float().cpu()[:, 1], hn[:, 2].double(), N.PREC_BF16, "h cache", slack=2.0)
