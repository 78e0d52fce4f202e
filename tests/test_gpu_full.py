"""-m gpu: BASELINE.json configurations at (or near) their full sizes.

The oracle is only affordable on one clip, so the full-size checks combine (i) one-clip comparisons against the oracle
run on the box's host cores and (ii) size-independent properties at the BASELINE batch sizes: batch independence,
determinism, exact-vs-bf16 agreement, decode(indices) == decode(codes), tiled-encode == untiled-encode.
"exact" is the split-operand (fp16 hi|lo x 3 MMAs) tensor-core mode (VT_PREC_EXACT_TC): the 1e-3 / bit-exact gates below run on wgmma."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu


def make_cfg(version="v1_0", reg="kl", ch=128, ch_mult=(1, 2, 4, 4), z=4, interp=None):
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
    from oracle.make_golden import model_yaml
    cfg = model_yaml(version=version, reg=reg, ch=ch, ch_mult=ch_mult, z=z, interp=interp)
    cfg["params"]["decoder_config"]["params"] = dict(cfg["params"]["encoder_config"]["params"])
    return cfg


def build(cfg, seed=0):
    from vidtok_b200.compat_util import instantiate_from_config
    from vidtok_b200.synth import synth_state_dict
    model = instantiate_from_config(cfg)
    sd = synth_state_dict({k: tuple(v.shape) for k, v in model.state_dict().items()}, seed=seed)
    model.load_state_dict(sd)
    return model.cuda().eval(), sd


def oracle_for(cfg, sd):
    from oracle.vidtok_oracle import OracleModel, cfg_from_model_yaml
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    return OracleModel(cfg_from_model_yaml(cfg), sd)


def launches_of(fn):
    """run fn() under the library's per-launch profiler -> (result, {kernel: launches})"""
    import ctypes as C
    import json
    from vidtok_b200 import _native as N
    lib = N.lib()
    lib.vt_profile_start()
    out = fn()
    buf = C.create_string_buffer(1 << 16)
    n = lib.vt_profile_stop(buf, len(buf))
    prof = json.loads(buf.value.decode()) if n > 0 else {}
    return out, {k: v["launches"] for k, v in prof.items()}


def psnr(x, y):
    from vidtok_b200.dist import psnr_partial
    p = psnr_partial(x, y)
    return float(p[0] / p[1])


def test_config2_kl_488_one_clip_vs_oracle_and_batch8_properties():
    """configs[1]: vidtok_kl_causal_488_4chn, 17x256x256.  One clip against the oracle (EXACT <= 1e-3, BF16 PSNR within
    0.01 dB), then batch 8: the clip's result does not depend on its batch neighbours, and two runs are bit-identical."""
    from vidtok_b200.synth import synth_clip
    cfg = make_cfg()
    model, sd = build(cfg)
    x8 = synth_clip(8, 17, 256, 256)
    x1 = x8[:1]
    torch.manual_seed(4321)
    z_o, dec_o, _ = oracle_for(cfg, sd).forward(x1)
    with torch.no_grad():
        model.precision = "exact"
        torch.manual_seed(4321)
        (z_e, dec_e, _), ln = launches_of(lambda: model(x1.cuda()))
        dz, dd = float((z_e.cpu() - z_o).abs().max()), float((dec_e.cpu() - dec_o).abs().max())
        print(f"[config2] exact (fp16x3 wgmma) vs oracle: max|dz|={dz:.2e} max|ddec|={dd:.2e}; launches {ln}")
        assert dz <= 1e-3 and dd <= 1e-3
        assert ln.get("conv_tc3", 0) >= 100 and ln.get("conv_simt", 0) <= 1 and "conv_tc" not in ln, ln
        model.precision = "bf16"
        torch.manual_seed(4321)
        z_b, dec_b, _ = model(x1.cuda())
        p_b, p_o = psnr(x1, dec_b.cpu()), psnr(x1, dec_o)
        print(f"[config2] bf16 PSNR {p_b:.4f} vs oracle {p_o:.4f}; max|ddec|={float((dec_b.cpu() - dec_o).abs().max()):.3f}")
        assert abs(p_b - p_o) <= 0.01
        assert float((dec_b.cpu() - dec_o).abs().max()) <= 0.25
        # batch 8 (the bench workload)
        torch.manual_seed(99)
        noise = torch.randn(8, 4, 5, 32, 32)
        torch.manual_seed(99)
        za, da, _ = model(x8.cuda())
        torch.manual_seed(99)
        zb, db, _ = model(x8.cuda())
        assert torch.equal(za, zb) and torch.equal(da, db), "two identical runs differ"
        # clip 3 alone with the noise slice it saw inside the batch
        nat = model._rt.sync()
        from vidtok_b200 import _native as N
        z3, _, _, _ = nat.encode(x8[3:4].cuda().contiguous(), noise[3:4].cuda().contiguous(), N.PREC_BF16)
        d3 = nat.decode(z3, False, N.PREC_BF16)
        assert torch.equal(z3, za[3:4]) and torch.equal(d3, da[3:4]), "a clip's result depends on its batch neighbours"
        assert torch.isfinite(da).all()


def test_config3_fsq_488_codes_equal_at_full_size():
    """configs[2]: vidtok_fsq_causal_488_32768, 17x256x256: indices of the exact mode (fp16x3 on wgmma, asserted through
    the launch profile) equal the oracle's on two clips (raw mismatches reported; none allowed outside the 1e-4 tie guard
    band); the mixed mode (exact encoder, bf16 decoder) reproduces those indices bit for bit on the 8-clip batch;
    decode(indices) == decode(codes)."""
    from vidtok_b200.synth import synth_clip
    cfg = make_cfg(reg="fsq", z=5)
    model, sd = build(cfg)
    x8 = synth_clip(8, 17, 256, 256)
    om = oracle_for(cfg, sd)
    z_o, log_o, h_o = om.encode(x8[:2], return_pre=True)
    with torch.no_grad():
        model.precision = "exact"
        (z, log), ln = launches_of(lambda: model.encode(x8[:2].cuda(), return_reg_log=True))
        assert ln.get("conv_tc3", 0) >= 40 and ln.get("conv_simt", 0) == 0 and "conv_tc" not in ln, ln
        idx = log["indices"].cpu()
        bad = idx != log_o["indices"]
        pre = log_o["pre_round"]
        near = ((pre - pre.floor() - 0.5).abs() < 1e-4).any(dim=-1)
        print(f"[config3] exact (wgmma) FSQ raw mismatches {int(bad.sum())}/{bad.numel()} (outside tie band: {int((bad & ~near).sum())})")
        assert not (bad & ~near).any()
        assert int(bad.sum()) <= 2
        assert idx.dtype == torch.int32 and tuple(idx.shape) == (2, 5, 32, 32)
        if int(bad.sum()) == 0:
            assert torch.equal(z.cpu(), z_o)
        # the throughput configuration with exact codes: encoder fp16x3, decoder bf16
        model.precision = "mixed"
        (z8, dec8, log8), ln = launches_of(lambda: model(x8.cuda()))
        assert ln.get("conv_tc3", 0) >= 40 and ln.get("conv_tc", 0) >= 60, ln
        # same encoder arithmetic; a different batch size may pick a different tile plan (tap order of the K loop), so compare
        # against the oracle with the same criterion instead of bit-wise against the 2-clip run
        bad8 = log8["indices"][:2].cpu() != log_o["indices"]
        print(f"[config3] mixed (8 clips) FSQ raw mismatches on clips 0-1: {int(bad8.sum())}/{bad8.numel()} (outside tie band: {int((bad8 & ~near).sum())})")
        assert not (bad8 & ~near).any() and int(bad8.sum()) <= 2
        d_idx = model.decode(log8["indices"], decode_from_indices=True)
        assert torch.equal(dec8, d_idx)
        assert int(log8["indices"].min()) >= 0 and int(log8["indices"].max()) < 32768 and torch.isfinite(dec8).all()
        model.precision = "bf16"
        z8b, log8b = model.encode(x8[:2].cuda(), return_reg_log=True)
        mism = int((log8b["indices"].cpu() != log_o["indices"]).sum())
        print(f"[config3] bf16 FSQ mismatches on 2 clips: {mism}/{log_o['indices'].numel()} (informational: the reference's own bf16 run flips 3.75 %)")


def test_config4_v11_long_video_tiled():
    """configs[3]: vidtok_kl_causal_488_16chn v1.1, tiled t_chunk_enc=16 with overlap.  65x128x128 against the oracle
    (same chunk schedule), then 129x256x256: tiled encode == untiled encode (the survey's invariant), shapes, finiteness."""
    from vidtok_b200.synth import synth_clip
    cfg = make_cfg(version="v1_1", z=16, interp="trilinear")
    model, sd = build(cfg)
    model.use_tiling, model.t_chunk_enc, model.t_chunk_dec, model.use_overlap = True, 16, 4, True
    x = synth_clip(1, 65, 128, 128)
    om = oracle_for(cfg, sd)
    om.use_tiling, om.t_chunk_enc, om.t_chunk_dec, om.use_overlap = True, 16, 4, True
    torch.manual_seed(4321)
    z_o, dec_o, _ = om.forward(x)
    with torch.no_grad():
        model.precision = "exact"
        torch.manual_seed(4321)
        z_e, dec_e, _ = model(x.cuda())
        dz, dd = float((z_e.cpu() - z_o).abs().max()), float((dec_e.cpu() - dec_o).abs().max())
        print(f"[config4] 65x128x128 tiled exact vs oracle: max|dz|={dz:.2e} max|ddec|={dd:.2e}")
        assert dec_e.shape == x.shape and dz <= 1e-3 and dd <= 1e-3
        model.precision = "bf16"
        torch.manual_seed(4321)
        _, dec_b, _ = model(x.cuda())
        assert abs(psnr(x, dec_b.cpu()) - psnr(x, dec_o)) <= 0.01
        # full size
        xl = synth_clip(1, 129, 256, 256, seed=7)
        torch.manual_seed(1)
        z_t, dec_t, _ = model(xl.cuda())
        assert tuple(z_t.shape) == (1, 16, 33, 32, 32) and dec_t.shape == xl.shape and torch.isfinite(dec_t).all()
        # frames 0..16 come from decoder chunks [0,1] and [1,5] (+1 look-ahead latent), which see latents 0..5 only: the
        # tiled oracle on the 33-frame prefix produces the same 17 frames (same chunk schedule, same look-ahead)
        torch.manual_seed(1)
        z_p, dec_p, _ = om.forward(xl[:, :, :33])
        p_b, p_o = psnr(xl[:, :, :17], dec_t[:, :, :17].cpu()), psnr(xl[:, :, :17], dec_p[:, :, :17])
        dmax = float((dec_t[:, :, :17].cpu() - dec_p[:, :, :17]).abs().max())
        print(f"[config4] 129x256x256 bf16, first 17 frames vs tiled oracle: PSNR {p_b:.4f} vs {p_o:.4f}, max|d|={dmax:.3f}")
        assert abs(p_b - p_o) <= 0.01 and dmax <= 0.25
        model.precision = "exact"
        torch.manual_seed(1)
        z_x, dec_x, _ = model(xl[:, :, :33].cuda())
        dz, dd = float((z_x.cpu() - z_p).abs().max()), float((dec_x.cpu() - dec_p).abs().max())
        print(f"[config4] 33x256x256 tiled exact vs oracle: max|dz|={dz:.2e} max|ddec|={dd:.2e}")
        assert dz <= 1e-3 and dd <= 1e-3
    # tiled encode == untiled encode (SURVEY 0.9: 1.5e-6 in the reference) on the deterministic posterior mode
    cfg_m = make_cfg(version="v1_1", z=16, interp="trilinear")
    cfg_m["params"]["regularizer_config"]["params"] = {"sample": False}
    model_m, _ = build(cfg_m)
    model_m.t_chunk_enc, model_m.t_chunk_dec, model_m.use_overlap = 16, 4, True
    xs = xl[:, :, :49].cuda()
    with torch.no_grad():
        for prec, tol in (("exact", 5e-5), ("bf16", 0.08)):   # different chunk shapes -> different tile plans (accumulation order)
            model_m.precision = prec
            model_m.use_tiling = True
            z_tiled = model_m.encode(xs)
            model_m.use_tiling = False
            z_untiled = model_m.encode(xs)
            dt = float((z_tiled - z_untiled).abs().max())
            print(f"[config4] {prec}: max|z_tiled - z_untiled| = {dt:.2e} over {tuple(z_tiled.shape)}")
            assert tuple(z_tiled.shape) == (1, 16, 13, 32, 32) and dt <= tol, (prec, dt)


def test_config5_41616_high_res():
    """configs[4]: vidtok_kl_causal_41616_4chn.  17x128x128 against the oracle, then 4 clips of 17x512x512 (one GPU's
    share of the 32-clip batch): EXACT-vs-BF16 PSNR agreement and finiteness."""
    from vidtok_b200.synth import synth_clip
    cfg = make_cfg(ch_mult=(1, 2, 4, 4, 4))
    model, sd = build(cfg)
    x = synth_clip(1, 17, 128, 128)
    torch.manual_seed(4321)
    z_o, dec_o, _ = oracle_for(cfg, sd).forward(x)
    with torch.no_grad():
        model.precision = "exact"
        torch.manual_seed(4321)
        z_e, dec_e, _ = model(x.cuda())
        dz, dd = float((z_e.cpu() - z_o).abs().max()), float((dec_e.cpu() - dec_o).abs().max())
        print(f"[config5] 128x128 exact vs oracle: max|dz|={dz:.2e} max|ddec|={dd:.2e}")
        assert tuple(z_e.shape) == (1, 4, 5, 8, 8) and dz <= 1e-3 and dd <= 1e-3
        # one 17x256x256 clip against the oracle in both modes
        x2 = synth_clip(1, 17, 256, 256, seed=11)
        torch.manual_seed(4321)
        z_o2, dec_o2, _ = oracle_for(cfg, sd).forward(x2)
        torch.manual_seed(4321)
        z_e2, dec_e2, _ = model(x2.cuda())
        dz, dd = float((z_e2.cpu() - z_o2).abs().max()), float((dec_e2.cpu() - dec_o2).abs().max())
        print(f"[config5] 256x256 exact vs oracle: max|dz|={dz:.2e} max|ddec|={dd:.2e}")
        assert dz <= 1e-3 and dd <= 1e-3
        model.precision = "bf16"
        torch.manual_seed(4321)
        _, dec_b2, _ = model(x2.cuda())
        assert abs(psnr(x2, dec_b2.cpu()) - psnr(x2, dec_o2)) <= 0.01 and float((dec_b2.cpu() - dec_o2).abs().max()) <= 0.25
        xb = synth_clip(4, 17, 512, 512, seed=5).cuda()
        torch.manual_seed(3)
        zb, db, _ = model(xb)
        assert tuple(zb.shape) == (4, 4, 5, 32, 32) and db.shape == xb.shape and torch.isfinite(db).all()
        model.precision = "exact"
        torch.manual_seed(3)
        ze, de, _ = model(xb[:1])
        p_b, p_e = psnr(xb[:1].cpu(), db[:1].cpu()), psnr(xb[:1].cpu(), de.cpu())
        print(f"[config5] 512x512 PSNR bf16 {p_b:.4f} vs exact {p_e:.4f}; max|d|={float((db[:1] - de).abs().max()):.3f}")
        assert abs(p_b - p_e) <= 0.01
