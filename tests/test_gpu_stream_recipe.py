"""-m gpu: the reference's long-video recipe through streams (EncodeStream(t_chunk), DecodeStream(t_chunk, use_overlap)).

A stream with t_chunk runs the chunks of tile_encode / tile_decode whatever sizes the frames arrive in, on the same chunk
states and kernels, so its latents, indices, kl_loss and reconstructions are bitwise those of the tile paths in every
precision mode, and its values are the reference's long-video values (the fixtures were written by the unmodified
reference with use_overlap=True at meta["tiling_chunk"])."""
import itertools

import pytest
import torch

pytestmark = pytest.mark.gpu

from conftest import load_golden, resolved_model_cfg, synth_inputs, synth_weights  # noqa: E402
from test_fsq_aux_cpu import load_aux  # noqa: E402
from test_gpu_fsq_aux import E2E_BOUND, rel  # noqa: E402
from test_gpu_model import TOL, fsq_guard  # noqa: E402
from test_gpu_stream import SCHEDULES  # noqa: E402
from vidtok_b200 import _native as N  # noqa: E402


def _model(case, mode):
    from vidtok_b200.compat_util import instantiate_from_config
    d, meta = load_golden(case)
    model = instantiate_from_config(resolved_model_cfg(meta))
    missing, unexpected = model.load_state_dict(synth_weights(meta, d), strict=False)
    assert not missing and not unexpected
    model = model.to("cuda").eval()
    model.precision = mode
    return d, meta, model


def _ragged(T):
    out, sizes = [], itertools.cycle((3, 1, 7, 16, 2, 5))
    while sum(out) < T:
        out.append(min(next(sizes), T - sum(out)))
    return out


def _schedules(T):
    return {"ones": [1] * T, "all": [T], "ragged": _ragged(T)}


def _stream_encode(model, x, t_chunk, sched):
    """pushes, then flush -> (z, indices or None, reg_log of the flush)"""
    from vidtok_b200.streaming import EncodeStream
    B, _, T, H, W = x.shape
    enc = EncodeStream(model, B, H, W, t_chunk=t_chunk)
    zs, idx, t0 = [], [], 0
    for n in sched + [None]:
        z, log = enc.flush() if n is None else enc.push(x[:, :, t0:t0 + n])
        zs.append(z)
        if "indices" in log:
            idx.append(log["indices"])
        t0 += n or 0
    enc.close()
    return torch.cat(zs, dim=2), (torch.cat(idx, dim=1) if idx else None), log


def _stream_decode(model, z, t_chunk, use_overlap, sched):
    from vidtok_b200.streaming import DecodeStream
    dec = DecodeStream(model, z.shape[0], z.shape[3], z.shape[4], t_chunk=t_chunk, use_overlap=use_overlap)
    outs, t0 = [], 0
    for n in sched:
        outs.append(dec.push(z[:, :, t0:t0 + n]))
        t0 += n
    outs.append(dec.flush())
    dec.close()
    return torch.cat(outs, dim=2)


@pytest.mark.parametrize("case", ["tiny_kl_v11_tiled", "tiny_fsq_v11_tiled"])
def test_stream_recipe_matches_reference_fixture(case):
    """Ragged pushes through the recipe streams meet the gates test_exact_mode_matches_reference_fixture applies to the
    tiled forward of the same fixtures."""
    d, meta, model = _model(case, "exact")
    x = synth_inputs(meta, d).cuda()
    T = x.shape[2]
    tc, tdf = meta["tiling_chunk"], model.encoder.time_downsample_factor
    with torch.no_grad():
        torch.manual_seed(meta["noise_seed"])
        z, idx, log = _stream_encode(model, x, tc, _ragged(T))
        dec = _stream_decode(model, z, tc // tdf, True, _ragged(z.shape[2]))
    dec = dec[:, :, -T:].cpu()   # autoencoder_v1_1.py:340-341
    z = z.cpu()
    assert tuple(z.shape) == tuple(d["z"].shape) and tuple(dec.shape) == tuple(d["dec"].shape)
    dz = float((z - torch.from_numpy(d["z"])).abs().max())
    dd = float((dec - torch.from_numpy(d["dec"])).abs().max())
    print(f"[{case}] stream recipe: max|dz|={dz:.2e} max|ddec|={dd:.2e}")
    if "indices" in d:
        idx = idx.cpu()
        if "h" in d:
            nbad, n = fsq_guard(idx, d["indices"], d["h"], meta["model"]["params"]["regularizer_config"]["params"]["levels"])
            assert nbad <= max(1, n // 2000), (nbad, n)
        else:
            assert int((idx != torch.from_numpy(d["indices"])).sum()) == 0
        if int((idx != torch.from_numpy(d["indices"])).sum()) == 0:
            assert dz == 0.0 and dd <= TOL, (dz, dd)
        _, ameta = load_aux("tiled_" + case)
        got, want = float(log["aux_loss"]), ameta["reference"]["aux_loss"]
        print(f"[{case}] stream aux_loss {got:.9g} reference {want:.9g} relative error {rel(got, want):.3e}")
        assert log["aux_loss"].is_cuda and rel(got, want) <= E2E_BOUND
    else:
        assert dz <= TOL and dd <= TOL, (dz, dd)
        assert abs(float(log["kl_loss"]) - float(d["kl_loss"])) <= 1e-4 * abs(float(d["kl_loss"]))


# (frames, t_chunk): each video ends in a shorter chunk where its length allows one
BITWISE = {"tiny_kl_v11": (27, 8), "tiny_kl_v11_tiled": (43, 16), "tiny_fsq_v11_tiled": (38, 16), "tiny_fsq_888_v11": (27, 8)}


@pytest.mark.parametrize("mode", ["bf16", "fma", "exact"])
@pytest.mark.parametrize("case", list(BITWISE))
def test_stream_recipe_equals_tile_paths(case, mode):
    from vidtok_b200.synth import synth_clip
    d, meta, model = _model(case, mode)
    B, _, _, H, W = meta["input"]
    T, tc = BITWISE[case]
    tdf = model.encoder.time_downsample_factor
    x = synth_clip(B, T, H, W, seed=meta["input_seed"]).cuda()
    model.use_tiling, model.t_chunk_enc, model.t_chunk_dec = True, tc, tc // tdf
    nat = model._rt.sync()
    with torch.no_grad():
        torch.manual_seed(11)
        z_t, log_t = model.tile_encode(x)
        Tz = z_t.shape[2]
        x_t = {}
        for ov in (True, False):
            model.use_overlap = ov
            x_t[ov] = model.tile_decode(z_t)
        for name, sched in _schedules(T).items():
            torch.manual_seed(11)
            z, idx, log = _stream_encode(model, x, tc, sched)
            assert torch.equal(z, z_t), (name, float((z - z_t).abs().max()))
            if "indices" in log_t:
                assert torch.equal(idx, log_t["indices"]), name
                got, want = float(log["aux_loss"]), float(log_t["aux_loss"])
                assert rel(got, want) <= 1e-6, (name, got, want)
            else:
                assert torch.equal(log["kl_loss"], log_t["kl_loss"]), (name, float(log["kl_loss"]), float(log_t["kl_loss"]))
        for name, sched in _schedules(Tz).items():
            for ov in (True, False):
                xs = _stream_decode(model, z_t, tc // tdf, ov, sched)
                assert xs.shape[2] == nat.lib.vt_decode_video_frames(nat.handle, Tz, tc // tdf, int(ov)), (name, ov)
                assert torch.equal(xs, x_t[ov]), (name, ov, float((xs - x_t[ov]).abs().max()) if xs.shape == x_t[ov].shape else xs.shape)


@pytest.mark.parametrize("mode", ["bf16", "fma", "exact"])
@pytest.mark.parametrize("case", ["tiny_fsq_v10", "mid_fsq_v10"])
def test_v10_stream_aux_loss_is_the_whole_clips(case, mode):
    """A v1.0 stream's aux_loss treats all its tokens as one segment, as encode(whole) does.  In bf16 and fma the streamed
    pre-bound latents are the whole clip's bit for bit and so is the aux_loss (measured); exact's latents differ by fp32
    rounding (see test_gpu_stream), which moved mid_fsq_v10's aux_loss by 4.4e-7 relative (H100)."""
    from vidtok_b200.streaming import EncodeStream
    d, meta, model = _model(case, mode)
    x = synth_inputs(meta, d).cuda()
    B, _, _, H, W = x.shape
    _, ameta = load_aux("fix_" + case)
    with torch.no_grad():
        _, log_w = model.encode(x, return_reg_log=True)
        want = float(log_w["aux_loss"])
        for name, sched in SCHEDULES.items():
            enc = EncodeStream(model, B, H, W)
            t0 = 0
            for n in sched:
                _, log = enc.push(x[:, :, t0:t0 + n])
                t0 += n
            enc.close()
            got = float(log["aux_loss"])
            print(f"[{case} {mode} {name}] stream aux {got:.9g} whole clip {want:.9g} rel {rel(got, want):.3e} "
                  f"reference rel {rel(got, ameta['reference']['aux_loss']):.3e}")
            assert rel(got, want) <= 1e-6, (name, got, want)
            if mode == "exact":
                assert rel(got, ameta["reference"]["aux_loss"]) <= E2E_BOUND, (name, got)


def _refused(lib, fn, exc):
    lib.vt_launch_count(1)
    with pytest.raises(exc):
        fn()
    assert lib.vt_launch_count(1) == 0


def test_refusals_launch_nothing():
    from vidtok_b200.engine import _ptr, _stream_ptr
    from vidtok_b200.streaming import DecodeStream, EncodeStream
    lib = N.lib()
    _, _, v10 = _model("tiny_fsq_v10", "bf16")
    _, meta, v11 = _model("tiny_fsq_v11_tiled", "bf16")
    _, _, kl = _model("tiny_kl_v11", "bf16")
    for m in (v10, v11, kl):
        m._rt.sync()
    B, _, _, H, W = meta["input"]
    _refused(lib, lambda: EncodeStream(v10, B, H, W, t_chunk=16), ValueError)
    _refused(lib, lambda: DecodeStream(v10, B, 4, 4, t_chunk=4), ValueError)
    _refused(lib, lambda: DecodeStream(v11, B, 4, 4, use_overlap=True), ValueError)
    _refused(lib, lambda: DecodeStream(v10, B, 4, 4, use_overlap=True), ValueError)
    _refused(lib, lambda: EncodeStream(v11, B, H, W, t_chunk=6), ValueError)
    x = torch.zeros((B, 3, 5, H, W), device="cuda")
    with torch.no_grad():
        enc = EncodeStream(v11, B, H, W, t_chunk=16)
        z, _ = enc.push(x)
        z2, _ = enc.flush()
        _refused(lib, lambda: enc.push(x), RuntimeError)
        _refused(lib, lambda: enc.flush(), RuntimeError)
        enc.reset()
        assert torch.equal(enc.push(x)[0], z)
        z = torch.cat([z, z2], dim=2)
        dec = DecodeStream(v11, B, z.shape[3], z.shape[4], t_chunk=4, use_overlap=True)
        dec.push(z)
        dec.flush()
        _refused(lib, lambda: dec.push(z), RuntimeError)
        dec.reset()
        dec.push(z)
        enc.close()
        dec.close()
        # vt_encode_chunk_fsq_aux on a KL model: VT_ERR_INVALID before any launch
        enc = EncodeStream(kl, B, H, W)
        ws = enc.state.workspace(1)
        zc = torch.empty((B, 4, 1, enc.Hz, enc.Wz), device="cuda")
        stats, avg = torch.empty(2, device="cuda"), torch.empty(32768, device="cuda")
        lib.vt_launch_count(1)
        rc = lib.vt_encode_chunk_fsq_aux(enc.state.handle, 1, _ptr(x[:, :, :1].contiguous()), 3, 1, _ptr(zc), None, 100.0, _ptr(stats),
                                         _ptr(avg), _ptr(ws), ws.numel(), _stream_ptr(x.device))
        assert rc == -1 and b"FSQ model" in lib.vt_last_error(), (rc, lib.vt_last_error())
        assert lib.vt_launch_count(1) == 0
        enc.close()
