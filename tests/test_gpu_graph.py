"""-m gpu: the tokenizer inside CUDA graphs.

Whole clips: model(x), encode and decode (latents and FSQ indices) captured in the caller's torch.cuda.graph after one
eager call, replayed with new inputs and noise copied into the static tensors, equal the eager calls bit for bit.
Streams: the steady chunks of EncodeStream / DecodeStream are captured and replayed by the stream itself; the outputs stay
those of the eager streams (tile_encode / tile_decode for v1.1, the whole clip for v1.0).  Calls that cannot be captured
refuse with a clear error and leave the caller's capture and the model usable."""
import copy

import pytest
import torch

pytestmark = pytest.mark.gpu

from conftest import load_golden, resolved_model_cfg, synth_weights  # noqa: E402


def _model(case, mode, sample=True):
    from vidtok_b200.compat_util import instantiate_from_config
    d, meta = load_golden(case)
    cfg = copy.deepcopy(resolved_model_cfg(meta))
    if not sample:
        cfg["params"]["regularizer_config"]["params"] = {"sample": False}
    model = instantiate_from_config(cfg)
    missing, unexpected = model.load_state_dict(synth_weights(meta, d), strict=False)
    assert not missing and not unexpected
    model = model.to("cuda").eval()
    model.precision = mode
    return d, meta, model


def _clip(B, T, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand((B, 3, T, H, W), generator=g) * 2 - 1).cuda()


def _latent_noise(model, x, seed):
    Tz, Hz, Wz = model._rt.sync().latent_shape(*x.shape[2:])
    g = torch.Generator().manual_seed(seed)
    return torch.randn((x.shape[0], model.spec.z_channels, Tz, Hz, Wz), generator=g).cuda()


def _same(a, b):
    assert a.dtype == b.dtype and a.shape == b.shape and torch.equal(a, b)


def _same_log(a, b):
    assert a.keys() == b.keys()
    for k in a:
        _same(a[k], b[k])


@pytest.mark.parametrize("mode", ["bf16", "exact"])
@pytest.mark.parametrize("case,sample", [("tiny_kl_v10", True), ("tiny_kl_v10", False), ("tiny_fsq_v10", True),
                                         ("tiny_kl_v11", True)])
def test_whole_clip_capture_equals_eager(case, sample, mode):
    d, meta, model = _model(case, mode, sample)
    B, _, T, H, W = d["x"].shape
    kl_noise = model.spec.regularizer == "kl" and sample
    x_s = _clip(B, T, H, W, 0)
    with torch.no_grad():
        n_s = _latent_noise(model, x_s, 1) if kl_noise else None
        model(x_s, noise=n_s)                                  # the warm-up: loads the weights, sizes the workspace
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            z_g, dec_g, log_g = model(x_s, noise=n_s)
        for it in range(3):
            x = _clip(B, T, H, W, 10 + it)
            n = _latent_noise(model, x, 20 + it) if kl_noise else None
            x_s.copy_(x)
            if kl_noise:
                n_s.copy_(n)
            g.replay()
            z_e, dec_e, log_e = model(x, noise=n)
            torch.cuda.synchronize()
            _same(z_g, z_e)
            _same(dec_g, dec_e)
            _same_log(log_g, log_e)
            if model.spec.regularizer == "fsq":
                assert model.regularization.aux_enabled() and float(log_e["aux_loss"]) != 0.0


@pytest.mark.parametrize("mode", ["bf16", "exact"])
@pytest.mark.parametrize("case", ["tiny_fsq_v10", "tiny_fsq_v11_tiled"])
def test_decode_from_indices_capture_equals_eager(case, mode):
    d, meta, model = _model(case, mode)
    if hasattr(model, "use_tiling"):
        model.use_tiling = False
    B, _, _, H, W = d["x"].shape
    T = 17
    with torch.no_grad():
        idx_s = model.encode(_clip(B, T, H, W, 0), return_reg_log=True)[1]["indices"].clone()
        model.decode(idx_s, decode_from_indices=True)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            dec_g = model.decode(idx_s, decode_from_indices=True)
        for it in range(3):
            idx = model.encode(_clip(B, T, H, W, 5 + it), return_reg_log=True)[1]["indices"]
            idx_s.copy_(idx)
            g.replay()
            _same(dec_g, model.decode(idx, decode_from_indices=True))


def _encode_pushes(enc, x, sizes, noise_for=None):
    """x pushed in `sizes` frames, then flushed -> (z, indices or None, last reg_log)"""
    zs, idx, t0, log = [], [], 0, None
    for i, n in enumerate(sizes + [None]):
        if n is None:
            z, log = enc.flush()
        else:
            kw = {"noise": noise_for(i)} if noise_for else {}
            z, log = enc.push(x[:, :, t0:t0 + n], **kw)
            t0 += n
        zs.append(z)
        if "indices" in log:
            idx.append(log["indices"])
    return torch.cat(zs, dim=2), (torch.cat(idx, dim=1) if idx else None), log


def _decode_pushes(dec, z, n):
    outs = [dec.push(z[:, :, t0:t0 + n]) for t0 in range(0, z.shape[2], n)]
    outs.append(dec.flush())
    return torch.cat(outs, dim=2)


def _check_replays(stream, min_replays=4):
    """every graph key of the stream replayed at least min_replays times, at both cache parities"""
    keys = list(stream.graphs.graphs)
    assert keys, "no chunk was captured"
    for k in keys:
        assert stream.graphs.runs[k] >= min_replays, (k, dict(stream.graphs.runs))
    assert {k[2] for k in keys} == {0, 1}, keys


@pytest.mark.parametrize("case", ["tiny_kl_v10", "tiny_fsq_v10"])
def test_v10_streams_replay_equal_whole_clip(case):
    from vidtok_b200.streaming import DecodeStream, EncodeStream
    d, meta, model = _model(case, "bf16")
    B, _, _, H, W = d["x"].shape
    n_groups = 14
    T = 1 + 4 * n_groups
    kl = model.spec.regularizer == "kl"
    with torch.no_grad():
        enc = dec = None
        for video in range(2):   # the second video after reset() replays the graphs the first one captured
            x = _clip(B, T, H, W, 100 + video)
            noise = _latent_noise(model, x, 200 + video) if kl else None
            z_w, log_w = model.encode(x, return_reg_log=True, noise=noise)
            dec_w = model.decode(z_w)
            if enc is None:
                enc = EncodeStream(model, B, H, W)
                dec = DecodeStream(model, B, z_w.shape[3], z_w.shape[4])
            else:
                enc.reset()
                dec.reset()
            # frame 0 is the first chunk; each later push of 4 frames is one chunk of one latent frame
            z_s, idx_s, _ = _encode_pushes(enc, x, [1] + [4] * n_groups,
                                           (lambda i: noise[:, :, i:i + 1]) if kl else None)
            _same(z_s, z_w)
            if not kl:
                _same(idx_s, log_w["indices"])
            _same(_decode_pushes(dec, z_w, 1), dec_w)
        _check_replays(enc)
        _check_replays(dec)


@pytest.mark.parametrize("mode", ["bf16", "exact"])
@pytest.mark.parametrize("case", ["tiny_kl_v11_tiled", "tiny_fsq_v11_tiled"])
def test_v11_recipe_streams_replay_equal_tile_paths(case, mode):
    from vidtok_b200.streaming import DecodeStream, EncodeStream
    d, meta, model = _model(case, mode)
    B, _, _, H, W = d["x"].shape
    tdf = model.encoder.time_downsample_factor
    model.t_chunk_enc, model.t_chunk_dec = 2 * tdf, 2
    model.use_overlap = True
    n_chunks = 14
    T = 1 + 2 * tdf * n_chunks
    with torch.no_grad():
        enc = dec = None
        for video in range(2):
            x = _clip(B, T, H, W, 300 + video)
            torch.manual_seed(7 + video)
            z_t, log_t = model.tile_encode(x)
            x_t = model.tile_decode(z_t)
            if enc is None:
                enc = EncodeStream(model, B, H, W, t_chunk=model.t_chunk_enc)
                dec = DecodeStream(model, B, z_t.shape[3], z_t.shape[4], t_chunk=2, use_overlap=True)
            else:
                enc.reset()
                dec.reset()
            torch.manual_seed(7 + video)   # the stream draws the KL noise per chunk in tile_encode's order
            z_s, idx_s, log_s = _encode_pushes(enc, x, [1] + [2 * tdf] * n_chunks)
            _same(z_s, z_t)
            if "indices" in log_t:
                _same(idx_s, log_t["indices"])
                _same(log_s["aux_loss"], log_t["aux_loss"])
            else:
                _same(log_s["kl_loss"], log_t["kl_loss"])
            _same(_decode_pushes(dec, z_t, 1), x_t)
        _check_replays(enc)
        _check_replays(dec)


def test_replayed_push_does_no_host_synchronisation():
    from vidtok_b200.streaming import DecodeStream, EncodeStream
    d, meta, model = _model("tiny_fsq_v10", "bf16")
    B, _, _, H, W = d["x"].shape
    x = _clip(B, 1 + 4 * 8, H, W, 0)
    with torch.no_grad():
        enc = EncodeStream(model, B, H, W)
        zs = [enc.push(x[:, :, :1])[0]] + [enc.push(x[:, :, 1 + 4 * i:5 + 4 * i])[0] for i in range(6)]
        z = torch.cat(zs, dim=2)
        dec = DecodeStream(model, B, z.shape[3], z.shape[4])
        for t in range(6):
            dec.push(z[:, :, t:t + 1])
        torch.cuda.synchronize()
        assert enc.graphs.graphs and dec.graphs.graphs
        before = (enc.graphs.replays, dec.graphs.replays)
        torch.cuda.set_sync_debug_mode("error")
        try:
            enc.push(x[:, :, 25:29])
            dec.push(z[:, :, 6:7])
        finally:
            torch.cuda.set_sync_debug_mode(0)
        assert (enc.graphs.replays, dec.graphs.replays) == (before[0] + 1, before[1] + 1)


def _refused(fn, match):
    g = torch.cuda.CUDAGraph()
    with pytest.raises(RuntimeError, match=match):
        with torch.cuda.graph(g):
            fn()


def test_refusals_leave_the_model_usable():
    from vidtok_b200.streaming import EncodePool
    d, meta, model = _model("tiny_kl_v10", "bf16")
    B, _, T, H, W = d["x"].shape
    x = _clip(B, T, H, W, 0)
    with torch.no_grad():
        torch.manual_seed(1)
        want = model(x)
        # KL sampling without noise=: the CPU generator cannot be captured
        _refused(lambda: model(x), "noise=")
        torch.manual_seed(1)
        got = model(x)
        for a, b in zip(want[:2], got[:2]):
            _same(a, b)
        _same_log(want[2], got[2])

        # a capture before any eager call of the model: nothing is loaded, the workspace is not sized
        _, _, fresh = _model("tiny_kl_v10", "bf16")
        n = _latent_noise(model, x, 3)
        _refused(lambda: fresh.encode(x, noise=n), "eager call")
        _same(fresh.encode(x, noise=n), model.encode(x, noise=n))
        # a geometry the workspace was not sized for
        x_big = _clip(B, T, 2 * H, 2 * W, 4)
        n_big = _latent_noise(model, x_big, 5)
        _refused(lambda: model.encode(x_big, noise=n_big), "warm|eager")
        model.encode(x_big, noise=n_big)

        # a pool step: slot transplants upload host tables
        pool = EncodePool(model, capacity=2, H=H, W=W, t_chunk=4)
        a = pool.open()
        pool.push(a, x[:1, :, :5])
        _refused(pool.step, "cannot be captured")
        assert set(pool.step()) == {a}

    _, _, m11 = _model("tiny_kl_v11_tiled", "bf16")
    m11.use_tiling = True
    x11 = _clip(1, 33, 32, 32, 6)
    with torch.no_grad():
        torch.manual_seed(2)
        z_want = m11.tile_encode(x11)[0]
        _refused(lambda: m11.tile_encode(x11), "cannot be captured")
        _refused(lambda: m11.tile_decode(z_want), "cannot be captured")
        torch.manual_seed(2)
        _same(m11.tile_encode(x11)[0], z_want)
