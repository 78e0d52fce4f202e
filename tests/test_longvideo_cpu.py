"""CPU checks of long-video sharding: the temporal reach vt_temporal_reach reports is the reach the float64 oracle shows under
the tile_encode / tile_decode chunking (a true bound, and a tight one), the shard plan's arithmetic, and the refusals."""
import ctypes as C

import pytest
import torch

from conftest import load_golden, resolved_model_cfg

V11 = ["tiny_kl_v11_tiled", "tiny_fsq_v11_tiled", "tiny_fsq_888_v11", "tiny_kl_v11"]


def _native(meta):
    from vidtok_b200.compat_util import instantiate_from_config
    from vidtok_b200.engine import NativeModel
    return NativeModel(instantiate_from_config(resolved_model_cfg(meta)).spec)


def _latest_changed(a, b):
    diff = (a - b).abs().amax(dim=tuple(i for i in range(a.dim()) if i != 2))
    return int((diff > 0).nonzero().flatten().max())


@pytest.mark.parametrize("case", V11)
def test_reach_is_the_oracles_reach(case):
    """Perturb input frame j (latent j): no output past j + R changes, and for some j the output at j + R does."""
    from oracle.vidtok_oracle import OracleModel, cfg_from_model_yaml
    from vidtok_b200.longvideo import temporal_reach
    from vidtok_b200.synth import synth_state_dict
    d, meta = load_golden(case)
    nm = _native(meta)
    cfg = cfg_from_model_yaml(meta["model"])
    tdf = cfg.time_downsample_factor
    sd = synth_state_dict({k: tuple(v) for k, v in meta["shapes"].items()}, seed=meta["weights_seed"])
    om = OracleModel(cfg, sd, dtype=torch.float64)
    om.use_tiling, om.t_chunk_enc, om.t_chunk_dec = True, 2 * tdf, 2
    g = torch.Generator().manual_seed(0)
    # encoder: on the pre-bound latent (FSQ rounding would hide small far-reaching changes)
    R = temporal_reach(nm, False)
    c = om.t_chunk_enc
    T = 1 + c * ((R + 3 * c) // c)
    x = torch.randn((1, 3, T, 16, 16), generator=g, dtype=torch.float64)
    enc = lambda v: om.encode(v, noise_fn=lambda s: torch.zeros(s, dtype=torch.float64), return_pre=True)[2]
    h0, worst = enc(x), []
    for j in range(1, c + 2):
        x1 = x.clone()
        x1[:, :, j] += 1.0
        l = _latest_changed(enc(x1), h0)
        assert l < h0.shape[2] - 1, "the video is too short to see the reach"
        worst.append(1 + (l - 1) * tdf - j)
    assert max(worst) == R, (worst, R)
    for ov in (False, True):
        om.use_overlap = ov
        R = temporal_reach(nm, True, ov)
        Tz = 1 + 2 * ((R + 8) // 2)
        z = torch.randn((1, cfg.z_channels, Tz, 2, 2), generator=g, dtype=torch.float64)
        y0, worst = om.decode(z), []
        for j in range(0, 6):
            z1 = z.clone()
            z1[:, :, j] += 0.5
            t = _latest_changed(om.decode(z1), y0)
            assert t < y0.shape[2] - tdf
            worst.append(t // tdf - j)
        assert max(worst) == R, (ov, worst, R)


def _ask(nm, dec, ov):
    from vidtok_b200 import _native as N
    r = C.c_int32()
    return N.lib().vt_temporal_reach(nm.handle, dec, ov, C.byref(r)), r.value


def test_reach_refusals():
    from vidtok_b200 import _native as N
    for case, why in (("tiny_kl_v10", b"v1.1 model family"), ("tiny_kl_nc", b"non-causal")):
        d, meta = load_golden(case)
        rc, _ = _ask(_native(meta), 0, 0)
        assert rc != 0 and why in N.lib().vt_last_error()
    d, meta = load_golden("tiny_kl_v11")
    rc, _ = _ask(_native(meta), 0, 1)
    assert rc != 0 and b"decoder option" in N.lib().vt_last_error()


@pytest.mark.parametrize("lookahead", [False, True])
def test_shard_plan_arithmetic(lookahead):
    from vidtok_b200.longvideo import chunk_start_end, shard_plan
    seen = 0
    for c in (1, 2, 4, 8, 16):
        for R in (0, 1, 5, 46, 109):
            for T in list(range(1, 90, 7)) + [257, 513, 1025]:
                for S in (1, 2, 3, 5, 8):
                    try:
                        p = shard_plan(T, S, c, R, lookahead=lookahead)
                    except ValueError as e:
                        assert S > 1 and "shards need" in str(e)
                        continue
                    seen += 1
                    assert p.chunks == chunk_start_end(T, c)
                    # owned chunks partition the video's chunks, in order
                    assert [o for a, b in p.owned for o in range(a, b)] == list(range(len(p.chunks)))
                    assert all(b > a for a, b in p.owned)
                    for i, s in enumerate(p.starts):
                        assert s % c == 0 and 0 <= s and s + p.window <= T          # on the grid, inside the video
                        a, b = p.keep[i]
                        assert p.chunks[p.owned[i][0]][0] == s + a and p.chunks[p.owned[i][1] - 1][1] == s + b
                        if i:
                            assert a - 1 >= R                                   # warm-up after the window's first frame
                        if i < S - 1:
                            # a kept chunk is never the window's last one (short, or decoded without look-ahead)
                            last = chunk_start_end(p.window, c)[-1]
                            short = last[1] - last[0] < c and len(chunk_start_end(p.window, c)) > 1
                            assert b <= (last[0] if (lookahead or short) else last[1])
                    assert p.starts[-1] + p.window == T                         # the last window sees the end
                    assert 0 <= p.warmup_fraction < 1
    assert seen > 500


def test_shard_plan_refuses_too_many_shards():
    from vidtok_b200.longvideo import shard_plan
    with pytest.raises(ValueError, match="shards need"):
        shard_plan(1 + 16 * 8, 3, 16, 109)


def test_sharded_calls_refuse_v10_and_noncausal_models():
    from vidtok_b200.compat_util import instantiate_from_config
    from vidtok_b200.longvideo import decode_sharded, encode_sharded
    for case, why in (("tiny_kl_v10", "v1.1"), ("tiny_kl_nc", "non-causal")):
        d, meta = load_golden(case)
        model = instantiate_from_config(resolved_model_cfg(meta))
        with pytest.raises(ValueError, match=why):
            encode_sharded(model, torch.zeros(1, 3, 17, 16, 16), 2)
        with pytest.raises(ValueError, match=why):
            decode_sharded(model, torch.zeros(1, model.spec.z_channels, 5, 2, 2), 2)


def _zoo_v11():
    import gzip
    import json
    import os
    zoo = json.load(gzip.open(os.path.join(os.path.dirname(__file__), "golden", "zoo_manifest.json.gz"), "rt"))
    return {n: r for n, r in zoo.items() if n.startswith("vidtok_v1_1/")}


def _earliest(grad):
    """first frame (axis 2) with a nonzero gradient, per sample"""
    nz = grad.abs().amax(dim=(1, 3, 4)) > 0
    return [int(r.nonzero().flatten().min()) for r in nz]


@pytest.mark.parametrize("name", sorted(_zoo_v11()))
def test_zoo_reach_is_the_oracles_reach(name):
    """The seven shipped v1.1 configurations at full width, seeded weights, at 1 x 1 latent positions: the reach of every
    output frame of a chunk period, read from the oracle's gradient (one sample per output frame), is R at most and R for
    some frame, for the encoder and for the decoder with and without overlap."""
    from oracle.vidtok_oracle import OracleModel, cfg_from_model_yaml
    from vidtok_b200.compat_util import instantiate_from_config
    from vidtok_b200.engine import NativeModel
    from vidtok_b200.longvideo import temporal_reach
    from vidtok_b200.synth import synth_state_dict
    rec = _zoo_v11()[name]
    model = instantiate_from_config(rec["model"])
    nm = NativeModel(model.spec)
    cfg = cfg_from_model_yaml(rec["model"])
    tdf, f = cfg.time_downsample_factor, nm.spatial_factor()
    sd = synth_state_dict({k: tuple(v) for k, v in rec["shapes"].items()}, seed=0)
    om = OracleModel(cfg, sd)
    om.use_tiling, om.t_chunk_enc, om.t_chunk_dec = True, 2 * tdf, 2
    enc, dec = OracleModel.encode.__wrapped__, OracleModel.decode.__wrapped__
    g = torch.Generator().manual_seed(0)
    # encoder: latents l of one chunk period, sample k asks about latent ls[k]
    R = temporal_reach(nm, False)
    c = om.t_chunk_enc
    T = 1 + c * ((R + 2 * c) // c)
    Tz = 1 + (T - 1) // tdf
    ls = [Tz - 1 - k for k in range(c // tdf)]
    x = torch.randn((len(ls), 3, T, f, f), generator=g).requires_grad_()
    h = enc(om, x, noise_fn=lambda s: torch.zeros(s), return_pre=True)[2]
    sum(h[k, :, l].sum() for k, l in enumerate(ls)).backward()
    reach = [1 + (l - 1) * tdf - j for l, j in zip(ls, _earliest(x.grad))]
    assert min(_earliest(x.grad)) > 0 and max(reach) == R, (reach, R)
    for ov in (False, True):
        om.use_overlap = ov
        R = temporal_reach(nm, True, ov)
        Tz = 1 + 2 * ((R + 6) // 2)
        ts = [tdf * l + r for l in (Tz - 4, Tz - 3) for r in (0, tdf - 1)]   # first / last frame of a chunk period's latents
        z = torch.randn((len(ts), cfg.z_channels, Tz, 1, 1), generator=g).requires_grad_()
        y = dec(om, z)
        sum(y[k, :, t].sum() for k, t in enumerate(ts)).backward()
        reach = [t // tdf - j for t, j in zip(ts, _earliest(z.grad))]
        assert min(_earliest(z.grad)) > 0 and max(reach) == R, (ov, reach, R)
