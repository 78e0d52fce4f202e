"""-m gpu: pools (EncodePool / DecodePool) against each video run alone.

* A slot copied out of a chunk state to a batch-1 state and back (vt_chunk_state_copy_slots) continues bit for bit as if
  it had never moved, for the v1.0 and v1.1 encoders and decoders, with and without overlap, in bf16 and in the
  split-operand layout.
* Videos of different lengths, opened and closed at staggered steps with slots reused, give each video's own
  tile_encode / tile_decode (v1.1) or whole-clip encode / decode (v1.0): bit for bit in bf16 and fma, to fp32 rounding in
  exact and mixed (FSQ codes equal outside the 1e-4 tie band); per-slot kl_loss and aux_loss are the solo run's.
* A slot whose caches hold NaN and run idle changes no other slot's output by a bit, and a video opened in it afterwards
  equals its solo run."""
import gc
import random

import pytest
import torch

pytestmark = pytest.mark.gpu

from conftest import load_golden, resolved_model_cfg, synth_weights  # noqa: E402
from test_gpu_fsq_aux import rel  # noqa: E402
from test_gpu_model import fsq_guard  # noqa: E402
from vidtok_b200 import _native as N  # noqa: E402


@pytest.fixture(autouse=True)
def _release_models():
    """Each model parks the chunk caches of every batch size it ran in its own pool: return them between tests."""
    yield
    gc.collect()
    torch.cuda.empty_cache()


def _model(case, mode, sample=None):
    from vidtok_b200.compat_util import instantiate_from_config
    d, meta = load_golden(case)
    cfg = resolved_model_cfg(meta)
    if sample is not None:
        cfg["params"]["regularizer_config"]["params"] = {"sample": sample}
    model = instantiate_from_config(cfg)
    missing, unexpected = model.load_state_dict(synth_weights(meta, d), strict=False)
    assert not missing and not unexpected
    model = model.to("cuda").eval()
    model.precision = mode
    return model, meta


def _class488(reg, mode):
    """kl_causal_488_4chn / fsq_causal_488 (v1.1) at reduced width, synthetic weights"""
    from oracle.make_golden import model_yaml
    from vidtok_b200.compat_util import instantiate_from_config
    from vidtok_b200.synth import synth_state_dict
    cfg = model_yaml(version="v1_1", reg=reg, ch=32, ch_mult=(1, 2, 4, 4), z=4 if reg == "kl" else 5)
    cfg["params"]["decoder_config"]["params"] = dict(cfg["params"]["encoder_config"]["params"])
    model = instantiate_from_config(cfg)
    model.load_state_dict(synth_state_dict({k: tuple(v.shape) for k, v in model.state_dict().items()}, seed=3))
    model = model.cuda().eval()
    model.precision = mode
    return model


def _video(T, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand((1, 3, T, H, W), generator=g) * 2 - 1).cuda()


def _same(got, want, bitwise, what):
    assert got.shape == want.shape, (what, tuple(got.shape), tuple(want.shape))
    if bitwise:
        assert torch.equal(got, want), (what, float((got.float() - want.float()).abs().max()))
    else:
        err = float((got.float() - want.float()).abs().max())
        assert err <= 1e-4 * (1.0 + float(want.float().abs().max())), (what, err)


# ---- transplant round trip ------------------------------------------------------------------------------------------
def _enc_chunk(model, st, x, first):
    from vidtok_b200.engine import _ptr, _stream_ptr
    nat, s = model._rt.sync(), model.spec
    B, _, n, H, W = x.shape
    tz, hz, wz = nat.latent_shape(n, H, W)
    z = torch.empty((B, s.z_channels, tz, hz, wz), device="cuda")
    h = torch.empty((B, (2 if s.double_z else 1) * s.z_channels, tz, hz, wz), device="cuda")
    idx = torch.empty((B, tz, hz, wz), dtype=torch.int32, device="cuda") if s.regularizer == "fsq" else None
    kl = torch.empty((1,), device="cuda") if s.regularizer == "kl" else None
    noise = torch.zeros_like(z) if s.regularizer == "kl" and s.kl_sample else None
    ws = st.workspace(n)
    N.check(nat.lib.vt_encode_chunk_pre(st.handle, int(first), _ptr(x.contiguous()), 3, n, _ptr(noise), _ptr(z), _ptr(idx), _ptr(kl),
                                        _ptr(h), _ptr(ws), ws.numel(), _stream_ptr(x.device)))
    return torch.cat([h.flatten(1), z.flatten(1)], dim=1)


def _dec_chunk(model, st, z, first):
    from vidtok_b200.engine import _ptr, _stream_ptr
    nat, s = model._rt.sync(), model.spec
    B, _, n, hz, wz = z.shape
    f = nat.spatial_factor()
    To = nat.decoded_frames(n) if (first or s.version == 1) else n * s.time_downsample_factor
    out = torch.empty((B, s.out_ch, To, hz * f, wz * f), device="cuda")
    ws = st.workspace(n)
    N.check(nat.lib.vt_decode_chunk(st.handle, int(first), _ptr(z.contiguous()), s.z_channels, n, _ptr(out), _ptr(ws), ws.numel(),
                                    _stream_ptr(z.device)))
    return out


@pytest.mark.parametrize("mode", ["bf16", "exact"])
@pytest.mark.parametrize("case,decoder,overlap", [("tiny_kl_v10", False, False), ("tiny_kl_v10", True, False),
                                                  ("tiny_fsq_v11_tiled", False, False), ("tiny_fsq_v11_tiled", True, False),
                                                  ("tiny_kl_v11_tiled", True, True), ("tiny_kl_v11_tiled", False, False)])
def test_transplant_round_trip_continues_bit_for_bit(case, decoder, overlap, mode):
    """State A (batch 3) and its twin R run the same chunks.  After chunk 1, A's slot 1 is copied out to a batch-1 state,
    overwritten with the caches of an unrelated video, and copied back: A's next chunks equal R's in every slot, bit for
    bit, so every cache key went out and came back."""
    from vidtok_b200.engine import ChunkState
    model, meta = _model(case, mode)
    nat, prec = model._rt.sync(), model._rt.precision()
    _, _, _, H, W = meta["input"]
    tdf = model.spec.time_downsample_factor
    if decoder:
        H, W = H // nat.spatial_factor(), W // nat.spatial_factor()
        g = torch.Generator().manual_seed(5)
        data = torch.randn((3, model.spec.z_channels, 2 + 3 * 3, H, W), generator=g).cuda()
        junk_data = torch.randn((1, model.spec.z_channels, 2 + 3, H, W), generator=g).cuda()
        lens, run = [2, 3, 3, 3], _dec_chunk
    else:
        data = torch.cat([_video(1 + 3 * 2 * tdf, H, W, seed) for seed in range(3)], dim=0)
        junk_data = _video(1 + 2 * tdf, H, W, 9)
        lens, run = [1, 2 * tdf, 2 * tdf, 2 * tdf], _enc_chunk
    A, R = (ChunkState(nat, prec, 3, H, W, decoder, overlap) for _ in range(2))
    side, junk = (ChunkState(nat, prec, 1, H, W, decoder, overlap) for _ in range(2))
    with torch.no_grad():
        run(model, junk, junk_data[:, :, :lens[0]], True)
        run(model, junk, junk_data[:, :, lens[0]:lens[0] + lens[1]], False)
        t0 = 0
        for i, n in enumerate(lens):
            xa = data[:, :, t0:t0 + n]
            a, r = run(model, A, xa, i == 0), run(model, R, xa, i == 0)
            assert torch.equal(a, r), (i, float((a - r).abs().max()))
            if i == 1:
                side.copy_slots(A, [0], [1])
                A.copy_slots(junk, [1], [0])
                A.copy_slots(side, [1], [0])
            t0 += n
    for st in (A, R, side, junk):
        st.close()


# ---- pool equals solo -----------------------------------------------------------------------------------------------
def _drive(pool, feeds, seed, capacity):
    """Runs feeds {video: (tensor [1,C,T,...], open kwargs)} through the pool with staggered opens, random push sizes and
    closes that trail the last push by a few steps; a video waits for a free slot.  Returns ({video: output parts},
    {video: last reg_log}, {video: slot})."""
    rng = random.Random(seed)
    todo = sorted(feeds)
    slot_of, t0, outs, logs, slots, close_at = {}, {}, {v: [] for v in feeds}, {}, {}, {}
    step = 0
    while todo or slot_of:
        if todo and len(slot_of) < capacity and rng.random() < 0.7:
            v = todo.pop(0)
            slot_of[v] = pool.open(**feeds[v][1])
            slots.setdefault(v, slot_of[v])
            t0[v] = 0
        for v, s in list(slot_of.items()):
            T = feeds[v][0].shape[2]
            if t0[v] < T:
                n = min(T - t0[v], rng.choice((0, 1, 2, 3, 5, 8, 13)))
                if n:
                    pool.push(s, feeds[v][0][:, :, t0[v]:t0[v] + n])
                t0[v] += n
                if t0[v] == T:
                    close_at[v] = step + rng.choice((0, 1, 2))
        by_slot = {s: v for v, s in slot_of.items()}
        for s, got in pool.step().items():
            v = by_slot[s]
            if isinstance(got, tuple):
                outs[v].append(got[0])
                logs[v] = got[1]
                if "indices" in got[1]:
                    outs[v][-1] = (got[0], got[1]["indices"])
            else:
                outs[v].append(got)
        for v, s in list(slot_of.items()):
            if t0[v] == feeds[v][0].shape[2] and close_at[v] <= step:
                got = pool.close(s)
                if isinstance(got, tuple):
                    outs[v].append((got[0], got[1]["indices"]) if "indices" in got[1] else got[0])
                    logs[v] = got[1]
                else:
                    outs[v].append(got)
                del slot_of[v]
        step += 1
    return outs, logs, slots


def _cat_enc(parts):
    if parts and isinstance(parts[0], tuple):
        return torch.cat([p[0] for p in parts], dim=2), torch.cat([p[1] for p in parts], dim=1)
    return torch.cat(parts, dim=2), None


V11_LENGTHS = [17, 33, 9, 50, 1, 26, 12]


def _check_v11_pool(model, H, W, mode, t_chunk, seed, lengths=V11_LENGTHS, capacity=3):
    from vidtok_b200.streaming import DecodePool, EncodePool, EncodeStream
    bitwise = mode in ("bf16", "fma")
    tdf = model.spec.time_downsample_factor
    model.use_tiling, model.t_chunk_enc, model.t_chunk_dec = True, t_chunk, t_chunk // tdf
    xs = {v: _video(T, H, W, 100 + v) for v, T in enumerate(lengths)}
    ref = {}
    with torch.no_grad():
        for v, x in xs.items():
            torch.manual_seed(1000 + v)
            ref[v] = model.tile_encode(x)
        pool = EncodePool(model, capacity, H, W, t_chunk=t_chunk)
        feeds = {v: (x, {"generator": torch.Generator().manual_seed(1000 + v)}) for v, x in xs.items()}
        outs, logs, slots = _drive(pool, feeds, seed, capacity)
        assert len(set(slots.values())) < len(lengths), "no slot was reused"
        assert pool.counts["batched"] > 0 and pool.counts["transplants"] > 0, pool.counts
        pool.close_pool()
        for v in xs:
            z, idx = _cat_enc(outs[v])
            z_ref, log_ref = ref[v]
            if idx is None or bitwise or torch.equal(idx, log_ref["indices"]):   # FSQ codes follow the indices
                _same(z, z_ref, bitwise, ("z", v))
            if idx is not None:
                if bitwise:
                    assert torch.equal(idx, log_ref["indices"]), v
                else:
                    st = EncodeStream(model, 1, H, W, t_chunk=t_chunk, keep_pre_bound=True)
                    h = torch.cat([st.push(xs[v])[1]["h_pre"], st.flush()[1]["h_pre"]], dim=2)
                    st.close()
                    fsq_guard(idx.cpu(), log_ref["indices"].cpu(), h.cpu(), model.regularization.levels)
                got, want = float(logs[v]["aux_loss"]), float(log_ref["aux_loss"])
                assert rel(got, want) <= 1e-5, (v, got, want)
            else:
                got, want = float(logs[v]["kl_loss"]), float(log_ref["kl_loss"])
                assert rel(got, want) <= 1e-5, (v, got, want)
        for ov in (False, True):
            model.use_overlap = ov
            dref = {v: model.tile_decode(ref[v][0]) for v in xs}
            pool = DecodePool(model, capacity, ref[0][0].shape[3], ref[0][0].shape[4], t_chunk=t_chunk // tdf, use_overlap=ov)
            outs, _, _ = _drive(pool, {v: (ref[v][0], {}) for v in xs}, seed + 1, capacity)
            pool.close_pool()
            for v in xs:
                _same(torch.cat(outs[v], dim=2), dref[v], bitwise or mode == "mixed", ("decode", ov, v))


@pytest.mark.parametrize("mode", ["bf16", "fma", "exact", "mixed"])
@pytest.mark.parametrize("case", ["tiny_kl_v11_tiled", "tiny_fsq_v11_tiled"])
def test_v11_pool_equals_each_videos_tile_paths(case, mode):
    model, meta = _model(case, mode)
    _, _, _, H, W = meta["input"]
    _check_v11_pool(model, H, W, mode, 8, seed=hash(case) % 100)


@pytest.mark.parametrize("mode", ["bf16", "exact"])
@pytest.mark.parametrize("reg", ["kl", "fsq"])
def test_488_class_pool_equals_each_videos_tile_paths(reg, mode):
    _check_v11_pool(_class488(reg, mode), 64, 64, mode, 16, seed=3, lengths=[33, 17, 49, 5, 40], capacity=4)


@pytest.mark.parametrize("mode", ["bf16", "fma", "exact"])
@pytest.mark.parametrize("case", ["tiny_kl_v10", "tiny_fsq_v10"])
def test_v10_pool_equals_each_videos_whole_clip(case, mode):
    from vidtok_b200.streaming import DecodePool, EncodePool
    model, meta = _model(case, mode, sample=False if "kl" in case else None)
    _, _, _, H, W = meta["input"]
    bitwise = mode in ("bf16", "fma")
    lengths = [17, 33, 5, 1, 21, 13]
    xs = {v: _video(T, H, W, 200 + v) for v, T in enumerate(lengths)}
    with torch.no_grad():
        ref = {v: model.encode(x, return_reg_log=True) for v, x in xs.items()}
        pool = EncodePool(model, 3, H, W, t_chunk=8)
        outs, logs, _ = _drive(pool, {v: (x, {}) for v, x in xs.items()}, 5, 3)
        pool.close_pool()
        for v in xs:
            z, idx = _cat_enc(outs[v])
            z_ref, log_ref = ref[v]
            if idx is None or bitwise or torch.equal(idx, log_ref["indices"]):   # FSQ codes follow the indices
                _same(z, z_ref, bitwise, ("z", v))
            if idx is not None:
                mism = int((idx != log_ref["indices"]).sum())
                assert mism == 0 or (not bitwise and mism <= 1e-3 * idx.numel()), (v, mism)
                assert rel(float(logs[v]["aux_loss"]), float(log_ref["aux_loss"])) <= 1e-5, v
            else:
                assert rel(float(logs[v]["kl_loss"]), float(log_ref["kl_loss"])) <= 1e-5, v
        pool = DecodePool(model, 3, ref[0][0].shape[3], ref[0][0].shape[4], t_chunk=2)
        outs, _, _ = _drive(pool, {v: (ref[v][0], {}) for v in xs}, 6, 3)
        pool.close_pool()
        for v in xs:
            _same(torch.cat(outs[v], dim=2), model.decode(ref[v][0]), bitwise, ("decode", v))


# ---- isolation --------------------------------------------------------------------------------------------------------
def test_a_nan_slot_changes_no_other_slot():
    """bf16: slot 2's caches are filled with NaN (transplanted from a side state fed NaN frames) and run idle (on zeros)
    while videos in slots 0 and 1 run; they equal their solo tile_encode bit for bit.  Slot 2 still holds NaN afterwards,
    and a video opened in it then equals its own solo run."""
    from vidtok_b200.engine import ChunkState
    from vidtok_b200.streaming import EncodePool
    model, meta = _model("tiny_fsq_v11_tiled", "bf16")
    _, _, _, H, W = meta["input"]
    model.use_tiling, model.t_chunk_enc = True, 8
    nat, prec = model._rt.sync(), model._rt.precision()
    with torch.no_grad():
        xs = [_video(T, H, W, 300 + i) for i, T in enumerate((41, 33, 25))]
        ref = [model.tile_encode(x) for x in xs]
        pool = EncodePool(model, 3, H, W, t_chunk=8)
        a, b = pool.open(), pool.open()
        nan = ChunkState(nat, prec, 1, H, W, False, False)
        bad = torch.full((1, 3, 9, H, W), float("nan"), device="cuda")
        _enc_chunk(model, nan, bad[:, :, :1], True)
        _enc_chunk(model, nan, bad[:, :, 1:], False)
        pool.main.copy_slots(nan, [2], [0])
        outs = {a: [], b: []}
        for t0 in range(0, 41, 8):
            pool.push(a, xs[0][:, :, t0:t0 + 8])
            if t0 < 33:
                pool.push(b, xs[1][:, :, t0:t0 + 8])
            for s, (z, log) in pool.step().items():
                outs[s].append((z, log["indices"]))
        for s in (a, b):
            z, log = pool.close(s)
            outs[s].append((z, log["indices"]))
        for s, i in ((a, 0), (b, 1)):
            z, idx = _cat_enc(outs[s])
            assert torch.equal(z, ref[i][0]) and torch.equal(idx, ref[i][1]["indices"]), s
        probe = ChunkState(nat, prec, 1, H, W, False, False)
        probe.copy_slots(pool.main, [0], [2])
        assert torch.isnan(_enc_chunk(model, probe, torch.zeros((1, 3, 8, H, W), device="cuda"), False)).any()
        c = pool.open()
        assert c == 0      # the lowest free slot; open the NaN slot next
        d = pool.open()
        e = pool.open()
        assert e == 2
        pool.push(e, xs[2])
        parts = []
        for _ in range(4):
            got = pool.step()
            if e in got:
                parts.append((got[e][0], got[e][1]["indices"]))
        z, log = pool.close(e)
        parts.append((z, log["indices"]))
        z, idx = _cat_enc(parts)
        assert torch.equal(z, ref[2][0]) and torch.equal(idx, ref[2][1]["indices"])
        assert rel(float(log["aux_loss"]), float(ref[2][1]["aux_loss"])) <= 1e-5
        for s in (c, d):
            pool.close(s)
        pool.close_pool()
        nan.close()
        probe.close()


def test_pool_refusals():
    from vidtok_b200.streaming import DecodePool, EncodePool
    model, meta = _model("tiny_kl_v11_tiled", "bf16")
    _, _, _, H, W = meta["input"]
    pool = EncodePool(model, 2, H, W, t_chunk=8)
    s = pool.open()
    with pytest.raises(ValueError, match="expected"):
        pool.push(s, torch.zeros((1, 3, 4, H, W + 8), device="cuda"))      # another geometry
    with pytest.raises(ValueError, match="expected"):
        pool.push(s, torch.zeros((2, 3, 4, H, W), device="cuda"))          # one video per slot
    pool.open()
    with pytest.raises(RuntimeError, match="slots"):
        pool.open()
    pool.close(s)
    with pytest.raises(RuntimeError, match="no open video"):
        pool.push(s, torch.zeros((1, 3, 4, H, W), device="cuda"))
    with pytest.raises(ValueError, match="t_chunk"):
        EncodePool(model, 2, H, W)
    with pytest.raises(ValueError, match="multiple"):
        EncodePool(model, 2, H, W, t_chunk=6)
    dec = DecodePool(model, 2, 4, 4, t_chunk=2, use_overlap=True)
    with pytest.raises(ValueError, match="expected"):
        dec.push(dec.open(), torch.zeros((1, 4, 3, 4, 8), device="cuda"))
    pool.close_pool()
    dec.close_pool()
