"""CPU-side checks of the pools (EncodePool / DecodePool) without a GPU: the chunks PoolSchedule gives each video under
staggered opens, pushes and closes are the chunks of that video's own recipe stream run alone, and the refusals of the
scheduler, of the pool options and of vt_chunk_state_copy_slots (all before any device work)."""
import ctypes as C
import random

import pytest

from conftest import load_golden, resolved_model_cfg


def _simulate(sched, lengths, seed):
    """Videos of the given lengths through one PoolSchedule: each opens when a slot is free (at a random later step),
    pushes random amounts, and closes once all its frames are pushed (sometimes a few steps later).  Returns each
    video's chunks in the order they ran, and the chunk of every batched step."""
    rng = random.Random(seed)
    todo = list(range(len(lengths)))
    slot_of, left, got, batched, done_at = {}, {}, {v: [] for v in todo}, [], {}
    step = 0
    while todo or slot_of:
        if todo and rng.random() < 0.6 and sum(sched.busy) < sched.S:
            v = todo.pop(0)
            slot_of[v] = sched.open()
            left[v] = lengths[v]
        for v, s in list(slot_of.items()):
            if left[v]:
                n = min(left[v], rng.choice((0, 1, 3, 5, 8, 16, 17, 40)))
                sched.push(s, n)
                left[v] -= n
                if not left[v]:
                    done_at[v] = step + rng.choice((0, 0, 1, 3))
        joins, ready, chunk = sched.plan_step()
        by_slot = {s: v for v, s in slot_of.items()}
        for s, c in joins:
            got[by_slot[s]].append(c)
        if ready:
            batched.append(chunk)
            for s in ready:
                got[by_slot[s]].append(chunk)
        for v, s in list(slot_of.items()):
            if not left[v] and done_at[v] <= step:
                started, chunks = sched.close(s)
                assert started == (len(got[v]) > 0)
                got[v] += chunks
                del slot_of[v]
        step += 1
    return got, batched


LENGTHS = [1, 2, 17, 33, 50, 129, 40, 5]


@pytest.mark.parametrize("t_chunk", [4, 8, 16])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_encoder_plans_are_each_videos_recipe_chunks(t_chunk, seed):
    from vidtok_b200.streaming import PoolSchedule, recipe_encode_chunks
    sched = PoolSchedule(3, 1, 4, t_chunk, is_decoder=False)
    got, batched = _simulate(sched, LENGTHS, seed)
    for v, T in enumerate(LENGTHS):
        assert [n for n, _, _ in got[v]] == recipe_encode_chunks(T, True, t_chunk, True), (v, T, got[v])
    assert batched and all(c == (t_chunk, t_chunk, 0) for c in batched)
    assert not any(sched.busy)


@pytest.mark.parametrize("tdf", [2, 4, 8])
@pytest.mark.parametrize("overlap", [True, False])
@pytest.mark.parametrize("seed", [0, 1])
def test_decoder_plans_are_each_videos_recipe_chunks(tdf, overlap, seed):
    from vidtok_b200.streaming import PoolSchedule, recipe_decode_chunks
    lengths = [1, 2, 3, 5, 9, 17, 33, 12]
    for t_chunk in (1, 3, 16 // tdf):
        sched = PoolSchedule(4, 1, tdf, t_chunk, is_decoder=True, use_overlap=overlap)
        got, batched = _simulate(sched, lengths, seed)
        for v, Tz in enumerate(lengths):
            assert got[v] == recipe_decode_chunks(Tz, True, t_chunk, overlap, tdf, True), (t_chunk, v, Tz, got[v])
        look = int(overlap)
        assert all(c == (t_chunk + look, t_chunk, tdf * look) for c in batched)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_v10_plans_are_stream_chunks_of_each_video(seed):
    """v1.0: a video's chunks are those encode_chunks forms from pushes of 1 frame, then t_chunk frames, then the rest --
    valid stream chunks, so each video computes its whole clip; the decoder's are the stream's as well."""
    from vidtok_b200.streaming import PoolSchedule, encode_chunks, recipe_decode_chunks
    tdf, t_chunk = 4, 8
    lengths = [1, 5, 17, 33, 49, 9, 13]
    sched = PoolSchedule(3, 0, tdf, t_chunk, is_decoder=False)
    got, batched = _simulate(sched, lengths, seed)
    for v, T in enumerate(lengths):
        pushes = [1] + [t_chunk] * ((T - 1) // t_chunk) + ([(T - 1) % t_chunk] if (T - 1) % t_chunk else [])
        want, first = [], True
        for p in pushes:
            c = encode_chunks(p, first, tdf, 0)
            want += c
            first = False
        assert [n for n, _, _ in got[v]] == want, (v, T, got[v])
        assert want[0] % tdf == 1 and all(n % tdf == 0 for n in want[1:])
    dsched = PoolSchedule(3, 0, tdf, 3, is_decoder=True)
    got, _ = _simulate(dsched, [1, 2, 5, 9, 4], seed)
    for v, Tz in enumerate([1, 2, 5, 9, 4]):
        assert got[v] == recipe_decode_chunks(Tz, True, 3, False, tdf, True)


def test_v10_close_refuses_an_incomplete_group():
    from vidtok_b200.streaming import PoolSchedule
    sched = PoolSchedule(2, 0, 4, 8, is_decoder=False)
    s = sched.open()
    sched.push(s, 7)    # 1 + 4 + 2: the last two frames do not complete a group
    with pytest.raises(ValueError, match="group of 4"):
        sched.close(s)


def test_scheduler_refusals():
    from vidtok_b200.streaming import PoolSchedule
    sched = PoolSchedule(2, 1, 4, 16, is_decoder=False)
    a, b = sched.open(), sched.open()
    assert (a, b) == (0, 1)
    with pytest.raises(RuntimeError, match="all 2 slots"):
        sched.open()
    sched.push(a, 3)
    sched.close(a)
    with pytest.raises(RuntimeError, match="no open video"):
        sched.push(a, 1)           # closed
    with pytest.raises(RuntimeError, match="no open video"):
        sched.close(a)
    with pytest.raises(RuntimeError, match="no open video"):
        sched.push(5, 1)           # out of range
    assert sched.open() == a       # a freed slot is reused
    with pytest.raises(ValueError):
        PoolSchedule(0, 1, 4, 16, is_decoder=False)


def test_pool_option_refusals():
    from vidtok_b200.streaming import check_pool_recipe
    check_pool_recipe(1, 4, 16, False, False)
    check_pool_recipe(1, 4, 4, True, True)
    check_pool_recipe(0, 4, 8, False, False)
    check_pool_recipe(0, 4, 3, False, True)       # v1.0 decoder chunks count latent frames
    with pytest.raises(ValueError, match="t_chunk"):
        check_pool_recipe(1, 4, None, False, False)
    with pytest.raises(ValueError, match="multiple"):
        check_pool_recipe(0, 4, 6, False, False)
    with pytest.raises(ValueError, match="multiple"):
        check_pool_recipe(1, 4, 6, False, False)
    with pytest.raises(ValueError, match="use_overlap"):
        check_pool_recipe(0, 4, 4, True, True)


def test_non_causal_models_are_refused():
    from vidtok_b200.compat_util import instantiate_from_config
    from vidtok_b200.streaming import DecodePool, EncodePool
    _, meta = load_golden("tiny_kl_nc")
    model = instantiate_from_config(resolved_model_cfg(meta))
    with pytest.raises(ValueError, match="symmetric"):
        EncodePool(model, 4, 32, 32, t_chunk=16)
    with pytest.raises(ValueError, match="symmetric"):
        DecodePool(model, 4, 4, 4, t_chunk=4)


def test_copy_slots_refuses_mismatched_states():
    """vt_chunk_state_copy_slots refuses, before any device work, states that differ in model, precision, geometry,
    direction or use_overlap, one state as both ends, and slots out of range or listed twice."""
    from vidtok_b200 import _native as N
    from vidtok_b200.engine import ChunkState, NativeModel, TokenizerSpec
    lib = N.lib()
    kw = dict(version=1, ch=32, ch_mult=(1, 2, 4, 4), num_res_blocks=2, z_channels=4, double_z=True, norm_type="layernorm")
    nm, other = NativeModel(TokenizerSpec(**kw)), NativeModel(TokenizerSpec(**kw))
    base = ChunkState(nm, N.PREC_BF16, 4, 64, 64, False, False)
    cases = {
        "different models": ChunkState(other, N.PREC_BF16, 1, 64, 64, False, False),
        "precision": ChunkState(nm, N.PREC_EXACT_TC, 1, 64, 64, False, False),
        "geometry": ChunkState(nm, N.PREC_BF16, 1, 64, 128, False, False),
        "encoder and a decoder": ChunkState(nm, N.PREC_BF16, 1, 64, 64, True, False),
    }
    one = (C.c_int32 * 1)(0)
    for why, st in cases.items():
        for dst, src in ((base, st), (st, base)):
            assert lib.vt_chunk_state_copy_slots(dst.handle, src.handle, 1, one, one, None) == -1, why
            assert why.encode() in lib.vt_last_error(), (why, lib.vt_last_error())
    d1 = ChunkState(nm, N.PREC_BF16, 1, 16, 16, True, False)
    d2 = ChunkState(nm, N.PREC_BF16, 2, 16, 16, True, True)
    assert lib.vt_chunk_state_copy_slots(d2.handle, d1.handle, 1, one, one, None) == -1
    assert b"use_overlap" in lib.vt_last_error()
    assert lib.vt_chunk_state_copy_slots(base.handle, base.handle, 1, one, one, None) == -1
    assert b"same state" in lib.vt_last_error()
    side = ChunkState(nm, N.PREC_BF16, 1, 64, 64, False, False)
    bad = (C.c_int32 * 1)(4)
    assert lib.vt_chunk_state_copy_slots(base.handle, side.handle, 1, bad, one, None) == -1
    assert b"destination slot 4 of 4" in lib.vt_last_error()
    assert lib.vt_chunk_state_copy_slots(side.handle, base.handle, 1, one, bad, None) == -1
    assert b"source slot 4 of 4" in lib.vt_last_error()
    twice, src2 = (C.c_int32 * 2)(1, 1), (C.c_int32 * 2)(0, 0)
    assert lib.vt_chunk_state_copy_slots(base.handle, side.handle, 2, twice, src2, None) == -1
    assert b"listed twice" in lib.vt_last_error()
    # matching states with nothing written yet: nothing to copy, nothing launched
    assert lib.vt_chunk_state_copy_slots(base.handle, side.handle, 0, None, None, None) == 0
    for st in [base, side, d1, d2] + list(cases.values()):
        st.close()
