"""CPU-side checks of the streams' long-video recipe: the chunks an encode / decode stream forms from any push sizes are the
chunks of build_chunk_start_end (autoencoder_v1_1.py:218-228) and of the tile_decode loop (:322-330), the refusals of the
options, and the workspace query of vt_encode_chunk_fsq_aux (a dry run, no GPU)."""
import itertools
import random
from types import SimpleNamespace

import pytest

from conftest import load_golden, resolved_model_cfg

LENGTHS = (1, 2, 17, 33, 50, 129)


def _chunk_start_end(t, t_chunk_enc, t_chunk_dec=1, decoder_mode=False):
    from vidtok_b200.engine import AutoencodingEngineV11
    return AutoencodingEngineV11.build_chunk_start_end(SimpleNamespace(t_chunk_enc=t_chunk_enc, t_chunk_dec=t_chunk_dec), t,
                                                       decoder_mode=decoder_mode)


def _splits(T, seed=0):
    """Push schedules of T frames: every composition for small T, else single frames, one push and random splits."""
    if T <= 12:
        for cuts in itertools.product((0, 1), repeat=T - 1):
            sched, n = [], 1
            for c in cuts:
                if c:
                    sched.append(n)
                    n = 0
                n += 1
            yield sched + [n]
        return
    yield [1] * T
    yield [T]
    yield [3, 1, 7, 16] + [T - 27] if T > 27 else [T - 1, 1]
    rng = random.Random(seed * 1000 + T)
    for _ in range(200):
        sched, left = [], T
        while left:
            n = min(left, rng.choice((1, 2, 3, 5, 8, 15, 16, 17, 31, 40)))
            sched.append(n)
            left -= n
        yield sched


def _stream_encoder_spans(sched, t_chunk):
    from vidtok_b200.streaming import recipe_encode_chunks
    spans, first, pending, t0 = [], True, 0, 0
    for n in sched + [None]:
        final = n is None
        pending += 0 if final else n
        for c in recipe_encode_chunks(pending, first, t_chunk, final):
            spans.append([t0, t0 + c])
            t0 += c
            pending -= c
            first = False
    assert pending == 0
    return spans


def _stream_decoder_plan(sched, t_chunk, overlap, tdf):
    from vidtok_b200.streaming import recipe_decode_chunks
    plan, first, pending, t0 = [], True, 0, 0
    for n in sched + [None]:
        final = n is None
        pending += 0 if final else n
        for n_in, step, trim in recipe_decode_chunks(pending, first, t_chunk, overlap, tdf, final):
            plan.append((t0, n_in, trim))
            t0 += step
            pending -= step
            first = False
    assert pending == 0
    return plan


@pytest.mark.parametrize("T", LENGTHS)
@pytest.mark.parametrize("t_chunk", [4, 8, 16])
def test_encoder_chunks_follow_build_chunk_start_end_for_any_pushes(T, t_chunk):
    want = _chunk_start_end(T, t_chunk)
    for sched in _splits(T):
        assert _stream_encoder_spans(sched, t_chunk) == want, sched


@pytest.mark.parametrize("tdf", [2, 4, 8])
@pytest.mark.parametrize("overlap", [True, False])
def test_decoder_chunks_follow_the_tile_decode_loop(tdf, overlap):
    for t_chunk in sorted({1, 3, 16 // tdf}):
        for Tz in (1, 2, 3, 5, 9, 17, 33):
            # the reference loop: z[start:end+1] when the look-ahead frame exists, its last tdf decoded frames dropped
            want = []
            for start, end in _chunk_start_end(Tz, 16, t_chunk, decoder_mode=True):
                look = overlap and end + 1 <= Tz
                want.append((start, end - start + int(look), tdf if look else 0))
            for sched in _splits(Tz, seed=tdf):
                assert _stream_decoder_plan(sched, t_chunk, overlap, tdf) == want, (t_chunk, Tz, sched)


def test_a_chunk_waits_for_its_look_ahead_frame():
    from vidtok_b200.streaming import recipe_decode_chunks
    # 4-latent chunks after the first: 5 latents complete [0,1] (its look-ahead is latent 1) and [1,5) without look-ahead
    assert recipe_decode_chunks(5, True, 4, True, 4, False) == [(2, 1, 4)]
    assert recipe_decode_chunks(6, True, 4, True, 4, False) == [(2, 1, 4), (5, 4, 4)]
    assert recipe_decode_chunks(4, False, 4, True, 4, True) == [(4, 4, 0)]
    assert recipe_decode_chunks(4, False, 4, False, 4, False) == [(4, 4, 0)]


def test_recipe_option_refusals():
    from vidtok_b200.streaming import check_recipe
    check_recipe(1, 4, 16, False, False)
    check_recipe(1, 4, 4, True, True)
    check_recipe(1, 4, 3, False, True)            # decoder chunks count latent frames
    with pytest.raises(ValueError, match="v1.1"):
        check_recipe(0, 4, 16, False, False)       # v1.0 streams equal the whole clip for any chunking
    with pytest.raises(ValueError, match="multiple"):
        check_recipe(1, 4, 6, False, False)
    with pytest.raises(ValueError, match="use_overlap"):
        check_recipe(1, 4, None, True, True)
    with pytest.raises(ValueError, match="use_overlap"):
        check_recipe(0, 4, None, True, True)
    with pytest.raises(ValueError, match="2x, 4x or 8x"):
        check_recipe(1, 16, 1, True, True)


@pytest.mark.parametrize("case,kw", [("tiny_fsq_v10", dict(t_chunk=16)), ("tiny_kl_v11", dict(t_chunk=6))])
def test_stream_options_are_refused_before_the_model_is_loaded(case, kw):
    """A CPU model would fail with a RuntimeError when the stream loads it; the options are checked first."""
    from vidtok_b200.compat_util import instantiate_from_config
    from vidtok_b200.streaming import DecodeStream, EncodeStream
    _, meta = load_golden(case)
    model = instantiate_from_config(resolved_model_cfg(meta))
    with pytest.raises(ValueError):
        EncodeStream(model, 1, 32, 32, **kw)
    with pytest.raises(ValueError):
        DecodeStream(model, 1, 4, 4, use_overlap=True)


def test_chunk_fsq_aux_workspace_query():
    import ctypes as C
    from vidtok_b200 import _native as N
    from vidtok_b200.engine import ChunkState, NativeModel, TokenizerSpec
    lib = N.lib()
    kw = dict(version=1, ch=64, ch_mult=(1, 2, 4, 4), num_res_blocks=2, double_z=False, norm_type="layernorm")
    fsq = NativeModel(TokenizerSpec(z_channels=5, regularizer="fsq", fsq_levels=(8, 8, 8, 8, 8), **kw))
    enc = ChunkState(fsq, N.PREC_EXACT_TC, 1, 256, 256, False, False)
    base = lib.vt_chunk_workspace_bytes(enc.handle, 16)
    ws = lib.vt_chunk_fsq_aux_workspace_bytes(enc.handle, 16)
    h_bytes = 1 * 5 * 4 * 32 * 32 * 4
    assert base > 0 and ws >= base + h_bytes, (base, ws)
    dec = ChunkState(fsq, N.PREC_EXACT_TC, 1, 32, 32, True, False)
    assert lib.vt_chunk_fsq_aux_workspace_bytes(dec.handle, 4) == -1 and b"decoder state" in lib.vt_last_error()
    kl = NativeModel(TokenizerSpec(z_channels=4, **dict(kw, double_z=True)))
    kenc = ChunkState(kl, N.PREC_EXACT_TC, 1, 256, 256, False, False)
    assert lib.vt_chunk_fsq_aux_workspace_bytes(kenc.handle, 16) == -1 and b"FSQ model" in lib.vt_last_error()
    big = NativeModel(TokenizerSpec(z_channels=3, regularizer="fsq", fsq_levels=(300, 2, 2), **kw))
    benc = ChunkState(big, N.PREC_EXACT_TC, 1, 256, 256, False, False)
    assert lib.vt_chunk_fsq_aux_workspace_bytes(benc.handle, 16) == -1 and b"FSQ aux loss" in lib.vt_last_error()
    # refused before anything runs: no device is touched on this path
    z = C.c_void_p(0x1000)
    rc = lib.vt_encode_chunk_fsq_aux(kenc.handle, 1, z, 3, 1, z, z, 100.0, z, z, z, 1 << 30, None)
    assert rc == -1 and b"FSQ model" in lib.vt_last_error()   # VT_ERR_INVALID
    for st in (enc, dec, kenc, benc):
        st.close()
