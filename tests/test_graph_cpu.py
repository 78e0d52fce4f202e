"""CPU-side checks of CUDA graph capture: which stream chunks run eagerly and which graph each other chunk replays, the
capture / replay / eager life of a graph key, and the capture symbols of the C ABI."""
import ctypes as C

import pytest

from vidtok_b200 import _native as N
from vidtok_b200.streaming import (ChunkGraphs, chunk_graph_key, encode_chunks, recipe_decode_chunks,
                                   recipe_encode_chunks)

PUSHES = (1, 3, 4, 16, 17)


def test_capture_symbols_are_bound():
    lib = N.lib()
    for name in ("vt_chunk_state_reserve", "vt_chunk_state_parity", "vt_chunk_state_advance"):
        assert name in N.EXPORTS and getattr(lib, name).restype is C.c_int32
    assert N.ERR_CAPTURE == -6
    # null states are refused, not dereferenced
    assert lib.vt_chunk_state_parity(None) == -1
    assert lib.vt_chunk_state_advance(None) == -1
    assert lib.vt_chunk_state_reserve(None, 4, None) == -1


def _keys(chunk_lists, entry="plain"):
    """(chunk, key) over a stream's plans: chunk_lists is one list of chunk lengths per push (the last flagged final);
    every chunk flips the cache parity, as every cache commits on every chunk"""
    out, first, parity = [], True, 0
    for i, (chunks, final) in enumerate(chunk_lists):
        for n in chunks:
            out.append((n, chunk_graph_key(n, first, final, entry, parity)))
            first, parity = False, parity ^ 1
    return out


def _encoder_plans(push, total, version, tdf, t_chunk):
    plans, avail, first, fed = [], 0, True, 0
    while fed < total:
        t = min(push, total - fed)
        fed += t
        avail += t
        cs = encode_chunks(avail, first, tdf, version) if t_chunk is None else recipe_encode_chunks(avail, first, t_chunk, False)
        plans.append((cs, False))
        avail -= sum(cs)
        first = first and not cs
    if t_chunk is not None:
        plans.append((recipe_encode_chunks(avail, first, t_chunk, True), True))
    return plans


@pytest.mark.parametrize("push", PUSHES)
@pytest.mark.parametrize("version,t_chunk", [(0, None), (1, None), (1, 16)])
def test_encoder_chunk_keys(push, version, t_chunk):
    tdf, total = 4, 1 + 16 * 4
    keyed = _keys(_encoder_plans(push, total, version, tdf, t_chunk), "fsq_aux")
    assert sum(n for n, _ in keyed) == total if (version == 1 or t_chunk is None) else True
    assert keyed[0][1] is None                                   # the video's first chunk is eager
    for i, (n, key) in enumerate(keyed[1:], start=1):
        if t_chunk is not None and i == len(keyed) - 1 and n != t_chunk:
            assert key is None                                   # the flushed last chunk
            continue
        assert key == (n, "fsq_aux", i % 2)
        if t_chunk is not None:
            assert n == t_chunk
        else:
            assert n % tdf == 0
    if version == 1 and t_chunk is None:
        assert keyed[0][0] == 1


@pytest.mark.parametrize("push", PUSHES)
@pytest.mark.parametrize("use_overlap", [False, True])
def test_recipe_decoder_chunk_keys(push, use_overlap):
    tdf, t_chunk, total = 4, 4, 1 + 4 * 5
    plans, avail, first, fed = [], 0, True, 0
    while fed < total:
        t = min(push, total - fed)
        fed += t
        avail += t
        cs = recipe_decode_chunks(avail, first, t_chunk, use_overlap, tdf, False)
        plans.append(([n for n, _, _ in cs], False))
        avail -= sum(step for _, step, _ in cs)
        first = first and not cs
    plans.append(([n for n, _, _ in recipe_decode_chunks(avail, first, t_chunk, use_overlap, tdf, True)], True))
    keyed = _keys(plans)
    assert keyed[0] == (1 + use_overlap, None)
    flushed = len(plans[-1][0])   # with overlap the flush decodes the last chunk without look-ahead
    assert flushed == int(use_overlap)
    for i, (n, key) in enumerate(keyed[1:], start=1):
        if i >= len(keyed) - flushed:
            assert key is None and n <= t_chunk
        else:
            assert key == (t_chunk + use_overlap, "plain", i % 2)


def test_graph_life_of_a_key():
    """a key's first chunk runs eagerly, its second is captured, every later one replays; eager chunks stay eager"""
    g = ChunkGraphs()
    k = chunk_graph_key(4, False, False, "plain", 1)
    assert [g.action(None) for _ in range(3)] == ["eager"] * 3
    assert g.action(k) == "eager"
    assert g.action(k) == "capture"
    g.graphs[k] = {}
    assert [g.action(k) for _ in range(3)] == ["replay"] * 3
    assert g.action(chunk_graph_key(4, False, False, "plain", 0)) == "eager"
    assert g.action(chunk_graph_key(8, False, False, "plain", 1)) == "eager"
    assert chunk_graph_key(4, True, False, "plain", 0) is None
    assert chunk_graph_key(4, False, True, "pre", 0) is None
