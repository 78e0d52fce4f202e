"""CPU-side checks of streaming: chunk and frame counts of push schedules, rejection of non-causal models, and the dry-run
workspace of a streamed 1080p clip (vt_chunk_workspace_bytes, computed without a GPU)."""
import ctypes as C

import pytest

from conftest import load_golden, resolved_model_cfg


def _kl488(version=0):
    from vidtok_b200.engine import NativeModel, TokenizerSpec
    return NativeModel(TokenizerSpec(version=version, ch=128, ch_mult=(1, 2, 4, 4), num_res_blocks=2, z_channels=4, double_z=True,
                                     norm_type="layernorm"))


def test_push_schedules_frame_and_latent_counts():
    from vidtok_b200.streaming import encode_chunks
    nm = _kl488()
    # 1 + 4k frames give 1 + k latents, whatever the pushes
    for sched in ([1, 4, 4, 4, 4], [1, 16], [17], [3, 2, 7, 5], [2, 2, 2, 2, 2, 2, 2, 2, 1]):
        first, pending, chunks = True, 0, []
        for n in sched:
            c = encode_chunks(pending + n, first, 4, 0)
            pending += n - sum(c)
            first = first and not c
            chunks += c
        assert sum(chunks) == 17 and pending == 0, sched
        assert chunks[0] % 4 == 1 and all(c % 4 == 0 for c in chunks[1:]), (sched, chunks)
        assert nm.latent_shape(chunks[0], 256, 256)[0] + sum(c // 4 for c in chunks[1:]) == 5
    assert encode_chunks(3, True, 4, 0) == [1] and encode_chunks(2, False, 4, 0) == []
    assert encode_chunks(9, True, 4, 1) == [1, 8]       # v1.1: the first frame is a chunk of its own
    # decoding: the first latent gives 1 frame (tdf - 1 dropped), every later latent tdf frames
    assert nm.decoded_frames(1) == 1 and nm.decoded_frames(5) == 17
    assert _kl488(1).decoded_frames(1) == 4


def test_non_causal_models_are_rejected():
    from vidtok_b200 import _native as N
    from vidtok_b200.compat_util import instantiate_from_config
    from vidtok_b200.engine import NativeModel
    from vidtok_b200.streaming import EncodeStream
    d, meta = load_golden("tiny_kl_nc")
    model = instantiate_from_config(resolved_model_cfg(meta))
    with pytest.raises(ValueError, match="symmetric"):
        EncodeStream(model, 1, 32, 32)
    nm = NativeModel(model.spec)
    st = C.c_void_p()
    assert N.lib().vt_chunk_state_create(nm.handle, N.PREC_BF16, 1, 32, 32, 0, 0, C.byref(st)) == -1
    assert b"non-causal" in N.lib().vt_last_error()
    # v1.0 has no overlap look-ahead
    assert N.lib().vt_chunk_state_create(_kl488().handle, N.PREC_BF16, 1, 32, 32, 1, 1, C.byref(st)) == -1


def test_streamed_1080p_exact_workspace_is_bounded():
    """kl488 at 1080x1920 in exact: the whole 17-frame clip needs ~133 GB of workspace (more than an 80 GB card); a stream of
    4-frame chunks needs a fixed amount, whatever the video's length."""
    from vidtok_b200 import _native as N
    from vidtok_b200.engine import ChunkState
    nm = _kl488()
    lib = N.lib()
    whole17 = lib.vt_workspace_bytes(nm.handle, N.PREC_EXACT_TC, 1, 17, 1080, 1920)
    whole33 = lib.vt_workspace_bytes(nm.handle, N.PREC_EXACT_TC, 1, 33, 1080, 1920)
    assert whole17 > 100e9 and whole33 > 1.5 * whole17
    enc = ChunkState(nm, N.PREC_EXACT_TC, 1, 1080, 1920, False, False)
    dec = ChunkState(nm, N.PREC_EXACT_TC, 1, 135, 240, True, False)
    ws_enc = max(lib.vt_chunk_workspace_bytes(enc.handle, 1), lib.vt_chunk_workspace_bytes(enc.handle, 4))
    ws_dec = lib.vt_chunk_workspace_bytes(dec.handle, 1)
    assert 0 < ws_enc < 40e9 and 0 < ws_dec < 40e9, (ws_enc, ws_dec)
    enc.close()
    dec.close()
