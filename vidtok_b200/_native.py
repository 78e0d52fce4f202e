"""ctypes binding of include/vidtok_b200.h.  Loading fails loudly when the CUDA library is missing: there is no
CPU or PyTorch fallback on the product path."""
from __future__ import annotations

import ctypes as C
import os

VT_MAX_LEVELS = 8
# include/vidtok_b200.h: FMA32 (fp32 FMA kernels), BF16 (wgmma), EXACT_TC (fp16 hi|lo split operands, 3 MMAs per K step, on wgmma), MIXED
PREC_FMA32, PREC_BF16, PREC_EXACT_TC, PREC_MIXED = 0, 1, 2, 3
PREC_EXACT = PREC_EXACT_TC  # the parity mode
DTYPE_F32, DTYPE_BF16, DTYPE_F16 = 0, 1, 2   # VT_DTYPE_*
ERR_CAPTURE = -6   # VT_ERR_CAPTURE: refused while the stream captures a CUDA graph
_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libvidtok_b200.so")


class ModelDesc(C.Structure):
    _fields_ = [
        ("version", C.c_int32), ("ch", C.c_int32), ("num_levels", C.c_int32), ("ch_mult", C.c_int32 * VT_MAX_LEVELS),
        ("num_res_blocks", C.c_int32), ("in_channels", C.c_int32), ("out_ch", C.c_int32), ("z_channels", C.c_int32),
        ("double_z", C.c_int32), ("norm_type", C.c_int32), ("time_downsample_factor", C.c_int32),
        ("n_spatial_ds", C.c_int32), ("spatial_ds", C.c_int32 * VT_MAX_LEVELS),
        ("n_tempo_ds", C.c_int32), ("tempo_ds", C.c_int32 * VT_MAX_LEVELS),
        ("n_spatial_us", C.c_int32), ("spatial_us", C.c_int32 * VT_MAX_LEVELS),
        ("n_tempo_us", C.c_int32), ("tempo_us", C.c_int32 * VT_MAX_LEVELS),
        ("interpolation_mode", C.c_int32), ("regularizer", C.c_int32), ("fsq_num_levels", C.c_int32),
        ("fsq_levels", C.c_int32 * VT_MAX_LEVELS), ("kl_sample", C.c_int32), ("noncausal", C.c_int32),
    ]


class ConvDesc(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "B", "Ti", "Hi", "Wi", "Ci", "Co", "kt", "kh", "kw", "st", "sh", "sw", "pt", "ph0", "ph1", "pw0", "pw1",
        "ut", "uh", "uw", "res_mode")] + [("alpha", C.c_float)]


class ConvEx(C.Structure):
    _fields_ = [("d", ConvDesc)] + [(n, C.c_int32) for n in (
        "force_simt", "t_mode", "cacheT", "ln_mode", "ln_silu", "to_off", "out_f32_ncdhw", "res_mix", "res_t_mode", "pt_back",
        "res_pool_off")]


_P, _I32, _I64 = C.c_void_p, C.c_int32, C.c_int64
_SIGS = {
    "vt_last_error": (C.c_char_p, []),
    "vt_abi_version": (_I32, []),
    "vt_launch_count": (_I64, [_I32]),
    "vt_profile_start": (None, []),
    "vt_profile_start_detailed": (None, []),
    "vt_profile_stop": (_I32, [C.c_char_p, _I32]),
    "vt_model_create": (_I32, [C.POINTER(ModelDesc), _I32, C.POINTER(_P)]),
    "vt_model_destroy": (None, [_P]),
    "vt_model_num_params": (_I32, [_P]),
    "vt_model_param_info": (_I32, [_P, _I32, C.c_char_p, _I32, C.POINTER(_I64), C.POINTER(_I32)]),
    "vt_model_load_param": (_I32, [_P, C.c_char_p, _P, _I64, _I32, _P]),
    "vt_model_finalize": (_I32, [_P, _P]),
    "vt_latent_shape": (_I32, [_P, _I32, _I32, _I32, C.POINTER(_I32), C.POINTER(_I32), C.POINTER(_I32)]),
    "vt_decoded_frames": (_I32, [_P, _I32]),
    "vt_workspace_bytes": (_I64, [_P, _I32, _I32, _I32, _I32, _I32]),
    "vt_encode": (_I32, [_P, _I32, _P, _I32, _I32, _I32, _I32, _I32, _P, _P, _P, _P, _P, _P, _I64, _P]),
    "vt_decode": (_I32, [_P, _I32, _P, _I32, _I32, _I32, _I32, _I32, _I32, _P, _P, _I64, _P]),
    "vt_chunk_state_create": (_I32, [_P, _I32, _I32, _I32, _I32, _I32, _I32, C.POINTER(_P)]),
    "vt_chunk_state_destroy": (None, [_P]),
    "vt_chunk_workspace_bytes": (_I64, [_P, _I32]),
    "vt_encode_chunk": (_I32, [_P, _I32, _P, _I32, _I32, _P, _P, _P, _P, _P, _I64, _P]),
    "vt_encode_chunk_pre": (_I32, [_P, _I32, _P, _I32, _I32, _P, _P, _P, _P, _P, _P, _I64, _P]),
    "vt_chunk_fsq_aux_workspace_bytes": (_I64, [_P, _I32]),
    "vt_encode_chunk_fsq_aux": (_I32, [_P, _I32, _P, _I32, _I32, _P, _P, C.c_float, _P, _P, _P, _I64, _P]),
    "vt_decode_chunk": (_I32, [_P, _I32, _P, _I32, _I32, _P, _P, _I64, _P]),
    "vt_chunk_state_copy_slots": (_I32, [_P, _P, _I32, C.POINTER(_I32), C.POINTER(_I32), _P]),
    "vt_chunk_state_reserve": (_I32, [_P, _I32, _P]),
    "vt_chunk_state_parity": (_I32, [_P]),
    "vt_chunk_state_advance": (_I32, [_P]),
    "vt_encode_video_workspace_bytes": (_I64, [_P, _I32, _I32, _I32, _I32, _I32, _I32]),
    "vt_encode_video": (_I32, [_P, _I32, _P, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _P, _P, _P, _P, _P, _I64, _P]),
    "vt_encode_video_fsq_aux_workspace_bytes": (_I64, [_P, _I32, _I32, _I32, _I32, _I32, _I32]),
    "vt_encode_video_fsq_aux": (_I32, [_P, _I32, _P, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _P, _P, C.c_float, _P, _P, _P, _I64, _P]),
    "vt_decode_video_workspace_bytes": (_I64, [_P, _I32, _I32, _I32, _I32, _I32, _I32, _I32]),
    "vt_decode_video_frames": (_I32, [_P, _I32, _I32, _I32]),
    "vt_decode_video": (_I32, [_P, _I32, _P, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _P, _I32, _P, _I64, _P]),
    "vt_temporal_reach": (_I32, [_P, _I32, _I32, C.POINTER(_I32)]),
    "vt_video_u8_to_clip": (_I32, [_P, _P, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _P]),
    "vt_video_u8_to_clip_resized": (_I32, [_P, _P] + [_I32] * 11 + [_P]),
    "vt_clip_to_video_u8": (_I32, [_P, _P, _I32, _I32, _I32, _I32, _P]),
    "vt_frame_scores_workspace_bytes": (_I64, [_I32] * 5),
    "vt_frame_scores": (_I32, [_P, _I32, _P, _I32] + [_I32] * 5 + [_P, _P, _P, _P, _I64, _P]),
    "vt_lpips_create": (_I32, [_I32, C.POINTER(_P)]),
    "vt_lpips_destroy": (None, [_P]),
    "vt_lpips_num_params": (_I32, [_P]),
    "vt_lpips_param_info": (_I32, [_P, _I32, C.c_char_p, _I32, C.POINTER(_I64), C.POINTER(_I32)]),
    "vt_lpips_load_param": (_I32, [_P, C.c_char_p, _P, _I64, _I32, _P]),
    "vt_lpips_finalize": (_I32, [_P, _P]),
    "vt_lpips_pass_frames": (_I32, [_I32, _I32]),
    "vt_lpips_workspace_bytes": (_I64, [_P] + [_I32] * 6),
    "vt_lpips": (_I32, [_P, _I32, _P, _I32, _P, _I32] + [_I32] * 5 + [_P, _P, _P, _P, _I64, _P]),
    "vt_i3d_create": (_I32, [_I32, C.POINTER(_P)]),
    "vt_i3d_destroy": (None, [_P]),
    "vt_i3d_num_params": (_I32, [_P]),
    "vt_i3d_param_info": (_I32, [_P, _I32, C.c_char_p, _I32, C.POINTER(_I64), C.POINTER(_I32)]),
    "vt_i3d_load_param": (_I32, [_P, C.c_char_p, _P, _I64, _I32, _P]),
    "vt_i3d_finalize": (_I32, [_P, _P]),
    "vt_i3d_pass_clips": (_I32, [_P, _I32, _I32, _I32]),
    "vt_i3d_workspace_bytes": (_I64, [_P] + [_I32] * 6),
    "vt_i3d_features": (_I32, [_P, _I32, _P, _I32] + [_I32] * 5 + [_P, _P, _P, _I64, _P]),
    "vt_i3d_endpoint": (_I32, [_P, _I32, _P, _I32] + [_I32] * 5 + [C.c_char_p, _P, C.POINTER(_I64), _P, _I64, _P]),
    "vt_op_conv_relu": (_I32, [_I32, C.POINTER(ConvDesc), _P, _P, _P, _P, _P]),
    "vt_op_maxpool2x2": (_I32, [_I32, _P, _P, _I64, _I32, _I32, _I32, _P]),
    "vt_op_conv": (_I32, [_I32, _I32, C.POINTER(ConvDesc), _P, _P, _P, _P, _P, _P]),
    "vt_op_conv_ex": (_I32, [_I32, C.POINTER(ConvEx), _P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "vt_op_conv_regularize": (_I32, [_I32, C.POINTER(ConvDesc), _P, _P, _P, _I32, _I32, C.POINTER(_I32), _P, _P, _P, _P, _P, _P]),
    "vt_op_conv_regularize_ex": (_I32, [_I32, C.POINTER(ConvEx), _P, _P, _P, _P, _I32, _I32, C.POINTER(_I32), _P, _P, _P, _P, _P, _P]),
    "vt_op_conv_stem": (_I32, [_I32, _P, _P, _P, _P, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _P]),
    "vt_op_conv_stem_ex": (_I32, [_I32, _P, _P, _P, _P, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _P]),
    "vt_op_head_planes": (_I32, [_P, _P, _P, _P, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _P]),
    "vt_op_upsample_conv": (_I32, [_I32, _I32, _P, _P, _P, C.c_float, _P, _P, _I32, _P, _P, _I32, _I32, _I32, _I32, _I32, _I32, _P]),
    "vt_op_tblock": (_I32, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _I32, _P, _P, _I32, _I32, _I32, _I32, _I32, _P]),
    "vt_op_tblock_cached": (_I32, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _I32, _P, _P, _P, _P, _P, _P, _I32, _I32, _I32, _I32, _I32, _P]),
    "vt_op_layernorm": (_I32, [_I32, _P, _P, _P, _P, _I64, _I32, _I32, _P]),
    "vt_op_groupnorm": (_I32, [_I32, _P, _P, _P, _P, _I64, _I64, _I32, _I32, _I32, _P, _I64, _P]),
    "vt_op_attention": (_I32, [_I32, _P, _P, _P, _P, _I32, _I32, _I32, _P, _I64, _P]),
    "vt_op_attention_hw": (_I32, [_I32, _P, _P, _P, _P, _I32, _I32, _I32, _I32, _P, _I64, _P]),
    "vt_op_fsq": (_I32, [_P, _I32, C.POINTER(_I32), _I64, _I32, _P, _P, _P]),
    "vt_op_fsq_indices_to_codes": (_I32, [_P, _I32, C.POINTER(_I32), _I64, _I32, _P, _P]),
    "vt_op_kl": (_I32, [_P, _P, _I32, _I64, _I32, _I32, _P, _P, _P]),
    "vt_fsq_aux_workspace_bytes": (_I64, [_I32, C.POINTER(_I32), _I64]),
    "vt_fsq_aux_partials": (_I32, [_P, _I32, C.POINTER(_I32), _I64, _I32, C.c_float, _P, _P, _P, _I64, _P]),
    "vt_fsq_aux_finalize": (_I32, [_P, _P, _I32, _I32, C.POINTER(_I32), _I32, C.c_float, C.c_float, C.c_float, _P, _P, _P]),
}
EXPORTS = tuple(_SIGS.keys())

_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing. Build it with `python -c 'import __graft_entry__ as g; g.build()'`. "
                "vidtok_b200 has no CPU / PyTorch fallback."
            )
        l = C.CDLL(LIB_PATH)
        for name, (res, args) in _SIGS.items():
            fn = getattr(l, name)
            fn.restype = res
            fn.argtypes = args
        _lib = l
    return _lib


def check(rc: int):
    if rc != 0:
        raise RuntimeError(f"vidtok_b200 error {rc}: {lib().vt_last_error().decode(errors='replace')}")
