"""ctypes binding of the C-ABI kernel library ``libsvi_b200.so`` (declared in ``include/svi_b200.h``,
``include/svi_b200_lora.h``, ``include/svi_b200_rife.h``, ``include/svi_b200_esrgan.h``,
``include/svi_b200_fastblend.h``, ``include/svi_b200_fastblend_modes.h``,
``include/svi_b200_unianimate.h``, ``include/svi_b200_replace.h``,
``include/svi_b200_quality.h``, ``include/svi_b200_reward.h`` and ``include/svi_b200_processors.h``).

This is the only door between the Python host code and the hand-written sm_90a kernels.  There is no
fallback: if the shared library is missing or a call fails, a ``RuntimeError`` is raised.
"""
import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
# SVI_B200_LIB: another build of the same library (A/B measurements of compiler flags / kernel variants)
_LIB_PATH = os.environ.get("SVI_B200_LIB") or os.path.join(os.path.dirname(_HERE), "lib", "libsvi_b200.so")

ACT_NONE, ACT_GELU_TANH, ACT_SILU, ACT_GELU_ERF, ACT_RELU = 0, 1, 2, 3, 4

_c = ctypes
_vp, _i32, _i64, _f32 = _c.c_void_p, _c.c_int32, _c.c_int64, _c.c_float


class GemmEpilogue(_c.Structure):
    """Mirror of ``svi_gemm_epilogue`` (include/svi_b200.h)."""
    _fields_ = [
        ("out", _vp), ("ldo", _i64), ("out_is_f32", _i32), ("act", _i32),
        ("bias", _vp), ("gate", _vp), ("residual", _vp), ("ldr", _i64),
        ("sumsq", _vp), ("sumsq_groups", _i32), ("sumsq_group_cols", _i32),
        ("ln_stats", _vp), ("ln_u", _vp), ("ln_dim", _i32), ("ln_eps", _f32),
        ("a_next", _vp), ("ld_an", _i64), ("g_next", _vp), ("row_stats", _vp),
        ("sumsq_parts", _i32), ("w_e4m3", _i32),
    ]


class ConvDesc(_c.Structure):
    """Mirror of ``svi_conv_desc`` (include/svi_b200.h)."""
    _fields_ = [
        ("x_ring", _vp), ("ring_slots", _i32), ("in_H", _i32), ("in_W", _i32), ("C_in", _i32),
        ("w_packed", _vp), ("w_rows", _i32), ("w_ld", _i64),
        ("kt", _i32), ("kh", _i32), ("kw", _i32), ("pad_h", _i32), ("pad_w", _i32),
        ("H", _i32), ("W", _i32), ("T", _i32),
        ("slot", _i32 * 12),
        ("C_out", _i32), ("tile_w", _i32),
        ("out", _vp), ("out_frame_stride", _i64), ("out_ld", _i32),
        ("n_split", _i32), ("split_offset", _i64),
        ("bias", _vp),
        ("residual", _vp), ("res_frame_stride", _i64), ("res_ld", _i32),
        ("next_ring", _vp), ("next_frame_stride", _i64), ("next_ld", _i32), ("next_slot", _i32 * 4),
        ("next_gamma", _vp), ("next_silu", _i32), ("write_f32", _i32),
        ("variant", _i32),
    ]


class GemmLoRA(_c.Structure):
    """Mirror of ``svi_gemm_lora`` (include/svi_b200_lora.h)."""
    _fields_ = [("U", _vp), ("ldu", _i64), ("B", _vp), ("ldb", _i64), ("R", _i32), ("group_cols", _i32)]


# name -> (restype, argtypes); must list every symbol the header declares (checked by tests)
SIGNATURES = {
    "svi_abi_version": (_i32, []),
    "svi_last_error": (_c.c_char_p, []),
    "svi_sm_count": (_i32, []),
    "svi_gemm_bf16": (_i32, [_vp, _i64, _vp, _i64, _i32, _i32, _i32, _c.POINTER(GemmEpilogue), _vp]),
    "svi_attn_fwd": (_i32, [_vp, _i64, _vp, _i64, _vp, _i64, _vp, _i64, _i32, _i32, _i32, _f32, _i32, _vp, _c.c_size_t, _vp]),
    "svi_attn_workspace_bytes": (_c.c_size_t, [_i32, _i32, _i32]),
    "svi_attn_fwd_qscale": (_i32, [_vp, _i64, _vp, _i64, _vp, _i64, _vp, _i64, _i32, _i32, _i32, _f32, _i32, _vp, _i32, _i32, _i32, _f32,
                                   _vp, _c.c_size_t, _vp]),
    "svi_attn_plan": (None, [_i32, _i32, _i32, _c.c_size_t, _c.POINTER(_i32), _c.POINTER(_i32)]),
    "svi_attn_fwd_sp": (_i32, [_vp, _i64, _vp, _i64, _vp, _i64, _vp, _i64, _i32, _i32, _i32, _f32, _vp, _c.c_uint32, _i32, _i32, _vp, _c.c_size_t, _vp]),
    "svi_sp_alloc": (_i32, [_c.c_size_t, _c.POINTER(_vp), _c.c_char_p]),
    "svi_sp_free": (_i32, [_vp]),
    "svi_sp_open": (_i32, [_c.c_char_p, _c.POINTER(_vp)]),
    "svi_sp_close": (_i32, [_vp]),
    "svi_sp_push": (_i32, [_vp, _c.POINTER(_vp), _c.POINTER(_vp), _i32, _c.c_size_t, _vp, _vp]),
    "svi_layernorm_modulate": (_i32, [_vp, _i32, _i32, _f32, _vp, _vp, _vp, _vp, _vp, _vp]),
    "svi_layernorm_modulate_split": (_i32, [_vp, _i32, _i32, _f32, _vp, _vp, _vp, _vp, _vp, _i64, _i32, _vp]),
    "svi_rmsnorm_rope": (_i32, [_vp, _i64, _i32, _i32, _vp, _i32, _i32, _i32, _f32, _vp, _vp, _vp, _i32, _vp]),
    "svi_qk_norm_rope": (_i32, [_vp, _i64, _i32, _i32, _vp, _i32, _i32, _f32, _vp, _vp, _vp, _vp, _i32, _vp]),
    "svi_patchify_gather_split": (_i32, [_vp, _i32, _vp, _i32, _i32, _i32, _i32, _vp, _i32, _vp]),
    "svi_split_f32_to_bf16x2": (_i32, [_vp, _i64, _i32, _i32, _i32, _vp, _i64, _i32, _vp]),
    "svi_zero": (_i32, [_vp, _c.c_size_t, _vp]),
    "svi_ln_fold_prepare": (_i32, [_vp, _i32, _i32, _vp, _vp, _vp]),
    "svi_ln_fold_combine": (_i32, [_vp, _i32, _vp, _vp, _vp, _vp]),
    "svi_patchify_gather": (_i32, [_vp, _i32, _vp, _i32, _i32, _i32, _i32, _vp, _i32, _vp]),
    "svi_unpatchify": (_i32, [_vp, _i64, _i32, _i32, _i32, _i32, _vp, _vp]),
    "svi_cfg_euler_step": (_i32, [_vp, _vp, _vp, _i64, _f32, _f32, _f32, _vp]),
    "svi_cast_f32_to_bf16": (_i32, [_vp, _vp, _i64, _vp]),
    "svi_cast_bf16_to_f32": (_i32, [_vp, _vp, _i64, _vp]),
    "svi_act_f32_to_bf16": (_i32, [_vp, _vp, _i64, _i32, _vp]),
    "svi_add_rows": (_i32, [_vp, _vp, _i32, _i32, _i32, _vp, _vp]),
    "svi_axpby": (_i32, [_vp, _f32, _vp, _f32, _vp, _i64, _vp]),
    "svi_embedding_gather": (_i32, [_vp, _i32, _vp, _i32, _i64, _vp, _vp]),
    "svi_rmsnorm_affine": (_i32, [_vp, _i32, _i32, _f32, _vp, _vp, _vp]),
    "svi_layernorm_f32": (_i32, [_vp, _i32, _i32, _f32, _vp, _vp, _vp, _vp]),
    "svi_mul_bf16": (_i32, [_vp, _vp, _vp, _i64, _vp]),
    "svi_attn_small": (_i32, [_vp, _i64, _vp, _i64, _vp, _i64, _vp, _i64, _i32, _i32, _i32, _i32, _f32, _vp, _vp, _vp, _vp]),
    "svi_conv3d_causal": (_i32, [_c.POINTER(ConvDesc), _vp]),
    "svi_vae_norm_act": (_i32, [_vp, _i64, _i32, _i64, _vp, _i32, _vp, _i32, _vp]),
    "svi_vae_upsample2x": (_i32, [_vp, _i32, _i32, _i32, _vp, _vp]),
    "svi_vae_space_to_depth": (_i32, [_vp, _i32, _i32, _i32, _vp, _vp]),
    "svi_vae_space_to_depth_act": (_i32, [_vp, _i32, _i32, _i32, _i32, _vp, _vp]),
    "svi_vae_from_planar": (_i32, [_vp, _i32, _i64, _i64, _vp, _vp, _vp, _i32, _i32, _vp]),
    "svi_vae_to_planar": (_i32, [_vp, _i64, _i32, _i64, _vp, _vp, _i32, _vp, _i64, _vp]),
    "svi_softmax_rows": (_i32, [_vp, _i32, _i32, _i64, _f32, _vp, _i64, _vp]),
    "svi_frames_to_uint8": (_i32, [_vp, _i64, _i64, _vp, _vp]),
    "svi_col_stats_workspace_bytes": (_c.c_size_t, [_i64, _i32]),
    "svi_col_stats": (_i32, [_vp, _i64, _i64, _i32, _vp, _vp, _vp, _c.c_size_t, _vp]),
    "svi_col_norm_act": (_i32, [_vp, _i64, _i64, _i32, _vp, _vp, _f32, _vp, _vp, _i32, _vp, _i64, _vp]),
    "svi_conv1d_gather": (_i32, [_vp, _i32, _i64, _i64, _i32, _i32, _i32, _i32, _i32, _i32, _i64, _i32, _vp, _i64, _i32, _vp]),
    "svi_interp_layernorm": (_i32, [_vp, _i64, _i64, _i32, _i64, _f32, _vp, _vp, _vp, _i64, _vp]),
}

# the same for include/svi_b200_lora.h
LORA_SIGNATURES = {
    "svi_gemm_lora_bf16": (_i32, [_vp, _i64, _vp, _i64, _i32, _i32, _i32, _c.POINTER(GemmEpilogue), _c.POINTER(GemmLoRA), _vp]),
}


class RifeConvDesc(_c.Structure):
    """Mirror of ``svi_rife_conv_desc`` (include/svi_b200_rife.h)."""
    _fields_ = [
        ("x", _vp), ("N", _i32), ("in_H", _i32), ("in_W", _i32), ("C_in", _i32),
        ("w_packed", _vp), ("w_rows", _i32), ("w_ld", _i64),
        ("kh", _i32), ("kw", _i32), ("pad_h", _i32), ("pad_w", _i32),
        ("H", _i32), ("W", _i32), ("C_out", _i32), ("phase_cols", _i32), ("tile_w", _i32),
        ("bias", _vp), ("prelu", _vp), ("residual", _vp),
        ("out", _vp), ("out_img_stride", _i64), ("out_ld", _i32),
        ("out_bf16", _vp), ("bf_img_stride", _i64), ("bf_ld", _i32), ("bf_s2d", _i32),
    ]


class RifeBlockInput(_c.Structure):
    """Mirror of ``svi_rife_block_input`` (include/svi_b200_rife.h)."""
    _fields_ = [
        ("img0", _vp), ("img1", _vp), ("img_stride", _i64), ("state", _vp),
        ("pairs", _i32), ("H", _i32), ("W", _i32), ("h", _i32), ("w", _i32),
        ("src_scale", _f32), ("flow_mul", _f32), ("out", _vp),
    ]


class RifeUpdate(_c.Structure):
    """Mirror of ``svi_rife_update`` (include/svi_b200_rife.h)."""
    _fields_ = [
        ("heads", _vp), ("heads_ld", _i32),
        ("pairs", _i32), ("H", _i32), ("W", _i32), ("h", _i32), ("w", _i32),
        ("src_scale", _f32), ("flow_mul", _f32),
        ("img0", _vp), ("img1", _vp), ("img_stride", _i64),
        ("state", _vp), ("first", _i32),
        ("merged", _vp), ("merged_stride", _i64), ("clip", _i32),
        ("rgb", _vp), ("rgb_stride", _i64),
    ]


# the same for include/svi_b200_rife.h
RIFE_SIGNATURES = {
    "svi_rife_stage_frames": (_i32, [_vp, _i64, _vp, _vp]),
    "svi_rife_block_input_launch": (_i32, [_c.POINTER(RifeBlockInput), _vp]),
    "svi_rife_conv2d": (_i32, [_c.POINTER(RifeConvDesc), _vp]),
    "svi_rife_update_warp": (_i32, [_c.POINTER(RifeUpdate), _vp]),
}


class EsrganConvDesc(_c.Structure):
    """Mirror of ``svi_esrgan_conv_desc`` (include/svi_b200_esrgan.h)."""
    _fields_ = [
        ("x", _vp), ("N", _i32), ("H", _i32), ("W", _i32), ("C_in", _i32), ("in_ld", _i32),
        ("w_packed", _vp), ("w_rows", _i32), ("w_ld", _i64),
        ("C_out", _i32), ("tile_w", _i32),
        ("bias", _vp), ("slope", _f32),
        ("residual", _vp), ("res_scale", _f32), ("residual2", _vp), ("res2_scale", _f32),
        ("out", _vp), ("f_ld", _i32),
        ("out_bf16", _vp), ("bf_ld", _i32), ("bf_up2", _i32),
        ("out_u8", _vp),
    ]


# the same for include/svi_b200_esrgan.h
ESRGAN_SIGNATURES = {
    "svi_esrgan_stage_frames": (_i32, [_vp, _i64, _vp, _vp]),
    "svi_esrgan_conv2d": (_i32, [_c.POINTER(EsrganConvDesc), _vp]),
}


class FastblendStepDesc(_c.Structure):
    """Mirror of ``svi_fastblend_step_desc`` (include/svi_b200_fastblend.h)."""
    _fields_ = [
        ("src_guide", _vp), ("src_style", _vp), ("tgt_guide", _vp), ("tgt_style", _vp),
        ("nnf_in", _vp), ("err_in", _vp), ("nnf_out", _vp), ("err_out", _vp),
        ("B", _i32), ("H", _i32), ("W", _i32), ("patch_size", _i32), ("mode", _i32), ("dir", _i32),
        ("draw", _c.c_uint32), ("radius", _i32), ("guide_weight", _f32),
    ]


class FastblendTableDesc(_c.Structure):
    """Mirror of ``svi_fastblend_table_desc`` (include/svi_b200_fastblend.h)."""
    _fields_ = [
        ("op", _i32), ("n_pix", _i64),
        ("a", _vp), ("a_type", _i32), ("sa", _c.c_double),
        ("b", _vp), ("b_type", _i32), ("sb", _c.c_double),
        ("c", _vp), ("c_type", _i32), ("sc", _c.c_double),
        ("out", _vp), ("out_type", _i32),
    ]


# the same for include/svi_b200_fastblend.h
FASTBLEND_SIGNATURES = {
    "svi_fastblend_stage_frames": (_i32, [_vp, _i64, _vp, _vp]),
    "svi_fastblend_downsample": (_i32, [_vp, _i32, _i32, _i32, _i32, _vp, _vp]),
    "svi_fastblend_nnf_identity": (_i32, [_vp, _i32, _i32, _i32, _vp]),
    "svi_fastblend_nnf_upscale": (_i32, [_vp, _i32, _i32, _i32, _vp, _vp]),
    "svi_fastblend_remap": (_i32, [_vp, _vp, _i32, _i32, _i32, _i32, _vp, _vp]),
    "svi_fastblend_step": (_i32, [_c.POINTER(FastblendStepDesc), _vp]),
    "svi_fastblend_table": (_i32, [_c.POINTER(FastblendTableDesc), _vp]),
}
FB_CURRENT, FB_NEIGHBOUR, FB_RANDOM = 0, 1, 2
FB_U8, FB_F32, FB_F64 = 0, 1, 2
FB_MEAN, FB_HALF, FB_WSUM = 0, 1, 2


class FastblendCandidateDesc(_c.Structure):
    """Mirror of ``svi_fastblend_candidate_desc`` (include/svi_b200_fastblend_modes.h)."""
    _fields_ = [
        ("nnf_in", _vp), ("nnf_out", _vp), ("B", _i32), ("H", _i32), ("W", _i32), ("mode", _i32), ("dir", _i32),
        ("draw", _c.c_uint32), ("radius", _i32), ("shift", _i32), ("pairwise", _i32),
    ]


class FastblendSelectDesc(_c.Structure):
    """Mirror of ``svi_fastblend_select_desc`` (include/svi_b200_fastblend_modes.h)."""
    _fields_ = [
        ("src_guide", _vp), ("src_style", _vp), ("tgt_guide", _vp), ("tgt_style", _vp), ("cand", _vp),
        ("nnf_in", _vp), ("err_in", _vp), ("nnf_out", _vp), ("err_out", _vp),
        ("B", _i32), ("H", _i32), ("W", _i32), ("patch_size", _i32), ("select", _i32), ("style_shared", _i32),
        ("pairwise", _i32), ("guide_weight", _f32),
    ]


# the same for include/svi_b200_fastblend_modes.h (the balanced / accurate / interpolation modes)
FASTBLEND_MODES_SIGNATURES = {
    "svi_fastblend_candidate": (_i32, [_c.POINTER(FastblendCandidateDesc), _vp]),
    "svi_fastblend_select": (_i32, [_c.POINTER(FastblendSelectDesc), _vp]),
    "svi_fastblend_batch_mean": (_i32, [_vp, _i32, _i64, _vp, _vp]),
    "svi_fastblend_running_mean": (_i32, [_vp, _i32, _c.c_double, _vp, _f32, _i64, _vp, _vp]),
    "svi_fastblend_to_u8": (_i32, [_vp, _i32, _i64, _vp, _vp]),
}
FB_TRACK = 3

# the same for include/svi_b200_unianimate.h
UNIANIMATE_SIGNATURES = {
    "svi_window_accumulate": (_i32, [_vp, _i32, _i32, _i64, _i32, _vp, _i32, _i32, _vp]),
    "svi_window_normalize": (_i32, [_vp, _vp, _i32, _i32, _i64, _vp, _vp]),
}

# the same for include/svi_b200_replace.h
REPLACE_SIGNATURES = {
    "svi_replace_mask_stage": (_i32, [_vp, _vp, _i32, _i32, _i64, _vp, _vp, _i32, _vp]),
}
SEG_U8, SEG_F32 = 0, 1

# the same for include/svi_b200_quality.h
QUALITY_SIGNATURES = {
    "svi_quality_attn": (_i32, [_vp, _i64, _vp, _i64, _vp, _i64, _vp, _i64, _i32, _i32, _i32, _i32, _f32, _i32, _vp]),
    "svi_quality_stage_pixels": (_i32, [_vp, _i32, _i32, _i32, _vp, _vp, _i32, _vp]),
    "svi_quality_embed_ln": (_i32, [_vp, _vp, _vp, _i32, _i32, _i32, _f32, _vp, _vp, _vp, _vp]),
    "svi_quality_quick_gelu": (_i32, [_vp, _i64, _i32, _i32, _vp, _i64, _vp]),
    "svi_quality_pool": (_i32, [_vp, _i64, _i32, _i32, _i32, _vp, _i32, _i64, _vp, _vp]),
    "svi_quality_score": (_i32, [_vp, _i32, _vp, _i32, _i32, _vp, _f32, _vp, _vp, _vp]),
}
QUALITY_MAX_L = 320
POOL_FIRST, POOL_ARGMAX, POOL_EOS = 0, 1, 2

# the same for include/svi_b200_reward.h
REWARD_SIGNATURES = {
    "svi_reward_attn": (_i32, [_vp, _i64, _vp, _i64, _vp, _i64, _vp, _i64, _i32, _i32, _i32, _i32, _i32, _i64, _vp, _i64,
                               _f32, _vp]),
    "svi_reward_layernorm": (_i32, [_vp, _i32, _i32, _f32, _vp, _vp, _vp, _vp, _vp]),
    "svi_reward_embed": (_i32, [_vp, _vp, _vp, _i32, _i32, _i32, _vp, _vp]),
    "svi_reward_swiglu": (_i32, [_vp, _i64, _i32, _i32, _vp, _i64, _vp]),
    "svi_reward_rope": (_i32, [_vp, _i64, _i32, _i32, _i32, _vp, _vp, _vp]),
    "svi_reward_cond_mask": (_i32, [_vp, _i32, _vp, _i32, _i32, _f32, _vp, _vp, _vp]),
    "svi_reward_head": (_i32, [_vp, _i64, _i32, _i32, _i32, _vp, _f32, _vp, _vp]),
}

# the same for include/svi_b200_processors.h
PROCESSORS_SIGNATURES = {
    "svi_luma_sum_u8": (_i32, [_vp, _i32, _i64, _vp, _vp]),
    "svi_enhance_blend_u8": (_i32, [_vp, _i32, _i64, _vp, _f32, _vp, _vp]),
    "svi_sharpen_u8": (_i32, [_vp, _i32, _i32, _i32, _f32, _vp, _vp]),
    "svi_rife_average_u8": (_i32, [_vp, _vp, _i32, _i64, _vp, _vp]),
}

_lib = None


def lib_path():
    return _LIB_PATH


def load():
    """Load the kernel library (once).  Raises RuntimeError if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_LIB_PATH):
        raise RuntimeError(
            f"svi_b200: native kernel library not found at {_LIB_PATH}. Build it with "
            f"`python -c 'import __graft_entry__ as g; g.build()'` (or `make`) — there is no CPU fallback.")
    lib = ctypes.CDLL(_LIB_PATH)
    for name, (res, args) in (SIGNATURES | LORA_SIGNATURES | RIFE_SIGNATURES | ESRGAN_SIGNATURES |
                        FASTBLEND_SIGNATURES | FASTBLEND_MODES_SIGNATURES | UNIANIMATE_SIGNATURES | REPLACE_SIGNATURES | QUALITY_SIGNATURES |
                        REWARD_SIGNATURES | PROCESSORS_SIGNATURES).items():
        fn = getattr(lib, name)  # AttributeError if the symbol is missing: fail loudly
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def require_cuda(device, what):
    """Every engine calls this first: the kernels exist for sm_90a only, so anything but a CUDA device is an error (there is
    no CPU path), and the library must be loadable."""
    if torch.device(device).type != "cuda":
        raise RuntimeError(f"svi_b200: {what} runs only on a CUDA device (sm_90a kernels; no CPU fallback)")
    load()


def _check(rc, name):
    if rc != 0:
        msg = load().svi_last_error().decode("utf-8", "replace")
        raise RuntimeError(f"{name} failed (status {rc}): {msg}")


def _stream():
    return _vp(torch.cuda.current_stream().cuda_stream)


def _ptr(t, dtype=None, name="tensor"):
    if t is None:
        return None
    if not t.is_cuda:
        raise RuntimeError(f"svi_b200: {name} must be a CUDA tensor (no CPU fallback)")
    if dtype is not None and t.dtype != dtype:
        raise RuntimeError(f"svi_b200: {name} must be {dtype}, got {t.dtype}")
    return _vp(t.data_ptr())


def _rowmajor(t, name):
    if t.dim() != 2 or t.stride(1) != 1:
        raise RuntimeError(f"svi_b200: {name} must be 2-D with unit inner stride, got {tuple(t.shape)} / {t.stride()}")
    return t.stride(0)


def sm_count():
    return load().svi_sm_count()


def gemm(a, w, out, bias=None, act=ACT_NONE, gate=None, residual=None, sumsq=None, sumsq_group_cols=0, ln=None, emit=None):
    """out = epilogue(a[M,K] @ w[N,K]^T); a bf16, w bf16 or float8_e4m3fn; out f32 or bf16 (may be a column slice view).
    An e4m3 w is converted exactly to bf16 inside the kernel (weight-only FP8): the result is bit-identical to passing
    w.to(torch.bfloat16); it needs K % 16 == 0 and a row stride that is a multiple of 16.
    ln = (stats f32 [M,2], u f32 [N], dim, eps): LayerNorm folded into the GEMM (consumer side, svi_gemm_epilogue);
    emit = (a_next bf16 [M,N], g_next f32 [N], row_stats f32 [M,2]): producer side."""
    ep, lda, ldw, (M, N, K) = _gemm_args(a, w, out, bias, act, gate, residual, sumsq, sumsq_group_cols, ln, emit)
    rc = load().svi_gemm_bf16(_ptr(a, torch.bfloat16, "a"), lda, _ptr(w, name="w"), ldw,
                              M, N, K, ctypes.byref(ep), _stream())
    _check(rc, "svi_gemm_bf16")
    return out


def gemm_lora(a, w, out, u, b, R, group_cols=0, bias=None, act=ACT_NONE, gate=None, residual=None, sumsq=None,
              sumsq_group_cols=0, ln=None, emit=None):
    """gemm() plus an unmerged LoRA term ahead of the epilogue (svi_gemm_lora_bf16, include/svi_b200_lora.h):
    out = epilogue(a @ w^T + u[:, g R:(g+1) R] @ b^T) with g = column // group_cols (0: one group).  u bf16 [M, >= groups R]
    holds alpha * x A^T (row-strided views allowed, e.g. a column offset into a wider U), b bf16 [N, >= R]; R % 64 == 0.
    act: none or GELU-tanh; ln / emit (the LayerNorm fold) are refused by the library."""
    ep, lda, ldw, (M, N, K) = _gemm_args(a, w, out, bias, act, gate, residual, sumsq, sumsq_group_cols, ln, emit)
    if u.shape[0] != M or b.shape[0] != N:
        raise RuntimeError(f"svi_b200.gemm_lora: u must have M={M} rows and b N={N} rows, got u{tuple(u.shape)} b{tuple(b.shape)}")
    groups = N // group_cols if group_cols else 1
    if u.shape[1] < groups * R or b.shape[1] < R:
        raise RuntimeError(f"svi_b200.gemm_lora: u needs >= {groups} x R columns and b >= R (R={R}), got u{tuple(u.shape)} "
                           f"b{tuple(b.shape)}")
    lo = GemmLoRA()
    lo.U, lo.ldu = _ptr(u, torch.bfloat16, "u"), _rowmajor(u, "u")
    lo.B, lo.ldb = _ptr(b, torch.bfloat16, "b"), _rowmajor(b, "b")
    lo.R, lo.group_cols = int(R), int(group_cols)
    rc = load().svi_gemm_lora_bf16(_ptr(a, torch.bfloat16, "a"), lda, _ptr(w, name="w"), ldw, M, N, K, ctypes.byref(ep),
                                   ctypes.byref(lo), _stream())
    _check(rc, "svi_gemm_lora_bf16")
    return out


def _gemm_args(a, w, out, bias, act, gate, residual, sumsq, sumsq_group_cols, ln, emit):
    """(epilogue, lda, ldw, (M, N, K)) of one gemm / gemm_lora call, after the host-side checks."""
    if a.dtype != torch.bfloat16:
        raise RuntimeError(f"svi_b200.gemm: a must be bf16 (only the weight may be float8_e4m3fn), got {a.dtype}")
    if w.dtype not in (torch.bfloat16, torch.float8_e4m3fn):
        raise RuntimeError(f"svi_b200.gemm: w must be bf16 or float8_e4m3fn (e5m2 and other formats are not supported), "
                           f"got {w.dtype}")
    if emit is not None and emit[0].dtype != torch.bfloat16:
        raise RuntimeError(f"svi_b200.gemm: emit's a_next must be bf16, got {emit[0].dtype}")
    lda, ldw, ldo = _rowmajor(a, "a"), _rowmajor(w, "w"), _rowmajor(out, "out")
    M, K = a.shape
    N = w.shape[0]
    if w.shape[1] != K or out.shape[0] != M or out.shape[1] != N:
        raise RuntimeError(f"svi_b200.gemm: shape mismatch a{tuple(a.shape)} w{tuple(w.shape)} out{tuple(out.shape)}")
    w_e4m3 = w.dtype == torch.float8_e4m3fn
    if w_e4m3 and (K % 16 or ldw % 16):
        raise RuntimeError(f"svi_b200.gemm: an e4m3 w needs K and its row stride to be multiples of 16 (K={K}, stride={ldw})")
    ep = GemmEpilogue()
    ep.w_e4m3 = int(w_e4m3)
    ep.out = _ptr(out, name="out")
    ep.ldo = ldo
    if out.dtype == torch.float32:
        ep.out_is_f32 = 1
    elif out.dtype == torch.bfloat16:
        ep.out_is_f32 = 0
    else:
        raise RuntimeError(f"svi_b200.gemm: out must be f32 or bf16, got {out.dtype}")
    ep.act = act
    ep.bias = _ptr(bias, torch.float32, "bias")
    ep.gate = _ptr(gate, torch.float32, "gate")
    if residual is not None:
        ep.residual = _ptr(residual, torch.float32, "residual")
        ep.ldr = _rowmajor(residual, "residual")
    if sumsq is not None:
        # [M, groups]: atomicAdd per group (the buffer must be zero);  [M, groups, parts] contiguous, parts = group_cols / 128:
        # every 128-column segment stores its partial sum (reproducible, no zeroing) — see svi_gemm_epilogue.sumsq_parts
        ep.sumsq = _ptr(sumsq, torch.float32, "sumsq")
        ep.sumsq_groups = sumsq.shape[1]
        ep.sumsq_group_cols = sumsq_group_cols
        if sumsq.dim() == 3:
            if not sumsq.is_contiguous() or sumsq.shape[2] * 128 != sumsq_group_cols:
                raise RuntimeError("svi_b200.gemm: partial sumsq must be contiguous [M, groups, sumsq_group_cols / 128]")
            ep.sumsq_parts = sumsq.shape[2]
    if ln is not None:
        stats, u, dim, eps = ln
        if tuple(stats.shape) != (M, 2) or not stats.is_contiguous() or u.numel() != N:
            raise RuntimeError("svi_b200.gemm: ln stats must be contiguous [M,2] and u [N]")
        ep.ln_stats, ep.ln_u = _ptr(stats, torch.float32, "ln_stats"), _ptr(u, torch.float32, "ln_u")
        ep.ln_dim, ep.ln_eps = int(dim), float(eps)
    if emit is not None:
        a_next, g_next, row_stats = emit
        if a_next.shape[0] != M or a_next.shape[1] != N or tuple(row_stats.shape) != (M, 2) or not row_stats.is_contiguous():
            raise RuntimeError("svi_b200.gemm: emit needs a_next [M,N] and contiguous row_stats [M,2]")
        ep.a_next, ep.ld_an = _ptr(a_next, torch.bfloat16, "a_next"), _rowmajor(a_next, "a_next")
        ep.g_next, ep.row_stats = _ptr(g_next, torch.float32, "g_next"), _ptr(row_stats, torch.float32, "row_stats")
    return ep, lda, ldw, (M, N, K)


def attention(q, k, v, out, num_heads, scale=None, accumulate=False, workspace=None):
    """out[Lq, H*128] (+)= softmax(q k^T * scale) v per head; q,k,v,out bf16 2-D (column-slice views allowed).
    workspace: optional device scratch (attention_workspace_bytes) that lets the launch slice its last wave of units."""
    ldq, ldk, ldv, ldo = (_rowmajor(t, n) for t, n in ((q, "q"), (k, "k"), (v, "v"), (out, "out")))
    if scale is None:
        scale = 128 ** -0.5
    rc = load().svi_attn_fwd(_ptr(q, torch.bfloat16, "q"), ldq, _ptr(k, torch.bfloat16, "k"), ldk,
                             _ptr(v, torch.bfloat16, "v"), ldv, _ptr(out, torch.bfloat16, "out"), ldo,
                             q.shape[0], k.shape[0], num_heads, float(scale), int(bool(accumulate)),
                             *_workspace(workspace), _stream())
    _check(rc, "svi_attn_fwd")
    return out


def attention_qscale(q, k, v, out, num_heads, q_sumsq, q_dim, q_eps, scale=None, accumulate=False, workspace=None):
    """attention() on an UN-normalised q whose full-width RMSNorm factor rsqrt(q_sumsq[r] / q_dim + q_eps) is applied inside
    the softmax (svi_attn_fwd_qscale); q_sumsq f32 [Lq, n] (column 0 is used) or [Lq, n, parts] (the partials of group 0)."""
    ldq, ldk, ldv, ldo = (_rowmajor(t, n) for t, n in ((q, "q"), (k, "k"), (v, "v"), (out, "out")))
    if scale is None:
        scale = 128 ** -0.5
    if q_sumsq.shape[0] != q.shape[0]:
        raise RuntimeError("svi_b200.attention_qscale: q_sumsq must have one row per query row")
    rc = load().svi_attn_fwd_qscale(_ptr(q, torch.bfloat16, "q"), ldq, _ptr(k, torch.bfloat16, "k"), ldk,
                                    _ptr(v, torch.bfloat16, "v"), ldv, _ptr(out, torch.bfloat16, "out"), ldo,
                                    q.shape[0], k.shape[0], num_heads, float(scale), int(bool(accumulate)),
                                    _ptr(q_sumsq, torch.float32, "q_sumsq"), *_sumsq_layout(q_sumsq), int(q_dim),
                                    float(q_eps), *_workspace(workspace), _stream())
    _check(rc, "svi_attn_fwd_qscale")
    return out


def _sumsq_layout(ss):
    """(floats per row, partials per group) of a row-sum-of-squares buffer: [M, groups] or contiguous [M, groups, parts]."""
    if ss.dim() == 3:
        if not ss.is_contiguous():
            raise RuntimeError("svi_b200: a partial sumsq buffer [M, groups, parts] must be contiguous")
        return ss.shape[1] * ss.shape[2], ss.shape[2]
    return _rowmajor(ss, "sumsq"), 0


def _workspace(ws):
    if ws is None:
        return None, 0
    if not ws.is_cuda or not ws.is_contiguous():
        raise RuntimeError("svi_b200: attention workspace must be a contiguous CUDA tensor")
    return _vp(ws.data_ptr()), ws.numel() * ws.element_size()


def attention_plan(units, kv_tiles, sms, workspace_bytes):
    """(n_full, split) the attention launch would use — pure host logic (svi_attn_plan)."""
    a, b = _i32(), _i32()
    load().svi_attn_plan(units, kv_tiles, sms, workspace_bytes, ctypes.byref(a), ctypes.byref(b))
    return a.value, b.value


def attention_workspace_bytes(Lq, Lk, num_heads):
    return int(load().svi_attn_workspace_bytes(Lq, Lk, num_heads))


def attention_sp(q, k, v, out, num_heads, kv_flags, kv_epoch, kv_chunk_rows, kv_self_chunk, scale=None, workspace=None):
    """Self-attention over the rank's full K|V buffer whose remote rows are still being pushed by the peers
    (svi_attn_fwd_sp): kv_flags int32 [n_chunks] device tensor inside the symmetric allocation."""
    ldq, ldk, ldv, ldo = (_rowmajor(t, n) for t, n in ((q, "q"), (k, "k"), (v, "v"), (out, "out")))
    if scale is None:
        scale = 128 ** -0.5
    rc = load().svi_attn_fwd_sp(_ptr(q, torch.bfloat16, "q"), ldq, _ptr(k, torch.bfloat16, "k"), ldk,
                                _ptr(v, torch.bfloat16, "v"), ldv, _ptr(out, torch.bfloat16, "out"), ldo,
                                q.shape[0], k.shape[0], num_heads, float(scale), _ptr(kv_flags, torch.int32, "kv_flags"),
                                int(kv_epoch) & 0xFFFFFFFF, int(kv_chunk_rows), int(kv_self_chunk), *_workspace(workspace),
                                _stream())
    _check(rc, "svi_attn_fwd_sp")
    return out


class _RawCuda:
    """Exposes a raw device allocation to torch through __cuda_array_interface__ (zero copy)."""

    def __init__(self, ptr, nbytes):
        self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "version": 3}


def sp_alloc(nbytes, device):
    """Symmetric (peer-mappable) allocation: returns (ptr:int, handle:bytes[64], uint8 tensor view of it)."""
    ptr = _vp()
    handle = ctypes.create_string_buffer(64)
    _check(load().svi_sp_alloc(nbytes, ctypes.byref(ptr), handle), "svi_sp_alloc")
    view = torch.as_tensor(_RawCuda(ptr.value, nbytes), device=device)
    return ptr.value, handle.raw, view


def sp_free(ptr):
    _check(load().svi_sp_free(_vp(ptr)), "svi_sp_free")


def sp_open(handle):
    ptr = _vp()
    _check(load().svi_sp_open(handle, ctypes.byref(ptr)), "svi_sp_open")
    return ptr.value


def sp_close(ptr):
    _check(load().svi_sp_close(_vp(ptr)), "svi_sp_close")


def sp_push(src_ptr, peer_dst, peer_flag, nbytes, epoch_word_ptr, stream):
    """Copy-engine push of this rank's rows + flag word to every peer on `stream` (a torch.cuda.Stream)."""
    n = len(peer_dst)
    arr = _vp * n
    rc = load().svi_sp_push(_vp(src_ptr), arr(*peer_dst), arr(*peer_flag), n, nbytes, _vp(epoch_word_ptr),
                            _vp(stream.cuda_stream))
    _check(rc, "svi_sp_push")


def layernorm_modulate(x, out, eps, gamma=None, beta=None, scale=None, shift=None):
    """out(bf16)[M,D] = LN(x f32 [M,D]) (*gamma + beta) * (1 + scale) + shift."""
    M, D = x.shape
    if not x.is_contiguous() or not out.is_contiguous():
        raise RuntimeError("svi_b200.layernorm_modulate: x and out must be contiguous")
    rc = load().svi_layernorm_modulate(_ptr(x, torch.float32, "x"), M, D, float(eps),
                                       _ptr(gamma, torch.float32, "gamma"), _ptr(beta, torch.float32, "beta"),
                                       _ptr(scale, torch.float32, "scale"), _ptr(shift, torch.float32, "shift"),
                                       _ptr(out, torch.bfloat16, "out"), _stream())
    _check(rc, "svi_layernorm_modulate")
    return out


def layernorm_modulate_split(x, out, eps, gamma=None, beta=None, scale=None, shift=None):
    """out bf16 [M, 2D]: columns [0, D) = bf16(v), [D, 2D) = bf16(v - bf16(v)), v = layernorm_modulate(x)."""
    M, D = x.shape
    if not x.is_contiguous() or not out.is_contiguous() or tuple(out.shape) != (M, 2 * D):
        raise RuntimeError("svi_b200.layernorm_modulate_split: x [M,D] and out [M,2D] must be contiguous")
    rc = load().svi_layernorm_modulate_split(_ptr(x, torch.float32, "x"), M, D, float(eps),
                                             _ptr(gamma, torch.float32, "gamma"), _ptr(beta, torch.float32, "beta"),
                                             _ptr(scale, torch.float32, "scale"), _ptr(shift, torch.float32, "shift"),
                                             _ptr(out, torch.bfloat16, "out"), 2 * D, D, _stream())
    _check(rc, "svi_layernorm_modulate_split")
    return out


def qk_norm_rope(qk, sumsq, eps, wq, wk, rope_cos, rope_sin, row_offset=0):
    """In place on bf16 qk[M, 2D] (q | k side by side, row-strided view allowed): RMSNorm + RoPE of both in one launch;
    sumsq f32 [M, >=2] (columns 0, 1)."""
    ld = _rowmajor(qk, "qk")
    M, D2 = qk.shape
    rc = load().svi_qk_norm_rope(_ptr(qk, torch.bfloat16, "qk"), ld, M, D2 // 2, _ptr(sumsq, torch.float32, "sumsq"),
                                 *_sumsq_layout(sumsq), float(eps), _ptr(wq, torch.float32, "wq"),
                                 _ptr(wk, torch.float32, "wk"), _ptr(rope_cos, torch.float32, "rope_cos"),
                                 _ptr(rope_sin, torch.float32, "rope_sin"), row_offset, _stream())
    _check(rc, "svi_qk_norm_rope")
    return qk


def split_f32_to_bf16x2(src, dst, act=ACT_NONE):
    """dst bf16 [M, 2K] = [bf16(v) | bf16(v - bf16(v))], v = act(src f32 [M, K]) (row-strided views allowed)."""
    M, K = src.shape
    if tuple(dst.shape) != (M, 2 * K):
        raise RuntimeError("svi_b200.split_f32_to_bf16x2: dst must be [M, 2K]")
    rc = load().svi_split_f32_to_bf16x2(_ptr(src, torch.float32, "src"), _rowmajor(src, "src"), M, K, act,
                                        _ptr(dst, torch.bfloat16, "dst"), _rowmajor(dst, "dst"), K, _stream())
    _check(rc, "svi_split_f32_to_bf16x2")
    return dst


def ln_fold_prepare(mods, layers, g_out, rows):
    """mods f32 [>= 6*layers, D] -> g_out f32 [layers, 2, D] (1 + scale), rows bf16 [layers, 2, 4, D] (svi_ln_fold_prepare)."""
    D = mods.shape[1]
    if not (mods.is_contiguous() and g_out.is_contiguous() and rows.is_contiguous()) or g_out.numel() != layers * 2 * D \
            or rows.numel() != layers * 8 * D:
        raise RuntimeError("svi_b200.ln_fold_prepare: contiguous mods [6L,D], g_out [L,2,D], rows [L,2,4,D] required")
    _check(load().svi_ln_fold_prepare(_ptr(mods, torch.float32, "mods"), layers, D, _ptr(g_out, torch.float32, "g_out"),
                                      _ptr(rows, torch.bfloat16, "rows"), _stream()), "svi_ln_fold_prepare")


def ln_fold_combine(o4, bias, u, c):
    """o4 f32 [4, N] -> u = o4[0] + o4[1], c = o4[2] + o4[3] + bias (svi_ln_fold_combine); u, c contiguous f32 [N]."""
    N = o4.shape[1]
    if not o4.is_contiguous() or u.numel() != N or c.numel() != N or not u.is_contiguous() or not c.is_contiguous():
        raise RuntimeError("svi_b200.ln_fold_combine: contiguous o4 [4,N], u [N], c [N] required")
    _check(load().svi_ln_fold_combine(_ptr(o4, torch.float32, "o4"), N, _ptr(bias, torch.float32, "bias"),
                                      _ptr(u, torch.float32, "u"), _ptr(c, torch.float32, "c"), _stream()), "svi_ln_fold_combine")


def zero_(t):
    """t.zero_() as one cudaMemsetAsync node on the current stream (contiguous CUDA tensor)."""
    if not t.is_cuda or not t.is_contiguous():
        raise RuntimeError("svi_b200.zero_: contiguous CUDA tensor required (no CPU fallback)")
    _check(load().svi_zero(_vp(t.data_ptr()), t.numel() * t.element_size(), _stream()), "svi_zero")
    return t


def rmsnorm_rope(t, sumsq, sumsq_col, eps, weight, rope_cos=None, rope_sin=None, row_offset=0):
    """In place on bf16 t[M, D] (row-strided view allowed): full-width RMSNorm + optional RoPE."""
    ldt = _rowmajor(t, "t")
    M, D = t.shape
    ss_ld, ss_parts = _sumsq_layout(sumsq)
    rc = load().svi_rmsnorm_rope(_ptr(t, torch.bfloat16, "t"), ldt, M, D, _ptr(sumsq, torch.float32, "sumsq"),
                                 ss_ld, sumsq_col, ss_parts, float(eps), _ptr(weight, torch.float32, "weight"),
                                 _ptr(rope_cos, torch.float32, "rope_cos"), _ptr(rope_sin, torch.float32, "rope_sin"),
                                 row_offset, _stream())
    _check(rc, "svi_rmsnorm_rope")
    return t


def patchify_gather(x, y, tokens, split=False):
    """x f32 [C0,F,H,W] (+ y f32 [C1,F,H,W]) -> tokens bf16 [L, Kpad]; split: tokens [L, 2 Kpad] = [hi | lo] two-term form."""
    C0, F, H, W = x.shape
    C1 = 0 if y is None else y.shape[0]
    if not x.is_contiguous() or (y is not None and not y.is_contiguous()) or not tokens.is_contiguous():
        raise RuntimeError("svi_b200.patchify_gather: tensors must be contiguous")
    fn = load().svi_patchify_gather_split if split else load().svi_patchify_gather
    rc = fn(_ptr(x, torch.float32, "x"), C0, _ptr(y, torch.float32, "y"), C1, F, H, W,
            _ptr(tokens, torch.bfloat16, "tokens"), tokens.shape[1] // (2 if split else 1), _stream())
    _check(rc, "svi_patchify_gather")
    return tokens


def unpatchify(head_out, out):
    """head_out f32 [L, ld>=4C] -> out f32 [C,F,H,W]."""
    C, F, H, W = out.shape
    rc = load().svi_unpatchify(_ptr(head_out, torch.float32, "head_out"), _rowmajor(head_out, "head_out"),
                               C, F, H, W, _ptr(out, torch.float32, "out"), _stream())
    _check(rc, "svi_unpatchify")
    return out


def cfg_euler_step(latents, v_cond, v_uncond, cfg, sigma, sigma_next):
    rc = load().svi_cfg_euler_step(_ptr(latents, torch.float32, "latents"), _ptr(v_cond, torch.float32, "v_cond"),
                                   _ptr(v_uncond, torch.float32, "v_uncond"), latents.numel(), float(cfg),
                                   float(sigma), float(sigma_next), _stream())
    _check(rc, "svi_cfg_euler_step")
    return latents


def cast_f32_to_bf16(src, dst, act=ACT_NONE):
    if act == ACT_NONE:
        rc = load().svi_cast_f32_to_bf16(_ptr(src, torch.float32, "src"), _ptr(dst, torch.bfloat16, "dst"),
                                         src.numel(), _stream())
    else:
        rc = load().svi_act_f32_to_bf16(_ptr(src, torch.float32, "src"), _ptr(dst, torch.bfloat16, "dst"),
                                        src.numel(), act, _stream())
    _check(rc, "svi_cast_f32_to_bf16")
    return dst


def cast_bf16_to_f32(src, dst):
    rc = load().svi_cast_bf16_to_f32(_ptr(src, torch.bfloat16, "src"), _ptr(dst, torch.float32, "dst"),
                                     src.numel(), _stream())
    _check(rc, "svi_cast_bf16_to_f32")
    return dst


def add_rows(table, t, out):
    rows, D = table.shape
    if not (table.is_contiguous() and t.is_contiguous() and out.is_contiguous()) or rows % t.shape[0]:
        raise RuntimeError("svi_b200.add_rows: contiguous tensors with rows % rows_t == 0 required")
    rc = load().svi_add_rows(_ptr(table, torch.float32, "table"), _ptr(t, torch.float32, "t"), rows, t.shape[0], D,
                             _ptr(out, torch.float32, "out"), _stream())
    _check(rc, "svi_add_rows")
    return out


def axpby(a, alpha, b, beta, out):
    """out = alpha * a + beta * b (f32, same shape, contiguous; out may alias a or b)."""
    if not (a.is_contiguous() and b.is_contiguous() and out.is_contiguous()) or a.shape != b.shape or a.shape != out.shape:
        raise RuntimeError("svi_b200.axpby: a, b, out must be contiguous and of one shape")
    rc = load().svi_axpby(_ptr(a, torch.float32, "a"), float(alpha), _ptr(b, torch.float32, "b"), float(beta),
                          _ptr(out, torch.float32, "out"), a.numel(), _stream())
    _check(rc, "svi_axpby")
    return out


# --------------------------------------------------------------------------------------------- encoders
def embedding_gather(ids, table, out):
    """out f32 [n, dim] = rows ids (int64 [n]) of table bf16 [vocab, dim]."""
    n, (vocab, dim) = ids.numel(), table.shape
    if ids.dtype != torch.int64 or not ids.is_contiguous() or not table.is_contiguous() or not out.is_contiguous():
        raise RuntimeError("svi_b200.embedding_gather: ids must be contiguous int64, table / out contiguous")
    rc = load().svi_embedding_gather(_ptr(ids, name="ids"), n, _ptr(table, torch.bfloat16, "table"), dim, vocab,
                                     _ptr(out, torch.float32, "out"), _stream())
    _check(rc, "svi_embedding_gather")
    return out


def rmsnorm_affine(x, weight, eps, out):
    M, D = x.shape
    if not x.is_contiguous() or not out.is_contiguous():
        raise RuntimeError("svi_b200.rmsnorm_affine: x and out must be contiguous")
    rc = load().svi_rmsnorm_affine(_ptr(x, torch.float32, "x"), M, D, float(eps), _ptr(weight, torch.float32, "weight"),
                                   _ptr(out, torch.bfloat16, "out"), _stream())
    _check(rc, "svi_rmsnorm_affine")
    return out


def layernorm_f32(x, gamma, beta, eps, out):
    M, D = x.shape
    if not x.is_contiguous() or not out.is_contiguous():
        raise RuntimeError("svi_b200.layernorm_f32: x and out must be contiguous")
    rc = load().svi_layernorm_f32(_ptr(x, torch.float32, "x"), M, D, float(eps), _ptr(gamma, torch.float32, "gamma"),
                                  _ptr(beta, torch.float32, "beta"), _ptr(out, torch.float32, "out"), _stream())
    _check(rc, "svi_layernorm_f32")
    return out


def mul_bf16(a, b, out):
    if not (a.is_contiguous() and b.is_contiguous() and out.is_contiguous()) or a.shape != b.shape or a.shape != out.shape:
        raise RuntimeError("svi_b200.mul_bf16: a, b, out must be contiguous and of one shape")
    rc = load().svi_mul_bf16(_ptr(a, torch.bfloat16, "a"), _ptr(b, torch.bfloat16, "b"), _ptr(out, torch.bfloat16, "out"),
                             a.numel(), _stream())
    _check(rc, "svi_mul_bf16")
    return out


def attention_small(q, k, v, out, num_heads, head_dim, scale, bias_table=None, bucket=None, key_mask=None):
    """Short-sequence attention with any head_dim <= 128, optional bucketed relative-position bias and key mask."""
    ldq, ldk, ldv, ldo = (_rowmajor(t, n) for t, n in ((q, "q"), (k, "k"), (v, "v"), (out, "out")))
    if bucket is not None and (bucket.dtype != torch.int32 or tuple(bucket.shape) != (q.shape[0], k.shape[0]) or not bucket.is_contiguous()):
        raise RuntimeError("svi_b200.attention_small: bucket must be contiguous int32 [Lq, Lk]")
    if key_mask is not None and (key_mask.dtype != torch.int32 or key_mask.numel() != k.shape[0]):
        raise RuntimeError("svi_b200.attention_small: key_mask must be int32 [Lk]")
    rc = load().svi_attn_small(_ptr(q, torch.bfloat16, "q"), ldq, _ptr(k, torch.bfloat16, "k"), ldk, _ptr(v, torch.bfloat16, "v"), ldv,
                               _ptr(out, torch.bfloat16, "out"), ldo, q.shape[0], k.shape[0], num_heads, head_dim, float(scale),
                               _ptr(bias_table, torch.float32, "bias_table"), _ptr(bucket, name="bucket"),
                               _ptr(key_mask, name="key_mask"), _stream())
    _check(rc, "svi_attn_small")
    return out


# --------------------------------------------------------------------------------------------- VAE
def conv3d_causal(desc):
    """Launch svi_conv3d_causal with a filled ConvDesc (pointers as ints)."""
    _check(load().svi_conv3d_causal(ctypes.byref(desc), _stream()), "svi_conv3d_causal")


def vae_norm_act(x, n_pix, C, ldx, gamma, silu, out, Cpad):
    rc = load().svi_vae_norm_act(_ptr(x, torch.float32, "x"), n_pix, C, ldx, _ptr(gamma, torch.float32, "gamma"),
                                 int(bool(silu)), _ptr(out, torch.bfloat16, "out"), Cpad, _stream())
    _check(rc, "svi_vae_norm_act")
    return out


def vae_upsample2x(x, H, W, C, out):
    _check(load().svi_vae_upsample2x(_ptr(x, torch.float32, "x"), H, W, C, _ptr(out, torch.bfloat16, "out"), _stream()),
           "svi_vae_upsample2x")
    return out


def vae_space_to_depth(x, H, W, C, out):
    _check(load().svi_vae_space_to_depth(_ptr(x, torch.float32, "x"), H, W, C, _ptr(out, torch.bfloat16, "out"), _stream()),
           "svi_vae_space_to_depth")
    return out


def vae_space_to_depth_act(x, H, W, C, act, out):
    _check(load().svi_vae_space_to_depth_act(_ptr(x, torch.float32, "x"), H, W, C, act, _ptr(out, torch.bfloat16, "out"), _stream()),
           "svi_vae_space_to_depth_act")
    return out


def vae_from_planar(x, C, n_pix, scale, shift, out, ldo, out_is_bf16, ldc=None):
    rc = load().svi_vae_from_planar(_ptr(x, torch.float32, "x"), C, n_pix, n_pix if ldc is None else ldc,
                                    _ptr(scale, torch.float32, "scale"), _ptr(shift, torch.float32, "shift"),
                                    _ptr(out, name="out"), ldo, int(bool(out_is_bf16)), _stream())
    _check(rc, "svi_vae_from_planar")
    return out


def vae_to_planar(x, ldx, C, n_pix, pre_shift, scale, clamp, out, ldc=None):
    rc = load().svi_vae_to_planar(_ptr(x, torch.float32, "x"), ldx, C, n_pix, _ptr(pre_shift, torch.float32, "pre_shift"),
                                  _ptr(scale, torch.float32, "scale"), int(bool(clamp)), _ptr(out, torch.float32, "out"),
                                  n_pix if ldc is None else ldc, _stream())
    _check(rc, "svi_vae_to_planar")
    return out


def frames_to_uint8(video, out):
    """video f32 [3, T, H, W] (contiguous, CUDA) -> out uint8 [T, H, W, 3]: clip((v + 1) * 127.5, 0, 255) truncated."""
    C, T, H, W = video.shape
    if C != 3 or not video.is_contiguous() or not out.is_contiguous() or out.dtype != torch.uint8 or out.numel() != 3 * T * H * W:
        raise RuntimeError("svi_b200.frames_to_uint8: video must be contiguous f32 [3,T,H,W], out contiguous uint8 [T,H,W,3]")
    _check(load().svi_frames_to_uint8(_ptr(video, torch.float32, "video"), T * H * W, T * H * W, _ptr(out, name="out"), _stream()),
           "svi_frames_to_uint8")
    return out


def softmax_rows(s, N, scale, p):
    rc = load().svi_softmax_rows(_ptr(s, torch.float32, "s"), s.shape[0], N, _rowmajor(s, "s"), float(scale),
                                 _ptr(p, torch.bfloat16, "p"), _rowmajor(p, "p"), _stream())
    _check(rc, "svi_softmax_rows")
    return p


# --------------------------------------------------------------------------------------------- wav2vec2 audio encoder
def col_stats_workspace_bytes(T, C):
    return int(load().svi_col_stats_workspace_bytes(int(T), int(C)))


def col_stats(x, mean, var, workspace):
    """mean / var f32 [C] = per-column mean and biased variance of x f32 [T, C] (row-strided view allowed) over its rows;
    reproducible (fixed-order fp64 reduction).  workspace: CUDA tensor of >= col_stats_workspace_bytes(T, C) bytes."""
    T, C = x.shape
    if mean.numel() != C or var.numel() != C or not mean.is_contiguous() or not var.is_contiguous():
        raise RuntimeError("svi_b200.col_stats: mean and var must be contiguous [C]")
    if not workspace.is_cuda or not workspace.is_contiguous():
        raise RuntimeError("svi_b200.col_stats: workspace must be a contiguous CUDA tensor")
    rc = load().svi_col_stats(_ptr(x, torch.float32, "x"), _rowmajor(x, "x"), T, C, _ptr(mean, torch.float32, "mean"),
                              _ptr(var, torch.float32, "var"), _vp(workspace.data_ptr()),
                              workspace.numel() * workspace.element_size(), _stream())
    _check(rc, "svi_col_stats")


def col_norm_act(x, mean, var, eps, gamma, beta, act, out):
    """out bf16 [T, C] = act((x - mean) * rsqrt(var + eps) * gamma + beta), per column (row-strided views allowed)."""
    T, C = x.shape
    if tuple(out.shape) != (T, C):
        raise RuntimeError("svi_b200.col_norm_act: out must be [T, C]")
    rc = load().svi_col_norm_act(_ptr(x, torch.float32, "x"), _rowmajor(x, "x"), T, C, _ptr(mean, torch.float32, "mean"),
                                 _ptr(var, torch.float32, "var"), float(eps), _ptr(gamma, torch.float32, "gamma"),
                                 _ptr(beta, torch.float32, "beta"), int(act), _ptr(out, torch.bfloat16, "out"),
                                 _rowmajor(out, "out"), _stream())
    _check(rc, "svi_col_norm_act")
    return out


def conv1d_gather(src, out, kernel, stride, pad_left=0, pad_right=0, col0=0, C=None, split=False):
    """im2col of a channels-last Conv1d: out bf16 [T_out, >= Kpad (2 Kpad with split)] (tap, channel) columns of the
    column window [col0, col0 + C) of src f32 / bf16 [T_in, ld]; T_out = out.shape[0], Kpad = out.shape[1] (/ 2 with split)."""
    T_in, width = src.shape
    C = width - col0 if C is None else C
    if src.dtype not in (torch.float32, torch.bfloat16) or src.stride(1) != 1 or col0 + C > width:
        raise RuntimeError("svi_b200.conv1d_gather: src must be f32 or bf16 with unit inner stride and col0 + C <= width")
    kpad = out.shape[1] // (2 if split else 1)
    rc = load().svi_conv1d_gather(_ptr(src, name="src"), int(src.dtype == torch.float32), src.stride(0), T_in, int(col0), int(C),
                                  int(kernel), int(stride), int(pad_left), int(pad_right), out.shape[0], int(bool(split)),
                                  _ptr(out, torch.bfloat16, "out"), _rowmajor(out, "out"), kpad, _stream())
    _check(rc, "svi_conv1d_gather")
    return out


def interp_layernorm(x, T_out, gamma, beta, eps, out):
    """out bf16 [T_out, C] = LayerNorm(linear_interpolation(x f32 [T_in, C], T_out)) * gamma + beta."""
    T_in, C = x.shape
    if out.shape[0] != T_out or out.shape[1] != C:
        raise RuntimeError("svi_b200.interp_layernorm: out must be [T_out, C]")
    rc = load().svi_interp_layernorm(_ptr(x, torch.float32, "x"), _rowmajor(x, "x"), T_in, C, int(T_out), float(eps),
                                     _ptr(gamma, torch.float32, "gamma"), _ptr(beta, torch.float32, "beta"),
                                     _ptr(out, torch.bfloat16, "out"), _rowmajor(out, "out"), _stream())
    _check(rc, "svi_interp_layernorm")
    return out


# --------------------------------------------------------------------------------------------- RIFE (include/svi_b200_rife.h)
def _contig(t, dtype, name):
    if t is None:
        return None
    if not t.is_contiguous():
        raise RuntimeError(f"svi_b200: {name} must be contiguous")
    return _ptr(t, dtype, name)


def _frames_view(t, name, C):
    """(pointer, stride between frames) of an f32 / uint8 [n, H, W, C] view whose frames are each contiguous."""
    n, H, W, c = t.shape
    if c != C or t.stride()[1:] != (W * C, C, 1):
        raise RuntimeError(f"svi_b200: {name} must be [n, H, W, {C}] with contiguous frames, got {tuple(t.shape)} / {t.stride()}")
    return t.stride(0)


def rife_stage_frames(rgb, out):
    """out f32 [n, H, W, 4] = B, G, R, 0 of uint8 rgb [n, H, W, 3] / 255 (svi_rife_stage_frames)."""
    if rgb.dtype != torch.uint8 or rgb.shape[-1] != 3 or out.shape[-1] != 4 or rgb.numel() // 3 != out.numel() // 4:
        raise RuntimeError("svi_b200.rife_stage_frames: rgb must be uint8 [..., 3] and out f32 [..., 4] of as many pixels")
    _check(load().svi_rife_stage_frames(_contig(rgb, torch.uint8, "rgb"), rgb.numel() // 3, _contig(out, torch.float32, "out"),
                                        _stream()), "svi_rife_stage_frames")
    return out


def rife_block_input(img0, img1, state, h, w, src_scale, flow_mul, out):
    """out bf16 [2 pairs, h/2, w/2, 48]: both directions' space-to-depth block input (svi_rife_block_input_launch).
    img0 / img1 f32 [pairs, H, W, 4] views sharing one frame stride; state f32 [pairs, H, W, 12] or None (first block)."""
    P, H, W, _ = img0.shape
    s0, s1 = _frames_view(img0, "img0", 4), _frames_view(img1, "img1", 4)
    if img1.shape != img0.shape or s0 != s1 or tuple(out.shape) != (2 * P, h // 2, w // 2, 48):
        raise RuntimeError("svi_b200.rife_block_input: img0 / img1 must match and out must be [2 pairs, h/2, w/2, 48]")
    if state is not None and tuple(state.shape) != (P, H, W, 12):
        raise RuntimeError("svi_b200.rife_block_input: state must be [pairs, H, W, 12]")
    d = RifeBlockInput()
    d.img0, d.img1, d.img_stride = _ptr(img0, torch.float32, "img0"), _ptr(img1, torch.float32, "img1"), s0
    d.state = _contig(state, torch.float32, "state")
    d.pairs, d.H, d.W, d.h, d.w = P, H, W, int(h), int(w)
    d.src_scale, d.flow_mul = float(src_scale), float(flow_mul)
    d.out = _contig(out, torch.bfloat16, "out")
    _check(load().svi_rife_block_input_launch(ctypes.byref(d), _stream()), "svi_rife_block_input_launch")
    return out


def rife_conv2d(x, w, kh, kw, pad, C_out, phase_cols, bias, tile_w, prelu=None, residual=None, out=None, out_bf16=None,
                bf_s2d=False):
    """svi_rife_conv2d on x bf16 [N, H, W, C_in] (output grid H x W, stride 1, top / left padding `pad`) with the packed
    weight w bf16 [>= C_out, >= kh kw ceil64(C_in)]: v = x * w + bias -> PReLU (prelu [C_out] or None) -> + residual.
    With C_out = 4 phase_cols the columns are the 2 x 2 sub-pixel phases of a destination grid 2H x 2W.
    out f32 [N, Hd, Wd, out_ld]; out_bf16 bf16 [N, Hd, Wd, bf_ld] or, with bf_s2d, [N, Hd/2, Wd/2, bf_ld] space-to-depth."""
    N, H, W, C_in = x.shape
    d = RifeConvDesc()
    d.x, d.N, d.in_H, d.in_W, d.C_in = _contig(x, torch.bfloat16, "x"), N, H, W, C_in
    d.w_packed, d.w_rows, d.w_ld = _ptr(w, torch.bfloat16, "w"), w.shape[0], _rowmajor(w, "w")
    d.kh, d.kw, d.pad_h, d.pad_w, d.H, d.W = kh, kw, pad, pad, H, W
    d.C_out, d.phase_cols, d.tile_w = C_out, phase_cols, tile_w
    if bias.numel() < C_out or (prelu is not None and prelu.numel() < C_out):
        raise RuntimeError("svi_b200.rife_conv2d: bias and prelu need C_out entries")
    d.bias, d.prelu = _contig(bias, torch.float32, "bias"), _contig(prelu, torch.float32, "prelu")
    lay = out if out is not None else residual
    if residual is not None and out is not None and residual.shape != out.shape:
        raise RuntimeError("svi_b200.rife_conv2d: residual must have the shape of out")
    if lay is not None:
        if lay.dim() != 4 or lay.shape[0] != N:
            raise RuntimeError("svi_b200.rife_conv2d: out / residual must be [N, Hd, Wd, out_ld]")
        d.out_img_stride, d.out_ld = lay[0].numel(), lay.shape[3]
    d.residual, d.out = _contig(residual, torch.float32, "residual"), _contig(out, torch.float32, "out")
    if out_bf16 is not None:
        if out_bf16.dim() != 4 or out_bf16.shape[0] != N:
            raise RuntimeError("svi_b200.rife_conv2d: out_bf16 must be [N, ., ., bf_ld]")
        d.out_bf16, d.bf_img_stride, d.bf_ld = _contig(out_bf16, torch.bfloat16, "out_bf16"), out_bf16[0].numel(), out_bf16.shape[3]
        d.bf_s2d = int(bool(bf_s2d))
    rife_conv2d_desc(d)


def rife_conv2d_desc(desc):
    """Launch svi_rife_conv2d with a filled RifeConvDesc (pointers as ints)."""
    _check(load().svi_rife_conv2d(ctypes.byref(desc), _stream()), "svi_rife_conv2d")


def rife_update_warp(heads, src_scale, flow_mul, img0, img1, state, first, merged=None, clip=False, rgb=None):
    """svi_rife_update_warp: heads f32 [2 pairs, h, w, ld] -> state f32 [pairs, H, W, 12] (updated in place); merged f32
    [pairs, H, W, 4] view (B, G, R blend, sigmoid(mask)) and rgb uint8 [pairs, H, W, 3] view, each optional."""
    P, H, W, _ = img0.shape
    s0, s1 = _frames_view(img0, "img0", 4), _frames_view(img1, "img1", 4)
    if img1.shape != img0.shape or s0 != s1 or heads.shape[0] != 2 * P or tuple(state.shape) != (P, H, W, 12):
        raise RuntimeError("svi_b200.rife_update_warp: img0 / img1 [pairs, H, W, 4], heads [2 pairs, h, w, ld] and state "
                           "[pairs, H, W, 12] required")
    d = RifeUpdate()
    d.heads, d.heads_ld = _contig(heads, torch.float32, "heads"), heads.shape[3]
    d.pairs, d.H, d.W, d.h, d.w = P, H, W, heads.shape[1], heads.shape[2]
    d.src_scale, d.flow_mul = float(src_scale), float(flow_mul)
    d.img0, d.img1, d.img_stride = _ptr(img0, torch.float32, "img0"), _ptr(img1, torch.float32, "img1"), s0
    d.state, d.first = _contig(state, torch.float32, "state"), int(bool(first))
    if merged is not None:
        if merged.shape[0] != P:
            raise RuntimeError("svi_b200.rife_update_warp: merged must have one frame per pair")
        d.merged, d.merged_stride = _ptr(merged, torch.float32, "merged"), _frames_view(merged, "merged", 4)
    d.clip = int(bool(clip))
    if rgb is not None:
        if rgb.shape[0] != P:
            raise RuntimeError("svi_b200.rife_update_warp: rgb must have one frame per pair")
        d.rgb, d.rgb_stride = _ptr(rgb, torch.uint8, "rgb"), _frames_view(rgb, "rgb", 3)
    _check(load().svi_rife_update_warp(ctypes.byref(d), _stream()), "svi_rife_update_warp")


# --------------------------------------------------------------------------------------------- ESRGAN (include/svi_b200_esrgan.h)
def esrgan_stage_frames(rgb, out):
    """out bf16 [n, H, W, 8] = bf16(R, G, B / 255), 0 x 5 of uint8 rgb [n, H, W, 3] (svi_esrgan_stage_frames)."""
    if rgb.dtype != torch.uint8 or rgb.shape[-1] != 3 or out.shape[-1] != 8 or rgb.numel() // 3 != out.numel() // 8:
        raise RuntimeError("svi_b200.esrgan_stage_frames: rgb must be uint8 [..., 3] and out bf16 [..., 8] of as many pixels")
    _check(load().svi_esrgan_stage_frames(_contig(rgb, torch.uint8, "rgb"), rgb.numel() // 3,
                                          _contig(out, torch.bfloat16, "out"), _stream()), "svi_esrgan_stage_frames")
    return out


def _channel_window(t, name):
    """(pointer, pitch) of a bf16 [N, H, W, c] view that is a channel window of a contiguous [N, H, W, pitch] buffer."""
    N, H, W, c = t.shape
    ld = t.stride(2)
    if t.stride(3) != 1 or ld < c or t.stride(1) != W * ld or t.stride(0) != H * W * ld:
        raise RuntimeError(f"svi_b200: {name} must be a channel window of a contiguous [N, H, W, pitch] buffer, got "
                           f"{tuple(t.shape)} / {t.stride()}")
    return _ptr(t, torch.bfloat16, name), ld


def esrgan_conv2d(x, w, C_out, bias, tile_w, slope=0.0, residual=None, res_scale=1.0, residual2=None, res2_scale=1.0,
                  out=None, out_bf16=None, bf_up2=False, out_u8=None):
    """svi_esrgan_conv2d: a 3x3, stride-1, padding-1 convolution of x (bf16 [N, H, W, C_in], a channel window x[..., :C_in]
    of a wider buffer allowed) with the packed weight w bf16 [>= C_out, >= 9 ceil64(C_in)]:
    v = acc + bias -> LeakyReLU(slope) -> v * res_scale + residual -> v * res2_scale + residual2.
    out, residual, residual2 f32 [N, H, W, f_ld] (contiguous); out_bf16 bf16 [N, Hd, Wd, C_out] channel window of a
    contiguous buffer, Hd x Wd = H x W or 2H x 2W with bf_up2; out_u8 uint8 [N, H, W, 3] (channels 0..2)."""
    N, H, W, C_in = x.shape
    d = EsrganConvDesc()
    d.x, d.in_ld = _channel_window(x, "x")
    d.N, d.H, d.W, d.C_in = N, H, W, C_in
    d.w_packed, d.w_rows, d.w_ld = _ptr(w, torch.bfloat16, "w"), w.shape[0], _rowmajor(w, "w")
    d.C_out, d.tile_w = C_out, tile_w
    if bias.numel() < C_out:
        raise RuntimeError("svi_b200.esrgan_conv2d: bias needs C_out entries")
    d.bias, d.slope = _contig(bias, torch.float32, "bias"), float(slope)
    f32 = [t for t in (out, residual, residual2) if t is not None]
    if f32:
        if any(t.shape != f32[0].shape for t in f32) or tuple(f32[0].shape[:3]) != (N, H, W):
            raise RuntimeError("svi_b200.esrgan_conv2d: out, residual and residual2 must be [N, H, W, f_ld] of one shape")
        d.f_ld = f32[0].shape[3]
    d.residual, d.res_scale = _contig(residual, torch.float32, "residual"), float(res_scale)
    d.residual2, d.res2_scale = _contig(residual2, torch.float32, "residual2"), float(res2_scale)
    d.out = _contig(out, torch.float32, "out")
    if out_bf16 is not None:
        up = 2 if bf_up2 else 1
        if tuple(out_bf16.shape) != (N, up * H, up * W, C_out):
            raise RuntimeError(f"svi_b200.esrgan_conv2d: out_bf16 must be [N, {up}H, {up}W, C_out], got {tuple(out_bf16.shape)}")
        d.out_bf16, d.bf_ld = _channel_window(out_bf16, "out_bf16")
        d.bf_up2 = int(bool(bf_up2))
    if out_u8 is not None:
        if tuple(out_u8.shape) != (N, H, W, 3):
            raise RuntimeError("svi_b200.esrgan_conv2d: out_u8 must be [N, H, W, 3]")
        d.out_u8 = _contig(out_u8, torch.uint8, "out_u8")
    esrgan_conv2d_desc(d)


def esrgan_conv2d_desc(desc):
    """Launch svi_esrgan_conv2d with a filled EsrganConvDesc (pointers as ints)."""
    _check(load().svi_esrgan_conv2d(ctypes.byref(desc), _stream()), "svi_esrgan_conv2d")


# --------------------------------------------------------------------------------------------- FastBlend (include/svi_b200_fastblend.h)
def _fb_frames(t, name, dtype=torch.float32, C=4):
    if t.dim() != 4 or t.shape[-1] != C or not t.is_contiguous():
        raise RuntimeError(f"svi_b200: {name} must be contiguous [B, H, W, {C}], got {tuple(t.shape)} / {t.stride()}")
    return _ptr(t, dtype, name)


def fastblend_stage_frames(rgb, out):
    """out f32 [..., 4] = R, G, B, 0 of uint8 rgb [..., 3] (svi_fastblend_stage_frames)."""
    if rgb.dtype != torch.uint8 or rgb.shape[-1] != 3 or out.shape[-1] != 4 or rgb.numel() // 3 != out.numel() // 4:
        raise RuntimeError("svi_b200.fastblend_stage_frames: rgb must be uint8 [..., 3] and out f32 [..., 4] of as many pixels")
    _check(load().svi_fastblend_stage_frames(_contig(rgb, torch.uint8, "rgb"), rgb.numel() // 3,
                                             _contig(out, torch.float32, "out"), _stream()), "svi_fastblend_stage_frames")
    return out


def fastblend_downsample(src, k, out):
    """out f32 [n, H/k, W/k, 4]: the integer-ratio INTER_AREA pyramid level of src f32 [n, H, W, 4]."""
    n, H, W, _ = src.shape
    if tuple(out.shape) != (n, H // k, W // k, 4):
        raise RuntimeError("svi_b200.fastblend_downsample: out must be [n, H/k, W/k, 4]")
    _check(load().svi_fastblend_downsample(_fb_frames(src, "src"), n, H, W, int(k), _fb_frames(out, "out"), _stream()),
           "svi_fastblend_downsample")
    return out


def fastblend_nnf_identity(nnf):
    """nnf int32 [B, H, W, 2] = (y, x)."""
    B, H, W, _ = nnf.shape
    _check(load().svi_fastblend_nnf_identity(_fb_frames(nnf, "nnf", torch.int32, 2), B, H, W, _stream()),
           "svi_fastblend_nnf_identity")
    return nnf


def fastblend_nnf_upscale(src, out):
    """out int32 [B, 2h, 2w, 2]: the field of an exactly doubled level from src int32 [B, h, w, 2]."""
    B, h, w, _ = src.shape
    if tuple(out.shape) != (B, 2 * h, 2 * w, 2):
        raise RuntimeError("svi_b200.fastblend_nnf_upscale: out must be [B, 2h, 2w, 2]")
    _check(load().svi_fastblend_nnf_upscale(_fb_frames(src, "src", torch.int32, 2), B, h, w,
                                            _fb_frames(out, "out", torch.int32, 2), _stream()), "svi_fastblend_nnf_upscale")
    return out


def fastblend_remap(style, nnf, patch_size, out):
    """out f32 [B, H, W, 4]: style f32 [B, H, W, 4] remapped through nnf int32 [B, H, W, 2] (svi_fastblend_remap)."""
    B, H, W, _ = style.shape
    if tuple(nnf.shape) != (B, H, W, 2) or out.shape != style.shape:
        raise RuntimeError("svi_b200.fastblend_remap: style, nnf and out must describe the same [B, H, W] pixels")
    _check(load().svi_fastblend_remap(_fb_frames(style, "style"), _fb_frames(nnf, "nnf", torch.int32, 2), B, H, W,
                                      int(patch_size), _fb_frames(out, "out"), _stream()), "svi_fastblend_remap")
    return out


def fastblend_step(src_guide, src_style, tgt_guide, tgt_style, nnf_in, err_in, nnf_out, err_out, patch_size, mode,
                   guide_weight, dir=0, draw=0, radius=0):
    """One PatchMatch step (svi_fastblend_step): frames f32 [B, H, W, 4], fields int32 [B, H, W, 2], errors f32 [B, H, W]."""
    B, H, W, _ = src_guide.shape
    if any(t.shape != src_guide.shape for t in (src_style, tgt_guide, tgt_style)) or tuple(nnf_in.shape) != (B, H, W, 2) \
            or nnf_out.shape != nnf_in.shape or tuple(err_out.shape) != (B, H, W) or (err_in is not None and err_in.shape != err_out.shape):
        raise RuntimeError("svi_b200.fastblend_step: frames, fields and errors must describe the same [B, H, W] pixels")
    d = FastblendStepDesc()
    d.src_guide, d.src_style = _fb_frames(src_guide, "src_guide"), _fb_frames(src_style, "src_style")
    d.tgt_guide, d.tgt_style = _fb_frames(tgt_guide, "tgt_guide"), _fb_frames(tgt_style, "tgt_style")
    d.nnf_in, d.nnf_out = _fb_frames(nnf_in, "nnf_in", torch.int32, 2), _fb_frames(nnf_out, "nnf_out", torch.int32, 2)
    d.err_in, d.err_out = _contig(err_in, torch.float32, "err_in"), _contig(err_out, torch.float32, "err_out")
    d.B, d.H, d.W, d.patch_size, d.mode, d.dir = B, H, W, int(patch_size), int(mode), int(dir)
    d.draw, d.radius, d.guide_weight = int(draw) & 0xFFFFFFFF, int(radius), float(guide_weight)
    _check(load().svi_fastblend_step(ctypes.byref(d), _stream()), "svi_fastblend_step")


_FB_TYPES = {torch.float32: FB_F32, torch.float64: FB_F64}


def fastblend_table(op, out, a, sa=0.0, b=None, sb=0.0, c=None, sc=0.0, a_u8=False, b_u8=False, c_u8=False):
    """svi_fastblend_table on [..., 4] frames of one pixel count.  An operand flagged `_u8` is a uint8 frame held as its f32
    values; out is f32 / f64 [..., 4], or uint8 [..., 3] for the WSUM's clipped, truncated bytes."""
    d = FastblendTableDesc()
    n = a.numel() // 4
    d.op, d.n_pix = int(op), n

    def operand(t, u8, name):
        if t.shape[-1] != 4 or t.numel() // 4 != n:
            raise RuntimeError(f"svi_b200.fastblend_table: {name} must be [..., 4] of {n} pixels")
        if t.dtype not in _FB_TYPES or (u8 and t.dtype != torch.float32):
            raise RuntimeError(f"svi_b200.fastblend_table: {name} must be f32 or f64 (a uint8 frame is held as f32)")
        return _contig(t, t.dtype, name), FB_U8 if u8 else _FB_TYPES[t.dtype]

    d.a, d.a_type = operand(a, a_u8, "a")
    d.b, d.b_type = operand(b, b_u8, "b")
    d.sa, d.sb, d.sc = float(sa), float(sb), float(sc)
    if c is not None:
        d.c, d.c_type = operand(c, c_u8, "c")
    if out.dtype == torch.uint8:
        if out.shape[-1] != 3 or out.numel() // 3 != n:
            raise RuntimeError("svi_b200.fastblend_table: a uint8 out must be [..., 3] of as many pixels")
        d.out, d.out_type = _contig(out, torch.uint8, "out"), FB_U8
    else:
        d.out, d.out_type = operand(out, False, "out")
    _check(load().svi_fastblend_table(ctypes.byref(d), _stream()), "svi_fastblend_table")
    return out


# --------------------------------------------------------------------------------------------- FastBlend modes (include/svi_b200_fastblend_modes.h)
def fastblend_candidate(nnf_in, nnf_out, mode, dir=0, draw=0, radius=0, shift=0, pairwise=False):
    """nnf_out int32 [B, H, W, 2] = the candidate field of nnf_in (svi_fastblend_candidate): a neighbour, random or
    tracking step."""
    B, H, W, _ = nnf_in.shape
    if nnf_out.shape != nnf_in.shape:
        raise RuntimeError("svi_b200.fastblend_candidate: nnf_in and nnf_out must be [B, H, W, 2] of one shape")
    d = FastblendCandidateDesc()
    d.nnf_in, d.nnf_out = _fb_frames(nnf_in, "nnf_in", torch.int32, 2), _fb_frames(nnf_out, "nnf_out", torch.int32, 2)
    d.B, d.H, d.W, d.mode, d.dir = B, H, W, int(mode), int(dir)
    d.draw, d.radius, d.shift, d.pairwise = int(draw) & 0xFFFFFFFF, int(radius), int(shift), int(bool(pairwise))
    _check(load().svi_fastblend_candidate(ctypes.byref(d), _stream()), "svi_fastblend_candidate")
    return nnf_out


def fastblend_select(src_guide, src_style, tgt_guide, tgt_style, cand, nnf_in, err_in, nnf_out, err_out, patch_size,
                     guide_weight, pairwise=False):
    """The error of the candidate field `cand` and the select (svi_fastblend_select).  frames f32 [B, H, W, 4]; tgt_style
    is [B, H, W, 4], one [H, W, 4] frame shared by every entry, or None with the pairwise error; nnf_in / err_in None
    write the candidate and its error unconditionally."""
    B, H, W, _ = src_guide.shape
    if any(t.shape != src_guide.shape for t in (src_style, tgt_guide)) or tuple(cand.shape) != (B, H, W, 2) \
            or nnf_out.shape != cand.shape or tuple(err_out.shape) != (B, H, W) \
            or (nnf_in is not None and nnf_in.shape != cand.shape) or (err_in is not None and err_in.shape != err_out.shape) \
            or (nnf_in is None) != (err_in is None):
        raise RuntimeError("svi_b200.fastblend_select: frames, fields and errors must describe the same [B, H, W] pixels")
    d = FastblendSelectDesc()
    d.src_guide, d.src_style = _fb_frames(src_guide, "src_guide"), _fb_frames(src_style, "src_style")
    d.tgt_guide = _fb_frames(tgt_guide, "tgt_guide")
    if tgt_style is not None:
        shared = tgt_style.dim() == 3
        if tuple(tgt_style.shape) != ((H, W, 4) if shared else (B, H, W, 4)) or not tgt_style.is_contiguous():
            raise RuntimeError("svi_b200.fastblend_select: tgt_style must be contiguous [B, H, W, 4] or [H, W, 4]")
        d.tgt_style, d.style_shared = _ptr(tgt_style, torch.float32, "tgt_style"), int(shared)
    d.cand = _fb_frames(cand, "cand", torch.int32, 2)
    d.nnf_in = None if nnf_in is None else _fb_frames(nnf_in, "nnf_in", torch.int32, 2)
    d.err_in, d.err_out = _contig(err_in, torch.float32, "err_in"), _contig(err_out, torch.float32, "err_out")
    d.nnf_out = _fb_frames(nnf_out, "nnf_out", torch.int32, 2)
    d.B, d.H, d.W, d.patch_size = B, H, W, int(patch_size)
    d.select, d.pairwise, d.guide_weight = int(nnf_in is not None), int(bool(pairwise)), float(guide_weight)
    _check(load().svi_fastblend_select(ctypes.byref(d), _stream()), "svi_fastblend_select")


def fastblend_batch_mean(src, out):
    """out f32 [H, W, 4] = the f32 mean over B of src f32 [B, H, W, 4], summed in b order (svi_fastblend_batch_mean)."""
    B = src.shape[0]
    if tuple(out.shape) != tuple(src.shape[1:]) or src.shape[-1] != 4:
        raise RuntimeError("svi_b200.fastblend_batch_mean: src must be [B, ..., 4] and out one entry of it")
    _check(load().svi_fastblend_batch_mean(_contig(src, torch.float32, "src"), B, out.numel() // 4,
                                           _contig(out, torch.float32, "out"), _stream()), "svi_fastblend_batch_mean")
    return out


def fastblend_running_mean(frame, s, result, divisor, out, frame_u8=False):
    """out f64 [..., 4] = f64(frame) * s + f64(result / f32(divisor)) (svi_fastblend_running_mean); frame is f64, or with
    frame_u8 a uint8 frame held as its f32 values; result f32."""
    n = out.numel() // 4
    if out.dtype != torch.float64 or out.shape[-1] != 4 or frame.numel() != out.numel() or result.numel() != out.numel():
        raise RuntimeError("svi_b200.fastblend_running_mean: frame, result and out must be [..., 4] of one pixel count")
    ftype = FB_U8 if frame_u8 else FB_F64
    _check(load().svi_fastblend_running_mean(_contig(frame, torch.float32 if frame_u8 else torch.float64, "frame"), ftype,
                                             float(s), _contig(result, torch.float32, "result"), float(divisor), n,
                                             _contig(out, torch.float64, "out"), _stream()), "svi_fastblend_running_mean")
    return out


def fastblend_to_u8(a, out, a_u8=False):
    """out uint8 [..., 3] = a f32 / f64 [..., 4] clipped to [0, 255] and truncated (svi_fastblend_to_u8)."""
    n = a.numel() // 4
    if a.shape[-1] != 4 or out.shape[-1] != 3 or out.numel() // 3 != n or a.dtype not in _FB_TYPES:
        raise RuntimeError("svi_b200.fastblend_to_u8: a must be f32 / f64 [..., 4] and out uint8 [..., 3] of as many pixels")
    atype = FB_U8 if a_u8 else _FB_TYPES[a.dtype]
    _check(load().svi_fastblend_to_u8(_contig(a, a.dtype, "a"), atype, n, _contig(out, torch.uint8, "out"), _stream()),
           "svi_fastblend_to_u8")
    return out


# --------------------------------------------------------------------------------------------- UniAnimate (include/svi_b200_unianimate.h)
def _latents_view(t, name):
    """(C, frames, h*w) of a contiguous f32 [1, C, frames, h, w] tensor."""
    if t.dim() != 5 or t.shape[0] != 1 or not t.is_contiguous():
        raise RuntimeError(f"svi_b200: {name} must be a contiguous [1, C, f, h, w] tensor, got {tuple(t.shape)}")
    return t.shape[1], t.shape[2], t.shape[3] * t.shape[4]


def window_accumulate(win, skip, sum_, start):
    """sum_[:, :, start + skip:start + cs] += win[:, :, skip:] (svi_window_accumulate); f32 [1, C, cs | F, h, w]."""
    C, cs, hw = _latents_view(win, "win")
    C2, F, hw2 = _latents_view(sum_, "sum")
    if (C2, hw2) != (C, hw):
        raise RuntimeError("svi_b200.window_accumulate: win and sum must have the same channels and frame size")
    _check(load().svi_window_accumulate(_ptr(win, torch.float32, "win"), C, cs, hw, int(skip),
                                        _ptr(sum_, torch.float32, "sum"), F, int(start), _stream()), "svi_window_accumulate")
    return sum_


def window_normalize(sum_, count, out):
    """out = sum_ / count[frame] (svi_window_normalize); sum_ and out f32 [1, C, F, h, w], count int32 [F]."""
    C, F, hw = _latents_view(sum_, "sum")
    if _latents_view(out, "out") != (C, F, hw) or tuple(count.shape) != (F,) or not count.is_contiguous():
        raise RuntimeError("svi_b200.window_normalize: out must match sum and count must be [F]")
    _check(load().svi_window_normalize(_ptr(sum_, torch.float32, "sum"), _ptr(count, torch.int32, "count"), C, F, hw,
                                       _ptr(out, torch.float32, "out"), _stream()), "svi_window_normalize")
    return out


# --------------------------------------------------------------------------------------------- Replace-Anyone (include/svi_b200_replace.h)
def replace_mask_stage(video, seg, masked, ring):
    """video f32 [3, T, H, W], seg uint8 or f32 [T, H, W] (contiguous) -> masked f32 [3, T, H, W] (or None) =
    video * keep, and ring bf16 [T, H, W, ldr] channels 0..3 = (masked, keep), keep = !(seg / 255 > 0)
    (svi_replace_mask_stage)."""
    if video.dim() != 4 or video.shape[0] != 3 or not video.is_contiguous():
        raise RuntimeError(f"svi_b200.replace_mask_stage: video must be a contiguous [3, T, H, W] tensor, got {tuple(video.shape)}")
    _, T, H, W = video.shape
    if tuple(seg.shape) != (T, H, W) or not seg.is_contiguous():
        raise RuntimeError(f"svi_b200.replace_mask_stage: seg must be a contiguous [T, H, W] = {(T, H, W)} tensor, "
                           f"got {tuple(seg.shape)}")
    seg_type = {torch.uint8: SEG_U8, torch.float32: SEG_F32}.get(seg.dtype)
    if seg_type is None:
        raise RuntimeError(f"svi_b200.replace_mask_stage: seg must be uint8 or float32, got {seg.dtype}")
    if masked is not None and (masked.shape != video.shape or not masked.is_contiguous()):
        raise RuntimeError("svi_b200.replace_mask_stage: masked must be contiguous and shaped like video")
    if ring.dim() != 4 or tuple(ring.shape[:3]) != (T, H, W) or not ring.is_contiguous():
        raise RuntimeError(f"svi_b200.replace_mask_stage: ring must be a contiguous [T, H, W, ldr] = {(T, H, W)} + (ldr,) "
                           f"tensor, got {tuple(ring.shape)}")
    _check(load().svi_replace_mask_stage(_ptr(video, torch.float32, "video"), _ptr(seg, name="seg"), seg_type, T, H * W,
                                         _ptr(masked, torch.float32, "masked"), _ptr(ring, torch.bfloat16, "ring"),
                                         ring.shape[3], _stream()), "svi_replace_mask_stage")
    return masked, ring


# --------------------------------------------------------------------------------------------- quality scoring (include/svi_b200_quality.h)
def quality_attn(q, k, v, out, batch, num_heads, head_dim, scale, causal=False):
    """softmax(q k^T * scale [+ causal mask]) v for `batch` sequences of L = rows / batch tokens (svi_quality_attn); q, k,
    v, out bf16 [batch * L, >= num_heads * head_dim] row-major views (column slices of the fused qkv output)."""
    ldq, ldk, ldv, ldo = (_rowmajor(t, n) for t, n in ((q, "q"), (k, "k"), (v, "v"), (out, "out")))
    rows = q.shape[0]
    if batch < 1 or rows % batch or any(t.shape[0] != rows for t in (k, v, out)):
        raise RuntimeError(f"svi_b200.quality_attn: q, k, v, out must have the same rows, a multiple of batch = {batch}")
    _check(load().svi_quality_attn(_ptr(q, torch.bfloat16, "q"), ldq, _ptr(k, torch.bfloat16, "k"), ldk,
                                   _ptr(v, torch.bfloat16, "v"), ldv, _ptr(out, torch.bfloat16, "out"), ldo, int(batch),
                                   rows // batch, int(num_heads), int(head_dim), float(scale), int(bool(causal)), _stream()),
           "svi_quality_attn")
    return out


def quality_stage_pixels(px, mean_std, out, patch):
    """px f32 [B, 3, S, S] -> out bf16 [B * (S/patch)^2, kpad] = (px - mean) / std in patch rows (svi_quality_stage_pixels);
    mean_std f32 [6] on the device."""
    if px.dim() != 4 or px.shape[1] != 3 or px.shape[2] != px.shape[3] or not px.is_contiguous():
        raise RuntimeError(f"svi_b200.quality_stage_pixels: px must be a contiguous [B, 3, S, S] tensor, got {tuple(px.shape)}")
    B, _, S, _ = px.shape
    if not out.is_contiguous() or out.dim() != 2 or out.shape[0] != B * (S // patch) ** 2:
        raise RuntimeError("svi_b200.quality_stage_pixels: out must be a contiguous [B * (S/patch)^2, kpad] tensor")
    if mean_std.numel() != 6 or not mean_std.is_contiguous():
        raise RuntimeError("svi_b200.quality_stage_pixels: mean_std must hold 6 floats")
    _check(load().svi_quality_stage_pixels(_ptr(px, torch.float32, "px"), B, S, int(patch),
                                           _ptr(mean_std, torch.float32, "mean_std"), _ptr(out, torch.bfloat16, "out"),
                                           out.shape[1], _stream()), "svi_quality_stage_pixels")
    return out


def quality_embed_ln(patch, cls, pos, gamma, beta, eps, out):
    """out f32 [B*(1+np), D] = LayerNorm([cls; patch rows of image b] + pos) per image (svi_quality_embed_ln)."""
    np_, D = pos.shape[0] - 1, pos.shape[1]
    if patch.dim() != 2 or patch.shape[1] != D or patch.shape[0] % np_ or not patch.is_contiguous():
        raise RuntimeError("svi_b200.quality_embed_ln: patch must be a contiguous [B * np, D] tensor")
    B = patch.shape[0] // np_
    if tuple(out.shape) != (B * (np_ + 1), D) or not out.is_contiguous() or not pos.is_contiguous():
        raise RuntimeError("svi_b200.quality_embed_ln: out must be a contiguous [B * (np + 1), D] tensor")
    if cls.numel() != D or gamma.numel() != D or beta.numel() != D:
        raise RuntimeError("svi_b200.quality_embed_ln: cls, gamma and beta must hold D floats")
    _check(load().svi_quality_embed_ln(_ptr(patch, torch.float32, "patch"), _ptr(cls, torch.float32, "cls"),
                                       _ptr(pos, torch.float32, "pos"), B, np_, D, float(eps),
                                       _ptr(gamma, torch.float32, "gamma"), _ptr(beta, torch.float32, "beta"),
                                       _ptr(out, torch.float32, "out"), _stream()), "svi_quality_embed_ln")
    return out


def quality_quick_gelu(x, out):
    """out bf16 = x * sigmoid(1.702 x) of x f32 (svi_quality_quick_gelu); both [M, N] row-major views."""
    ldx, ldy = _rowmajor(x, "x"), _rowmajor(out, "out")
    if x.shape != out.shape:
        raise RuntimeError("svi_b200.quality_quick_gelu: x and out must have the same shape")
    _check(load().svi_quality_quick_gelu(_ptr(x, torch.float32, "x"), ldx, x.shape[0], x.shape[1],
                                         _ptr(out, torch.bfloat16, "out"), ldy, _stream()), "svi_quality_quick_gelu")
    return out


def quality_pool(x, n_seq, out, mode=POOL_FIRST, ids=None, eos_id=0):
    """out f32 [n_seq, D] = one row per sequence of x f32 [n_seq * L, D] (svi_quality_pool): row 0, the argmax of ids
    (int64 [n_seq, L]) or the first row whose id is eos_id."""
    ldx = _rowmajor(x, "x")
    if n_seq < 1 or x.shape[0] % n_seq or tuple(out.shape) != (n_seq, x.shape[1]) or not out.is_contiguous():
        raise RuntimeError("svi_b200.quality_pool: x must hold n_seq sequences and out be a contiguous [n_seq, D] tensor")
    L = x.shape[0] // n_seq
    if ids is not None and (ids.dtype != torch.int64 or tuple(ids.shape) != (n_seq, L) or not ids.is_contiguous()):
        raise RuntimeError(f"svi_b200.quality_pool: ids must be contiguous int64 [{n_seq}, {L}]")
    _check(load().svi_quality_pool(_ptr(x, torch.float32, "x"), ldx, n_seq, L, x.shape[1], _ptr(ids, name="ids"), int(mode),
                                   int(eos_id), _ptr(out, torch.float32, "out"), _stream()), "svi_quality_pool")
    return out


def quality_score(img, txt=None, cos=None, w=None, bias=0.0, aes=None):
    """cos f32 [B, T] = normalised img [B, E] . normalised txt [T, E]; aes f32 [B] = w . normalised img + bias
    (svi_quality_score)."""
    B, E = img.shape
    T = 0 if txt is None else txt.shape[0]
    for t, n, shape in ((img, "img", (B, E)), (txt, "txt", (T, E)), (cos, "cos", (B, T)), (w, "w", (E,)), (aes, "aes", (B,))):
        if t is not None and (tuple(t.shape) != shape or not t.is_contiguous()):
            raise RuntimeError(f"svi_b200.quality_score: {n} must be a contiguous {shape} tensor, got {tuple(t.shape)}")
    _check(load().svi_quality_score(_ptr(img, torch.float32, "img"), B, _ptr(txt, torch.float32, "txt"), T, E,
                                    _ptr(w, torch.float32, "w"), float(bias), _ptr(cos, torch.float32, "cos"),
                                    _ptr(aes, torch.float32, "aes"), _stream()), "svi_quality_score")
    return cos, aes


# --------------------------------------------------------------------------------------------- cross-attention scorers (include/svi_b200_reward.h)
def reward_attn(q, k, v, out, batch, num_heads, scale, kv_heads=None, kv_shared=False, key_mask=None):
    """softmax(q k^T * scale, masked keys excluded) v, head width 64 (svi_reward_attn).  q, out bf16 [batch * Lq, >= 64 H]
    and k, v bf16 [batch * Lk (or Lk when kv_shared), >= 64 kv_heads] row-major views; kv_heads is num_heads (default) or
    1.  key_mask uint8 [batch, Lk], or [1, Lk] / [Lk] shared by every sequence."""
    ldq, ldk, ldv, ldo = (_rowmajor(t, n) for t, n in ((q, "q"), (k, "k"), (v, "v"), (out, "out")))
    kv_heads = num_heads if kv_heads is None else kv_heads
    rows = q.shape[0]
    if batch < 1 or rows % batch or out.shape[0] != rows or k.shape[0] != v.shape[0] or (not kv_shared and k.shape[0] % batch):
        raise RuntimeError(f"svi_b200.reward_attn: q / out rows must be a multiple of batch = {batch} and k, v agree")
    Lq = rows // batch
    Lk = k.shape[0] if kv_shared else k.shape[0] // batch
    mstride = 0
    if key_mask is not None:
        if key_mask.dtype != torch.uint8 or not key_mask.is_contiguous() or key_mask.shape[-1] != Lk or \
                key_mask.numel() not in (Lk, batch * Lk):
            raise RuntimeError(f"svi_b200.reward_attn: key_mask must be contiguous uint8 [{batch}, {Lk}] or [{Lk}]")
        mstride = Lk if key_mask.numel() == batch * Lk and batch > 1 else 0
    _check(load().svi_reward_attn(_ptr(q, torch.bfloat16, "q"), ldq, _ptr(k, torch.bfloat16, "k"), ldk,
                                  _ptr(v, torch.bfloat16, "v"), ldv, _ptr(out, torch.bfloat16, "out"), ldo, int(batch), Lq, Lk,
                                  int(num_heads), int(kv_heads), 0 if kv_shared else Lk, _ptr(key_mask, torch.uint8, "key_mask"),
                                  mstride, float(scale), _stream()), "svi_reward_attn")
    return out


def reward_layernorm(x, gamma, beta, eps, y, yb):
    """y f32 = LN(x) * gamma + beta (y may be x) and yb bf16 = the same values rounded (svi_reward_layernorm)."""
    M, D = x.shape
    if not (x.is_contiguous() and y.is_contiguous() and yb.is_contiguous()) or y.shape != x.shape or yb.shape != x.shape:
        raise RuntimeError("svi_b200.reward_layernorm: x, y, yb must be contiguous and of one shape")
    _check(load().svi_reward_layernorm(_ptr(x, torch.float32, "x"), M, D, float(eps), _ptr(gamma, torch.float32, "gamma"),
                                       _ptr(beta, torch.float32, "beta"), _ptr(y, torch.float32, "y"),
                                       _ptr(yb, torch.bfloat16, "yb"), _stream()), "svi_reward_layernorm")
    return y, yb


def reward_embed(patch, cls, pos, out):
    """out f32 [B*(1+np), D] = [cls; patch rows of image b] + pos per image (svi_reward_embed)."""
    np_, D = pos.shape[0] - 1, pos.shape[1]
    if patch.dim() != 2 or patch.shape[1] != D or patch.shape[0] % np_ or not patch.is_contiguous() or not pos.is_contiguous():
        raise RuntimeError("svi_b200.reward_embed: patch must be a contiguous [B * np, D] tensor")
    B = patch.shape[0] // np_
    if tuple(out.shape) != (B * (np_ + 1), D) or not out.is_contiguous() or cls.numel() != D:
        raise RuntimeError("svi_b200.reward_embed: out must be a contiguous [B * (np + 1), D] tensor and cls hold D floats")
    _check(load().svi_reward_embed(_ptr(patch, torch.float32, "patch"), _ptr(cls, torch.float32, "cls"),
                                   _ptr(pos, torch.float32, "pos"), B, np_, D, _ptr(out, torch.float32, "out"), _stream()),
           "svi_reward_embed")
    return out


def reward_swiglu(x, out):
    """out bf16 [M, F] = silu(g) * a of x f32 [M, 2F] = [a | g] (svi_reward_swiglu); row-major views."""
    ldx, ldy = _rowmajor(x, "x"), _rowmajor(out, "out")
    M, F2 = x.shape
    if F2 % 2 or tuple(out.shape) != (M, F2 // 2):
        raise RuntimeError("svi_b200.reward_swiglu: x must be [M, 2F] and out [M, F]")
    _check(load().svi_reward_swiglu(_ptr(x, torch.float32, "x"), ldx, M, F2 // 2, _ptr(out, torch.bfloat16, "out"), ldy,
                                    _stream()), "svi_reward_swiglu")
    return out


def reward_rope(x, L, cos, sin):
    """rotate-half RoPE in place on the 64-wide heads of x bf16 [M, 64 heads] (row-major view), position = row % L;
    cos, sin f32 [L, 32] (svi_reward_rope)."""
    ldx = _rowmajor(x, "x")
    M, W = x.shape
    if W % 64 or tuple(cos.shape) != (L, 32) or tuple(sin.shape) != (L, 32) or not (cos.is_contiguous() and sin.is_contiguous()):
        raise RuntimeError("svi_b200.reward_rope: x must be [M, 64 * heads] and cos, sin contiguous [L, 32]")
    _check(load().svi_reward_rope(_ptr(x, torch.bfloat16, "x"), ldx, M, int(L), W // 64, _ptr(cos, torch.float32, "cos"),
                                  _ptr(sin, torch.float32, "sin"), _stream()), "svi_reward_rope")
    return x


def reward_cond_mask(text, cond, threshold, ratio, keep):
    """ratio f32 [Lt] = max_j text[i] . cond[j] over its maximum, keep uint8 [Lt] = ratio > threshold
    (svi_reward_cond_mask); text f32 [Lt, E], cond f32 [Lc, E]."""
    (Lt, E), Lc = text.shape, cond.shape[0]
    if not (text.is_contiguous() and cond.is_contiguous() and ratio.is_contiguous() and keep.is_contiguous()) or \
            cond.shape[1] != E or ratio.numel() != Lt or keep.numel() != Lt:
        raise RuntimeError("svi_b200.reward_cond_mask: contiguous text [Lt, E], cond [Lc, E], ratio and keep [Lt] required")
    _check(load().svi_reward_cond_mask(_ptr(text, torch.float32, "text"), Lt, _ptr(cond, torch.float32, "cond"), Lc, E,
                                       float(threshold), _ptr(ratio, torch.float32, "ratio"), _ptr(keep, torch.uint8, "keep"),
                                       _stream()), "svi_reward_cond_mask")
    return ratio, keep


def reward_head(x, n_seq, w, bias, out):
    """out f32 [n_seq] = w . (row 0 of each sequence of x f32 [n_seq * L, E]) + bias (svi_reward_head)."""
    ldx = _rowmajor(x, "x")
    if n_seq < 1 or x.shape[0] % n_seq or w.numel() != x.shape[1] or out.numel() != n_seq or not out.is_contiguous():
        raise RuntimeError("svi_b200.reward_head: x must hold n_seq sequences, w E floats and out n_seq floats")
    _check(load().svi_reward_head(_ptr(x, torch.float32, "x"), ldx, n_seq, x.shape[0] // n_seq, x.shape[1],
                                  _ptr(w, torch.float32, "w"), float(bias), _ptr(out, torch.float32, "out"), _stream()),
           "svi_reward_head")
    return out


# --------------------------------------------------------------------------------------------- processors (include/svi_b200_processors.h)
def _u8_frames(t, name):
    """(F, H, W) of a contiguous uint8 [F, H, W, 3] CUDA tensor"""
    if t.dtype != torch.uint8 or t.dim() != 4 or t.shape[3] != 3 or not t.is_contiguous():
        raise RuntimeError(f"svi_b200: {name} must be contiguous uint8 [F, H, W, 3], got {t.dtype} {tuple(t.shape)}")
    _ptr(t, torch.uint8, name)
    return t.shape[:3]


def luma_sum_u8(rgb, sums):
    """sums int64 [F] = per frame, the integer sum of Pillow's L of uint8 rgb [F, H, W, 3] (svi_luma_sum_u8)."""
    F, H, W = _u8_frames(rgb, "rgb")
    if sums.dtype != torch.int64 or tuple(sums.shape) != (F,):
        raise RuntimeError("svi_b200.luma_sum_u8: sums must be int64 [F]")
    _check(load().svi_luma_sum_u8(_ptr(rgb), F, H * W, _contig(sums, torch.int64, "sums"), _stream()), "svi_luma_sum_u8")
    return sums


def enhance_blend_u8(rgb, degenerate, rate, out):
    """out uint8 [F, H, W, 3] = Image.blend(degenerate[f], rgb[f], rate) per frame; degenerate f32 [F] (svi_enhance_blend_u8)."""
    F, H, W = _u8_frames(rgb, "rgb")
    if out.shape != rgb.shape or tuple(degenerate.shape) != (F,):
        raise RuntimeError("svi_b200.enhance_blend_u8: out must have rgb's shape and degenerate one value per frame")
    _u8_frames(out, "out")
    _check(load().svi_enhance_blend_u8(_ptr(rgb), F, H * W, _contig(degenerate, torch.float32, "degenerate"), float(rate),
                                       _ptr(out), _stream()), "svi_enhance_blend_u8")
    return out


def sharpen_u8(rgb, rate, out):
    """out uint8 [F, H, W, 3] = Image.blend(rgb.filter(SMOOTH), rgb, rate) per frame (svi_sharpen_u8)."""
    F, H, W = _u8_frames(rgb, "rgb")
    if out.shape != rgb.shape:
        raise RuntimeError("svi_b200.sharpen_u8: out must have rgb's shape")
    _u8_frames(out, "out")
    _check(load().svi_sharpen_u8(_ptr(rgb), F, H, W, float(rate), _ptr(out), _stream()), "svi_sharpen_u8")
    return out


def rife_average_u8(frames, merged, out):
    """out[1:-1] uint8 RGB = ((frames[1:-1] + merged) / 2 * 255).clip(0, 255) truncated, from f32 BGR frames
    [F, H, W, 4] and merged [F - 2, H, W, 4]; out [F, H, W, 3] keeps its first and last frames (svi_rife_average_u8)."""
    F, H, W = _u8_frames(out, "out")
    if tuple(frames.shape) != (F, H, W, 4) or tuple(merged.shape) != (F - 2, H, W, 4):
        raise RuntimeError("svi_b200.rife_average_u8: frames must be [F, H, W, 4] and merged [F - 2, H, W, 4] for out "
                           "[F, H, W, 3]")
    _check(load().svi_rife_average_u8(_contig(frames, torch.float32, "frames"), _contig(merged, torch.float32, "merged"),
                                      F, H * W, _ptr(out), _stream()), "svi_rife_average_u8")
    return out
