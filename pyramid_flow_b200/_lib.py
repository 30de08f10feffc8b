"""ctypes binding of libpf_b200.so (the C-ABI declared in include/pf_b200.h).

PyTorch is used only for device memory and streams: every call passes raw `data_ptr()`s and the current CUDA stream.
There is no fallback: if the library is missing or the device is not sm_90, calls raise RuntimeError.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

_HERE = Path(__file__).resolve().parent
LIB_PATH = _HERE / "lib" / "libpf_b200.so"

# every symbol include/pf_b200.h declares (tests check the .so exports exactly these)
SYMBOLS = [
    "pf_last_error", "pf_version", "pf_device_check", "pf_warmup", "pf_set_option", "pf_get_option", "pf_launch_count",
    "pf_gemm_bf16", "pf_gemm_fp8", "pf_ln_modulate_fp8", "pf_quantize_rows_fp8",
    "pf_attn_build_schedule", "pf_attn_build_pair_schedule", "pf_attn_build_pair_masks", "pf_attn_build_group_schedule",
    "pf_attn_build_group_masks", "pf_attn_fwd_masked", "pf_attn_build_kv_schedule", "pf_attn_bwd_masked",
    "pf_attn_stage_pack", "pf_attn_stage_pack_bwd",
    "pf_attn_varlen_pack", "pf_attn_varlen_pack_bwd", "pf_attn_varlen_unpack", "pf_attn_varlen_unpack_bwd",
    "pf_ln_modulate", "pf_small_linear", "pf_timestep_embedding",
    "pf_patchify", "pf_unpatchify", "pf_cfg_euler_step", "pf_stage_hop",
    "pf_causal_conv3d", "pf_groupnorm_stats", "pf_groupnorm_apply", "pf_softmax_rows", "pf_pack_latent", "pf_blend_tiles",
    "pf_ctx_create", "pf_ctx_destroy", "pf_ctx_record_begin", "pf_ctx_record_end", "pf_ctx_replay", "pf_dit_step_flux",
    "pf_dit_step_mmdit", "pf_vae_decode_chunk",
    "pf_peer_alloc", "pf_peer_free", "pf_peer_export", "pf_peer_open", "pf_peer_close", "pf_peer_barrier", "pf_peer_bcast",
    "pf_attn_fwd_text", "pf_rms_norm_rows", "pf_embed_tokens",
    "pf_conv3d_pack", "pf_conv3d_wgrad_workspace", "pf_conv3d_wgrad",
    "pf_groupnorm_train_workspace", "pf_groupnorm_train_fwd", "pf_groupnorm_train_bwd",
    "pf_maxpool2x2", "pf_maxpool2x2_bwd", "pf_lpips_head_fwd", "pf_lpips_tap_bwd", "pf_lpips_dropout_mask",
]

PF_OPT_GEMM_STAGED_RESID, PF_OPT_GEMM_WAVE_TILING, PF_OPT_ATTN_PAIR_KERNEL, PF_OPT_ATTN_TILE_PHASE, PF_OPT_ATTN_TRIPLE_KERNEL = range(5)
PF_EPI_STORE_BF16, PF_EPI_GELU_BF16, PF_EPI_STORE_F32, PF_EPI_GATE_RESID, PF_EPI_QKV_ROPE, PF_EPI_QKV_GELU = range(6)
PF_EPI_GEGLU_BF16, PF_EPI_QUICK_GELU_BF16, PF_EPI_GELU_ERF_BF16 = range(6, 9)


class GemmDesc(C.Structure):
    _fields_ = [
        ("a", C.c_void_p), ("lda", C.c_int64),
        ("batches", C.c_int32), ("rows_per_batch", C.c_int32), ("row_begin", C.c_int32), ("row_count", C.c_int32),
        ("w", C.c_void_p), ("n", C.c_int32), ("k", C.c_int32),
        ("bias", C.c_void_p), ("epilogue", C.c_int32),
        ("out", C.c_void_p), ("ldo", C.c_int64),
        ("out_batch_rows", C.c_int32), ("out_row_begin", C.c_int32), ("out_col_begin", C.c_int32),
        ("gate", C.c_void_p), ("gate_batch_stride", C.c_int64),
        ("q_out", C.c_void_p), ("k_out", C.c_void_p), ("v_out", C.c_void_p),
        ("rope", C.c_void_p), ("q_norm_w", C.c_void_p), ("k_norm_w", C.c_void_p),
        ("norm_eps", C.c_float),
        ("heads", C.c_int32), ("head_dim", C.c_int32), ("seq_len", C.c_int32),
        ("n_split", C.c_int32), ("kernel_variant", C.c_int32),
        ("peer_qkv", C.c_void_p * 8),
        ("peer_count", C.c_int32), ("peer_heads", C.c_int32), ("peer_seq", C.c_int32), ("peer_row0", C.c_int32),
    ]


class AttnDesc(C.Structure):
    _fields_ = [
        ("q", C.c_void_p), ("k", C.c_void_p), ("v", C.c_void_p), ("out", C.c_void_p), ("ldo", C.c_int64),
        ("batch", C.c_int32), ("heads", C.c_int32), ("seq", C.c_int32), ("head_dim", C.c_int32),
        ("scale", C.c_float),
        ("seg", C.c_void_p), ("time", C.c_void_p), ("tile_sched", C.c_void_p),
        ("sched_stride", C.c_int32), ("variant", C.c_int32), ("q_row_begin", C.c_int32),
        ("pair_sched", C.c_void_p),
        ("pair_mask_index", C.c_void_p), ("pair_mask_bits", C.c_void_p),
        ("peer_out", C.c_void_p * 8),
        ("peer_count", C.c_int32), ("peer_chunk_rows", C.c_int32), ("peer_col_begin", C.c_int32),
        ("group_sched", C.c_void_p), ("group_mask_index", C.c_void_p), ("group_mask_bits", C.c_void_p),
        ("lse", C.c_void_p),
    ]


class AttnBwdDesc(C.Structure):
    _fields_ = [
        ("q", C.c_void_p), ("k", C.c_void_p), ("v", C.c_void_p),
        ("out", C.c_void_p), ("ldo", C.c_int64), ("out_batch_stride", C.c_int64),
        ("dout", C.c_void_p), ("lddo", C.c_int64), ("dout_batch_stride", C.c_int64), ("lse", C.c_void_p),
        ("batch", C.c_int32), ("heads", C.c_int32), ("seq", C.c_int32), ("head_dim", C.c_int32),
        ("scale", C.c_float),
        ("seg", C.c_void_p), ("time", C.c_void_p), ("tile_sched", C.c_void_p), ("kv_sched", C.c_void_p),
        ("sched_stride", C.c_int32),
        ("delta", C.c_void_p), ("dq", C.c_void_p), ("dk", C.c_void_p), ("dv", C.c_void_p),
    ]


class AttnPackDesc(C.Structure):
    _fields_ = [
        ("batch", C.c_int32), ("heads", C.c_int32), ("head_dim", C.c_int32), ("text_len", C.c_int32),
        ("rows", C.c_int32), ("row0", C.c_int32), ("src_rows", C.c_int32), ("n_stages", C.c_int32), ("stage", C.c_int32),
        ("video", C.c_void_p * 3), ("video_strides", (C.c_int64 * 3) * 3), ("video_f32", C.c_int32 * 3),
        ("text", C.c_void_p * 3), ("text_strides", (C.c_int64 * 3) * 3), ("text_f32", C.c_int32 * 3),
        ("freqs", C.c_void_p), ("freqs_batch_stride", C.c_int64), ("freqs_row_stride", C.c_int64),
        ("packed", C.c_void_p * 3),
    ]


VARLEN_MAX_STAGES = 8       # PF_ATTN_VARLEN_MAX_STAGES


class AttnVarlenLayout(C.Structure):
    _fields_ = [
        ("batch", C.c_int32), ("heads", C.c_int32), ("head_dim", C.c_int32), ("text_len", C.c_int32), ("src_rows", C.c_int32),
        ("n_stages", C.c_int32), ("stage_len", C.c_int32 * VARLEN_MAX_STAGES), ("stage_row0", C.c_int32 * VARLEN_MAX_STAGES),
        ("total", C.c_int32), ("row_map", C.c_void_p), ("pad_map", C.c_void_p),
    ]


class AttnVarlenPackDesc(C.Structure):
    _fields_ = [
        ("layout", AttnVarlenLayout),
        ("video", C.c_void_p * 3), ("video_strides", (C.c_int64 * 3) * 3), ("video_f32", C.c_int32 * 3),
        ("text", C.c_void_p * 3), ("text_strides", (C.c_int64 * 3) * 3), ("text_f32", C.c_int32 * 3),
        ("freqs", C.c_void_p * VARLEN_MAX_STAGES), ("freqs_batch_stride", C.c_int64 * VARLEN_MAX_STAGES),
        ("freqs_row_stride", C.c_int64 * VARLEN_MAX_STAGES),
        ("packed", C.c_void_p * 3),
    ]


class AttnVarlenUnpackDesc(C.Structure):
    _fields_ = [
        ("layout", AttnVarlenLayout),
        ("video", C.c_void_p), ("video_strides", C.c_int64 * 2), ("video_f32", C.c_int32),
        ("text", C.c_void_p), ("text_strides", C.c_int64 * 2), ("text_f32", C.c_int32),
        ("packed", C.c_void_p), ("ld_packed", C.c_int64),
    ]


class AttnTextDesc(C.Structure):
    _fields_ = [
        ("qkv", C.c_void_p), ("ld_qkv", C.c_int64), ("out", C.c_void_p), ("ldo", C.c_int64),
        ("batch", C.c_int32), ("heads", C.c_int32), ("seq", C.c_int32), ("head_dim", C.c_int32),
        ("scale", C.c_float), ("bias", C.c_void_p), ("key_mask", C.c_void_p), ("causal", C.c_int32),
    ]


class PeerGroup(C.Structure):
    _fields_ = [("ptr", C.c_void_p * 8), ("n", C.c_int32), ("my_index", C.c_int32)]


class ConvDesc(C.Structure):
    _fields_ = [
        ("x", C.c_void_p),
        ("b", C.c_int32), ("t", C.c_int32), ("h", C.c_int32), ("w", C.c_int32), ("cin", C.c_int32),
        ("wgt", C.c_void_p), ("bias", C.c_void_p),
        ("cout", C.c_int32), ("kt", C.c_int32), ("kh", C.c_int32), ("kw", C.c_int32),
        ("store_mode", C.c_int32),
        ("out", C.c_void_p), ("out_f32", C.c_int32),
        ("out_t_total", C.c_int32), ("out_t_offset", C.c_int32), ("out_c", C.c_int32),
        ("store_channels", C.c_int32),
        ("residual", C.c_void_p), ("res_t_total", C.c_int32), ("res_t_offset", C.c_int32),
        ("stride_t", C.c_int32), ("stride_h", C.c_int32), ("stride_w", C.c_int32), ("kernel_variant", C.c_int32),
        ("relu", C.c_int32), ("select", C.c_void_p),
    ]


class ConvPackDesc(C.Structure):
    _fields_ = [
        ("src", C.c_void_p), ("src_f32", C.c_int32),
        ("b", C.c_int32), ("c", C.c_int32), ("t", C.c_int32), ("h", C.c_int32), ("w", C.c_int32),
        ("strides", C.c_int64 * 5),
        ("dst", C.c_void_p), ("cpad", C.c_int32), ("t_total", C.c_int32), ("t_offset", C.c_int32),
        ("dil_t", C.c_int32), ("dil_h", C.c_int32), ("dil_w", C.c_int32),
        ("bias_grad", C.c_void_p), ("workspace", C.c_void_p), ("workspace_floats", C.c_int64),
    ]


class ConvWgradDesc(C.Structure):
    _fields_ = [
        ("x", C.c_void_p), ("dy", C.c_void_p), ("dy_t_total", C.c_int32),
        ("b", C.c_int32), ("t", C.c_int32), ("h", C.c_int32), ("w", C.c_int32),
        ("cin", C.c_int32), ("cout", C.c_int32), ("cin_real", C.c_int32), ("cout_real", C.c_int32),
        ("kt", C.c_int32), ("kh", C.c_int32), ("kw", C.c_int32),
        ("stride_t", C.c_int32), ("stride_h", C.c_int32), ("stride_w", C.c_int32),
        ("dw", C.c_void_p), ("workspace", C.c_void_p), ("workspace_floats", C.c_int64),
    ]


class GroupNormTrainDesc(C.Structure):
    _fields_ = [
        ("x", C.c_void_p), ("x_f32", C.c_int32),
        ("b", C.c_int32), ("c", C.c_int32), ("t", C.c_int32), ("h", C.c_int32), ("w", C.c_int32),
        ("x_strides", C.c_int64 * 5),
        ("groups", C.c_int32), ("eps", C.c_float), ("silu", C.c_int32),
        ("gamma", C.c_void_p), ("beta", C.c_void_p), ("stats", C.c_void_p),
        ("y", C.c_void_p), ("y_f32", C.c_int32),
        ("dy", C.c_void_p), ("dy_f32", C.c_int32), ("dy_strides", C.c_int64 * 5),
        ("dx", C.c_void_p), ("dgamma", C.c_void_p), ("dbeta", C.c_void_p),
        ("workspace", C.c_void_p), ("workspace_floats", C.c_int64),
    ]


LPIPS_MAX_TAPS = 5          # PF_LPIPS_MAX_TAPS
LPIPS_HEAD_BLOCKS = 32      # PF_LPIPS_HEAD_BLOCKS


class LpipsHeadDesc(C.Structure):
    _fields_ = [
        ("n", C.c_int32), ("taps", C.c_int32),
        ("f0", C.c_void_p * LPIPS_MAX_TAPS), ("f1", C.c_void_p * LPIPS_MAX_TAPS), ("lin", C.c_void_p * LPIPS_MAX_TAPS),
        ("c", C.c_int32 * LPIPS_MAX_TAPS), ("h", C.c_int32 * LPIPS_MAX_TAPS), ("w", C.c_int32 * LPIPS_MAX_TAPS),
        ("p", C.c_float), ("seed", C.c_void_p), ("val", C.c_void_p),
        ("workspace", C.c_void_p), ("workspace_floats", C.c_int64),
    ]


class LpipsTapBwdDesc(C.Structure):
    _fields_ = [
        ("n", C.c_int32), ("c", C.c_int32), ("h", C.c_int32), ("w", C.c_int32), ("tap", C.c_int32),
        ("f", C.c_void_p), ("f_other", C.c_void_p), ("lin", C.c_void_p),
        ("p", C.c_float), ("seed", C.c_void_p), ("grad", C.c_void_p),
        ("d_next", C.c_void_p), ("dz", C.c_void_p),
    ]


_lib = None
_warm_devices = set()


def load() -> C.CDLL:
    """dlopen the library and declare signatures. Works without a GPU (no CUDA call is made)."""
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.exists():
        raise RuntimeError(
            f"{LIB_PATH} is missing: run `python __graft_entry__.py` (build()) first. "
            "pyramid_flow_b200 has no fallback path.")
    lib = C.CDLL(str(LIB_PATH))
    missing = [s for s in SYMBOLS if not hasattr(lib, s)]
    if missing:
        raise RuntimeError(f"libpf_b200.so does not export: {missing}")
    lib.pf_last_error.restype = C.c_char_p
    lib.pf_launch_count.restype = C.c_int64
    lib.pf_gemm_bf16.argtypes = [C.POINTER(GemmDesc), C.c_void_p]
    lib.pf_gemm_fp8.argtypes = [C.POINTER(GemmDesc), C.c_void_p, C.c_void_p, C.c_void_p]
    lib.pf_ln_modulate_fp8.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                       C.c_int32, C.c_void_p, C.c_void_p, C.c_int64, C.c_float, C.c_void_p]
    lib.pf_quantize_rows_fp8.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int32, C.c_int32,
                                         C.c_int32, C.c_int32, C.c_int32, C.c_void_p]
    lib.pf_attn_fwd_masked.argtypes = [C.POINTER(AttnDesc), C.c_void_p]
    lib.pf_attn_bwd_masked.argtypes = [C.POINTER(AttnBwdDesc), C.c_void_p]
    lib.pf_attn_stage_pack.argtypes = [C.POINTER(AttnPackDesc), C.c_void_p]
    lib.pf_attn_stage_pack_bwd.argtypes = [C.POINTER(AttnPackDesc), C.c_void_p]
    for name in ("pf_attn_varlen_pack", "pf_attn_varlen_pack_bwd"):
        getattr(lib, name).argtypes = [C.POINTER(AttnVarlenPackDesc), C.c_void_p]
    for name in ("pf_attn_varlen_unpack", "pf_attn_varlen_unpack_bwd"):
        getattr(lib, name).argtypes = [C.POINTER(AttnVarlenUnpackDesc), C.c_void_p]
    lib.pf_attn_build_kv_schedule.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]
    lib.pf_attn_build_schedule.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]
    lib.pf_attn_build_pair_schedule.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]
    lib.pf_attn_build_pair_masks.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                             C.c_int64]
    lib.pf_attn_build_pair_masks.restype = C.c_int64
    lib.pf_attn_build_group_schedule.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]
    lib.pf_attn_build_group_masks.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                              C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
    lib.pf_attn_build_group_masks.restype = C.c_int64
    lib.pf_ctx_create.argtypes = [C.POINTER(C.c_void_p)]
    for name in ("pf_ctx_destroy", "pf_ctx_record_end"):
        getattr(lib, name).argtypes = [C.c_void_p]
    for name in ("pf_ctx_record_begin", "pf_ctx_replay", "pf_dit_step_flux", "pf_dit_step_mmdit", "pf_vae_decode_chunk"):
        getattr(lib, name).argtypes = [C.c_void_p, C.c_void_p]
    lib.pf_peer_alloc.argtypes = [C.c_int64, C.POINTER(C.c_void_p)]
    lib.pf_peer_free.argtypes = [C.c_void_p]
    lib.pf_peer_export.argtypes = [C.c_void_p, C.c_void_p]
    lib.pf_peer_open.argtypes = [C.c_void_p, C.POINTER(C.c_void_p)]
    lib.pf_peer_close.argtypes = [C.c_void_p]
    lib.pf_peer_barrier.argtypes = [C.POINTER(PeerGroup), C.c_void_p, C.c_void_p]
    lib.pf_peer_bcast.argtypes = [C.POINTER(PeerGroup), C.c_void_p, C.c_int64, C.c_int64, C.c_void_p]
    lib.pf_ln_modulate.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                   C.c_void_p, C.c_void_p, C.c_int64, C.c_float, C.c_void_p]
    lib.pf_small_linear.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p,
                                    C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]
    lib.pf_timestep_embedding.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p]
    lib.pf_patchify.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                C.c_void_p, C.c_int32, C.c_int32, C.c_void_p]
    lib.pf_unpatchify.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                  C.c_int32, C.c_void_p, C.c_int32, C.c_void_p]
    lib.pf_cfg_euler_step.argtypes = [C.c_void_p, C.c_float, C.c_float, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
    lib.pf_stage_hop.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_float,
                                 C.c_float, C.POINTER(C.c_float), C.c_void_p]
    lib.pf_blend_tiles.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_int64, C.c_int32, C.c_void_p]
    lib.pf_causal_conv3d.argtypes = [C.POINTER(ConvDesc), C.c_void_p]
    lib.pf_conv3d_pack.argtypes = [C.POINTER(ConvPackDesc), C.c_void_p]
    lib.pf_conv3d_wgrad.argtypes = [C.POINTER(ConvWgradDesc), C.c_void_p]
    lib.pf_conv3d_wgrad_workspace.argtypes = [C.POINTER(ConvWgradDesc)]
    lib.pf_conv3d_wgrad_workspace.restype = C.c_int64
    for name in ("pf_groupnorm_train_fwd", "pf_groupnorm_train_bwd"):
        getattr(lib, name).argtypes = [C.POINTER(GroupNormTrainDesc), C.c_void_p]
    lib.pf_groupnorm_train_workspace.argtypes = [C.POINTER(GroupNormTrainDesc)]
    lib.pf_groupnorm_train_workspace.restype = C.c_int64
    lib.pf_lpips_head_fwd.argtypes = [C.POINTER(LpipsHeadDesc), C.c_void_p]
    lib.pf_lpips_tap_bwd.argtypes = [C.POINTER(LpipsTapBwdDesc), C.c_void_p]
    lib.pf_maxpool2x2.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]
    lib.pf_maxpool2x2_bwd.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                      C.c_void_p]
    lib.pf_lpips_dropout_mask.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_float,
                                          C.c_void_p, C.c_void_p]
    lib.pf_groupnorm_stats.argtypes = [C.c_void_p, C.c_int32, C.c_int64, C.c_int32, C.c_int32, C.c_float, C.c_void_p,
                                       C.c_void_p, C.c_int64, C.c_void_p]
    lib.pf_groupnorm_apply.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int64, C.c_int32, C.c_int32,
                                       C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]
    lib.pf_softmax_rows.argtypes = [C.c_void_p, C.c_int64, C.c_int32, C.c_int64, C.c_float, C.c_void_p]
    lib.pf_pack_latent.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                   C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.pf_attn_fwd_text.argtypes = [C.POINTER(AttnTextDesc), C.c_void_p]
    lib.pf_rms_norm_rows.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                     C.c_float, C.c_void_p]
    lib.pf_embed_tokens.argtypes = [C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32,
                                    C.c_void_p, C.c_void_p]
    _lib = lib
    return lib


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        raise RuntimeError(f"libpf_b200 {what} failed ({rc}): {load().pf_last_error().decode()}")


def require_device() -> None:
    """Fail loudly unless the CUDA extension is usable on this machine (no CPU fallback exists)."""
    lib = load()
    check(lib.pf_device_check(), "pf_device_check")
    import torch
    dev = torch.cuda.current_device()
    if dev not in _warm_devices:
        check(lib.pf_warmup(), "pf_warmup")
        _warm_devices.add(dev)


def stream_ptr() -> int:
    import torch
    return torch.cuda.current_stream().cuda_stream


def set_option(key: int, value: int) -> None:
    check(load().pf_set_option(int(key), int(value)), "pf_set_option")


def get_option(key: int) -> int:
    return int(load().pf_get_option(int(key)))


def launch_count() -> int:
    return int(load().pf_launch_count())
