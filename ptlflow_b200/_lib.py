"""ctypes binding of libptlflow_b200.so (the C ABI declared in include/ptlflow_b200.h).

The library is the product: if it is missing this module raises -- there is no CPU or
PyTorch fallback for the hot path.  Build it with ``python -m ptlflow_b200.csrc.build``
(or ``__graft_entry__.build()``); the .so is kept in-tree under ptlflow_b200/lib/.
"""
from __future__ import annotations

import ctypes as C
import threading
import os
from typing import Optional

import torch

_PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_PKG, "lib", "libptlflow_b200.so")

PFB_MAX_LEVELS = 8
PFB_MAX_SRC = 4

F32, F16, BF16 = 0, 1, 2
_DTYPES = {torch.float32: F32, torch.float16: F16, torch.bfloat16: BF16}

EPI_LINEAR, EPI_RELU, EPI_GRU_ZR, EPI_GRU_Q, EPI_FLOW, EPI_RELU_APPEND_FLOW, EPI_AXPY, EPI_LINEAR_F32 = range(8)
EPI_GELU, EPI_RESIDUAL_GELU, EPI_LINEAR_APPEND_FLOW = range(8, 11)
# pfb_enc_conv_epilogue
ENC_CONV_LINEAR, ENC_CONV_BIAS_RELU, ENC_CONV_BIAS_RELU_RESIDUAL = range(3)

(L_CONVC1, L_CONVC2, L_CONVF1, L_CONVF2, L_CONV, L_GRU_ZR1, L_GRU_Q1, L_GRU_ZR2, L_GRU_Q2,
 L_FLOW1, L_FLOW2, L_MASK1, L_MASK2, L_AGG_V, L_FLOW2T,
 L_CTX_ZR1, L_CTX_Q1, L_CTX_ZR2, L_CTX_Q2, L_GRUX_ZR1, L_GRUX_Q1, L_GRUX_ZR2, L_GRUX_Q2, L_CONVC2F2, L_AGG_PROJ, L_COUNT) = range(26)
# pfb_variant: the refinement loop a RaftCfg describes
(VARIANT_RAFT, VARIANT_RAFT_SMALL, VARIANT_GMA, VARIANT_SKFLOW, VARIANT_SEA_RAFT, VARIANT_MS_RAFT_P, VARIANT_CCMR, VARIANT_FLOW1D,
 VARIANT_CSFLOW, VARIANT_SCV8, VARIANT_SCV4, VARIANT_COUNT) = range(12)


class ConvSrc(C.Structure):
    _fields_ = [("ptr", C.c_void_p), ("channels", C.c_int), ("stride", C.c_int), ("offset", C.c_int), ("is_f32", C.c_int)]


class ConvParams(C.Structure):
    _fields_ = [
        ("src", ConvSrc * PFB_MAX_SRC), ("nsrc", C.c_int),
        ("B", C.c_int), ("H", C.c_int), ("W", C.c_int), ("KH", C.c_int), ("KW", C.c_int),
        ("Cout", C.c_int), ("Cout_pad", C.c_int),
        ("weight", C.c_void_p), ("bias", C.c_void_p),
        ("epilogue", C.c_int), ("scale", C.c_float),
        ("out", C.c_void_p), ("out_stride", C.c_int), ("out_offset", C.c_int),
        ("aux_h", C.c_void_p), ("aux_z", C.c_void_p), ("hidden", C.c_int),
        ("coords", C.c_void_p), ("flow", C.c_void_p),
        ("dtype", C.c_int), ("impl", C.c_int),
        ("weight_k", C.c_void_p), ("Cin_pad", C.c_int), ("Cout_pad_k", C.c_int),
        ("addend", C.c_void_p), ("addend_stride", C.c_int), ("w_rows_per_sample", C.c_int),
        ("residual", C.c_void_p), ("residual_stride", C.c_int), ("residual_offset", C.c_int),
        ("post_w", C.c_void_p), ("post_b", C.c_void_p),
    ]


class Layer(C.Structure):
    _fields_ = [("weight", C.c_void_p), ("bias", C.c_void_p), ("Cout", C.c_int), ("Cout_pad", C.c_int),
                ("Cin", C.c_int), ("KH", C.c_int), ("KW", C.c_int),
                ("weight_k", C.c_void_p), ("Cin_pad", C.c_int), ("Cout_pad_k", C.c_int)]


class RaftCfg(C.Structure):
    _fields_ = [
        ("variant", C.c_int), ("dtype", C.c_int), ("B", C.c_int), ("H", C.c_int), ("W", C.c_int),
        ("feat_dim", C.c_int), ("corr_levels", C.c_int), ("corr_radius", C.c_int),
        ("hidden_dim", C.c_int), ("context_dim", C.c_int), ("iters", C.c_int), ("alternate_corr", C.c_int),
        ("out_h", C.c_int), ("out_w", C.c_int), ("pad_top", C.c_int), ("pad_left", C.c_int), ("impl", C.c_int),
        ("volume_layout", C.c_int), ("fork_flow", C.c_int), ("num_heads", C.c_int),
    ]


class RaftWeights(C.Structure):
    _fields_ = [("layers", Layer * L_COUNT)]


class RaftBuffers(C.Structure):
    _fields_ = [
        ("pyramid", C.POINTER(C.c_void_p)), ("fmap1", C.c_void_p), ("net", C.c_void_p), ("inp", C.c_void_p),
        ("coords", C.c_void_p), ("flow_up", C.c_void_p), ("flow_small", C.c_void_p),
        ("workspace", C.c_void_p), ("workspace_bytes", C.c_size_t),
        ("attention", C.c_void_p), ("agg_gamma", C.c_float), ("agg_score", C.c_void_p), ("pool_min_side", C.c_int),
    ]


# SKFlow (include/ptlflow_b200.h, a15)
PFB_SK_MAX_DW = 8
SK_CONVC1, SK_CONVC2, SK_CONVF2, SK_CONV, SK_GRU, SK_FLOW_HEAD, SK_BLOCKS = range(7)
KERNEL_CLASSES = 15  # PFB_KERNEL_CLASSES (12 = depthwise convolution, 13 = depthwise convolution + LayerNorm, 14 = 1D attention)
# pfb_profile_collect's classes by index, in the header's order
KERNEL_CLASS_NAMES = ("volume", "pool", "lookup", "onthefly", "conv", "upsample", "misc", "enc_affine", "enc_stats", "enc_conv1",
                      "flowconv", "gather", "depthwise", "dw_layernorm", "attn1d")
ATTN1D_CORR, ATTN1D_ATTN = 1, 2  # pfb_attn1d modes
ATTN1D_MAX_L = 1024  # PFB_ATTN1D_MAX_L


class PcBlock(C.Structure):
    _fields_ = [("ffn1a", Layer), ("ffn1b", Layer), ("pw", Layer), ("ffn2a", Layer), ("ffn2b", Layer),
                ("C", C.c_int), ("hid", C.c_int), ("n_dw", C.c_int), ("dw_k", C.c_int * PFB_SK_MAX_DW),
                ("dw_weight", C.c_void_p * PFB_SK_MAX_DW), ("dw_bias", C.c_void_p * PFB_SK_MAX_DW)]


class SkflowWeights(C.Structure):
    _fields_ = [("blocks", PcBlock * SK_BLOCKS), ("convf1", Layer), ("mask1", Layer), ("mask2", Layer),
                ("agg_v", Layer), ("agg_proj", Layer)]


# SEA-RAFT (include/ptlflow_b200.h, a16)
PFB_SR_MAX_BLOCKS = 8


class ConvNextBlock(C.Structure):
    _fields_ = [("dw_k", C.c_int), ("dw_weight", C.c_void_p), ("dw_bias", C.c_void_p), ("pw1", Layer), ("out", Layer)]


class SearaftWeights(C.Structure):
    _fields_ = [("init_conv", Layer), ("convc1", Layer), ("convc2", Layer), ("convf1", Layer), ("convf2", Layer), ("conv", Layer),
                ("num_blocks", C.c_int), ("blocks", ConvNextBlock * PFB_SR_MAX_BLOCKS), ("ln_eps", C.c_float),
                ("flow1", Layer), ("flow2", Layer), ("flow2t", Layer), ("mask1", Layer), ("mask2", Layer)]


# CCMR (include/ptlflow_b200.h, a18)
class XcitBlock(C.Structure):
    _fields_ = [("pos_proj", Layer), ("qk", Layer), ("v_weight", C.c_void_p), ("v_bias", C.c_void_p), ("proj_weight", C.c_void_p),
                ("proj_bias", C.c_void_p), ("temperature", C.c_void_p), ("ln3_weight", C.c_void_p), ("ln3_bias", C.c_void_p),
                ("dw1_weight", C.c_void_p), ("dw1_bias", C.c_void_p), ("gn_weight", C.c_void_p), ("gn_bias", C.c_void_p),
                ("dw2_weight", C.c_void_p), ("dw2_bias", C.c_void_p), ("fc1", Layer), ("fc2", Layer), ("ln_eps", C.c_float),
                ("gn_eps", C.c_float)]


class CcmrWeights(C.Structure):
    _fields_ = [("raft", RaftWeights), ("context", XcitBlock), ("aggregator", XcitBlock)]


_lib: Optional[C.CDLL] = None

# name -> (restype, argtypes); every symbol include/ptlflow_b200.h declares
_I, _P, _S = C.c_int, C.c_void_p, C.c_void_p
_PP = C.POINTER(C.c_void_p)
SIGNATURES = {
    "pfb_version": (_I, []),
    "pfb_last_error": (C.c_char_p, []),
    "pfb_device_arch": (_I, []),
    "pfb_stream_create": (_I, [_PP]),
    "pfb_stream_destroy": (_I, [_S]),
    "pfb_corr_volume_build": (_I, [_P, _P, _PP, _I, _I, _I, _I, _I, _I, _I, _S]),
    "pfb_corr_volume_build_ex": (_I, [_P, _P, _PP, _I, _I, _I, _I, _I, _I, _I, C.c_float, _I, _I, _S]),
    "pfb_corr_level_bytes": (C.c_size_t, [_I, _I, _I, _I, _I]),
    "pfb_corr_lookup": (_I, [_PP, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _S]),
    "pfb_corr_lookup_ex": (_I, [_PP, C.POINTER(C.c_int), C.POINTER(C.c_int), _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _S]),
    "pfb_corr_level_bytes_tiled": (C.c_size_t, [_I, _I, _I, _I, _I, _I]),
    "pfb_corr_volume_build_tiled": (_I, [_P, _P, _PP, _I, _I, _I, _I, _I, _I, _I, C.c_float, _I, _S]),
    "pfb_corr_lookup_tiled": (_I, [_PP, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _S]),
    "pfb_corr_lookup_tiled_ex": (_I, [_PP, C.POINTER(C.c_int), C.POINTER(C.c_int), _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _S]),
    "pfb_corr_level_sizes": (_I, [_I, _I, _I, _I, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "pfb_corr_lookup_onthefly": (_I, [_P, _PP, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _S]),
    "pfb_corr_lookup_onthefly_tc_workspace_bytes": (C.c_size_t, [_I, _I, _I]),
    "pfb_corr_lookup_onthefly_tc": (_I, [_P, _PP, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _S]),
    "pfb_alt_corr_forward": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _S]),
    "pfb_avg_pool2x2_nhwc": (_I, [_P, _P, _I, _I, _I, _I, _I, _S]),
    "pfb_conv2d": (_I, [C.POINTER(ConvParams), _S]),
    "pfb_conv2d_umma_plan": (_I, [C.POINTER(ConvParams), C.POINTER(_I), C.POINTER(_I), C.POINTER(C.c_size_t)]),
    "pfb_pack_conv_weight": (_I, [_P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _S]),
    "pfb_pack_bias": (_I, [_P, _P, _I, _I, _I, _S]),
    "pfb_pack_conv_weight_kmajor": (_I, [_P, _P, _I, _I, _I, _I, _I, _I, C.POINTER(C.c_int), _I, _I, _I, _I, _S]),
    "pfb_convex_upsample": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _S]),
    "pfb_upflow8": (_I, [_P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _S]),
    "pfb_softmax_rows": (_I, [_P, C.c_size_t, _I, _I, _S]),
    "pfb_attention_softmax_relpos": (_I, [_P, _P, _P, C.c_size_t, _P, C.c_size_t, _I, _I, _I, _I, _S]),
    "pfb_transpose_pm": (_I, [_P, _P, _I, _I, _I, _I, _I, _S]),
    "pfb_flow_tap_gather": (_I, [_P, _I, _P, _P, _P, _I, _I, _I, _S]),
    "pfb_context_split": (_I, [_P, _P, _P, _I, _I, _I, _I, _I, _I, _S]),
    "pfb_init_coords": (_I, [_P, _P, _I, _I, _I, _S]),
    "pfb_forward_interpolate": (_I, [_P, _P, _I, _I, _I, _S]),
    "pfb_raft_workspace_bytes": (C.c_size_t, [C.POINTER(RaftCfg)]),
    "pfb_raft_workspace_bytes_ex": (C.c_size_t, [C.POINTER(RaftCfg), C.c_int]),
    "pfb_raft_refine": (_I, [C.POINTER(RaftCfg), C.POINTER(RaftWeights), C.POINTER(RaftBuffers), _S]),
    "pfb_preprocess_frames": (_I, [_P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _S]),
    "pfb_preprocess_frames_ex": (_I, [_P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _S]),
    "pfb_instance_norm_workspace_bytes": (C.c_size_t, [_I, _I]),
    "pfb_instance_norm_act": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, C.c_float, _I, _I, _S]),
    "pfb_instance_norm_apply": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, C.c_float, _I, _I, _S]),
    "pfb_flow_conv7x7": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _S]),
    "pfb_first_conv7x7s2": (_I, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _S]),
    "pfb_bias_act": (_I, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _S]),
    "pfb_enc_conv3x3_supported": (_I, [_I, _I, _I]),
    "pfb_enc_conv3x3": (_I, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _S]),
    "pfb_launch_count": (C.c_ulonglong, [_I]),
    "pfb_profile_enable": (_I, [_I]),
    "pfb_profile_collect": (_I, [C.POINTER(C.c_double), C.POINTER(C.c_ulonglong), _I]),
    "pfb_raft_update_iter": (_I, [C.POINTER(RaftCfg), C.POINTER(RaftWeights), C.POINTER(RaftBuffers), _P, _P, _S]),
    "pfb_depthwise_conv_gelu": (_I, [_P, _I, _I, _P, _I, _I, _P, _P, _I, _I, _I, _I, _I, _I, _S]),
    "pfb_skflow_workspace_bytes": (C.c_size_t, [C.POINTER(RaftCfg)]),
    "pfb_skflow_refine": (_I, [C.POINTER(RaftCfg), C.POINTER(SkflowWeights), C.POINTER(RaftBuffers), _S]),
    "pfb_skflow_update_iter": (_I, [C.POINTER(RaftCfg), C.POINTER(SkflowWeights), C.POINTER(RaftBuffers), _P, _P, _S]),
    "pfb_depthwise_conv_layernorm": (_I, [_P, _I, _I, _P, _I, _I, _P, _P, _I, _I, _I, _I, _I, C.c_float, _I, _S]),
    "pfb_searaft_workspace_bytes": (C.c_size_t, [C.POINTER(RaftCfg)]),
    "pfb_searaft_refine": (_I, [C.POINTER(RaftCfg), C.POINTER(SearaftWeights), C.POINTER(RaftBuffers), _S]),
    "pfb_searaft_update_iter": (_I, [C.POINTER(RaftCfg), C.POINTER(SearaftWeights), C.POINTER(RaftBuffers), _P, _P, _S]),
    # MS-RAFT+ (a17)
    "pfb_corr_lookup_onthefly_ex": (_I, [_P, _PP, _P, _P, _I, _I, _I, _I, _I, _I, C.c_float, _I, _I, _I, _I, _S]),
    "pfb_corr_lookup_onthefly_tc_ex": (_I, [_P, _PP, _P, _P, _P, _I, _I, _I, _I, _I, _I, C.c_float, _I, _I, _S]),
    "pfb_group_norm_act": (_I, [_P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, C.c_float, _I, _I, _S]),
    "pfb_group_norm_apply": (_I, [_P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, C.c_float, _I, _I, _S]),
    "pfb_upsample2x_concat": (_I, [_P, _I, _P, _I, _P, _I, _I, _I, _I, _S]),
    "pfb_convex_upsample2x": (_I, [_P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _S]),
    "pfb_downflow": (_I, [_P, _P, _I, _I, _I, _I, _I, _S]),
    "pfb_msraft_workspace_bytes": (C.c_size_t, [C.POINTER(RaftCfg)]),
    "pfb_msraft_refine": (_I, [C.POINTER(RaftCfg), C.POINTER(RaftWeights), C.POINTER(RaftBuffers), C.c_float, _P, _S]),
    "pfb_msraft_update_iter": (_I, [C.POINTER(RaftCfg), C.POINTER(RaftWeights), C.POINTER(RaftBuffers), _P, _P, C.c_float, _S]),
    # CCMR (a18)
    "pfb_layernorm": (_I, [_P, _I, _I, _P, _I, _I, _P, _P, C.c_size_t, _I, C.c_float, _I, _S]),
    "pfb_depthwise_conv3x3_ex": (_I, [_P, _I, _I, _P, _I, _I, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _S]),
    "pfb_fourier_features": (_I, [_P, _I, _I, _I, _S]),
    "pfb_xca_stats_workspace_bytes": (C.c_size_t, [_I, _I]),
    "pfb_xca_stats": (_I, [_P, _I, _I, _I, _I, _I, _P, _P, _I, _S]),
    "pfb_xca_fold": (_I, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _S]),
    "pfb_convex_handover2x": (_I, [_P, _P, _P, _I, _I, _I, _I, _S]),
    "pfb_upflow2": (_I, [_P, _P, _I, _I, _I, _I, _I, _I, _I, _S]),
    "pfb_xcit_context": (_I, [C.POINTER(RaftCfg), C.POINTER(CcmrWeights), _P, _P, _P, C.c_size_t, _S]),
    "pfb_ccmr_workspace_bytes": (C.c_size_t, [C.POINTER(RaftCfg)]),
    "pfb_ccmr_refine": (_I, [C.POINTER(RaftCfg), C.POINTER(CcmrWeights), C.POINTER(RaftBuffers), C.c_float, _I, _P, _S]),
    "pfb_ccmr_update_iter": (_I, [C.POINTER(RaftCfg), C.POINTER(CcmrWeights), C.POINTER(RaftBuffers), _P, _P, C.c_float, _S]),
    # Flow1D (a19)
    "pfb_attn1d": (_I, [_P, _I, _P, _I, _P, _I, _P, _I, _I, _I, _I, _I, _I, _I, C.c_float, _I, _I, _S]),
    "pfb_corr1d_lookup": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _S]),
    # CSFlow (a20)
    "pfb_strip_table_width": (_I, [_I, _I]),
    "pfb_strip_means": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _S]),
    "pfb_strip_prepare": (_I, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _S]),
    "pfb_strip_lookup": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _S]),
    # SCV (a21)
    "pfb_knn_topk_workspace_bytes": (C.c_size_t, [_P, _P, _I, _I, _I, _I, _I, _I]),
    "pfb_knn_topk": (_I, [_P, _P, _P, _P, _P, C.c_size_t, _I, _I, _I, _I, C.c_float, _I, _I, _S]),
    "pfb_sparse_prepare": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _S]),
    "pfb_sparse_lookup": (_I, [_P, _P, _P, _I, _I, _I, _I, _I, _I, _S]),
    "pfb_convex_upsample4x": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _S]),
    # LLA-Flow (a22)
    "pfb_local_similar": (_I, [_P, _P, _P, _I, _I, _I, _I, _S]),
    "pfb_local_aggregate": (_I, [_P, _P, _P, C.c_float, _P, _I, _I, _I, _I, _S]),
    "pfb_shift_pack": (_I, [_P, _P, _P, _P, _P, C.c_float, _P, _P, _P, _I, _I, _I, _I, _S]),
    "pfb_shift_volume_tiled": (_I, [_P, _P, _PP, _I, _I, _I, _I, _I, _S]),
    # CRAFT (a23)
    "pfb_craft_clamp_flag": (_I, [_P, C.c_size_t, C.c_float, _P, _I, _S]),
    "pfb_craft_window_softmax": (_I, [_P, C.c_size_t, _I, _I, _P, _I, _I, _P, C.c_float, _I, _S]),
    "pfb_craft_mode_aggregate": (_I, [_P, _I, _I, _I, _P, C.c_float, _P, _I, _I, _P, _I, _I, _I, _I, _S]),
    "pfb_craft_volume_workspace_bytes": (C.c_size_t, [_I, _I, _I]),
    "pfb_craft_volume_norm": (_I, [_P, _I, C.c_float, _P, _I, _P, C.c_float, _P, _P, C.c_size_t, _I, _I, _I, _I, _S]),
    "pfb_craft_volume_tiled_workspace_bytes": (C.c_size_t, [_I, _I, _I]),
    "pfb_craft_volume_tiled": (_I, [_P, _P, _I, C.c_float, _P, _I, _P, C.c_float, _PP, _P, C.c_size_t, _I, _I, _I, _I, _I, _S]),
    "pfb_raft_workspace_motion": (_I, [C.POINTER(RaftCfg), C.POINTER(C.c_size_t), C.POINTER(C.c_int)]),
    "pfb_softsplat_workspace_bytes": (C.c_size_t, [_I, _I, _I, _I]),
    "pfb_softsplat_average": (_I, [_P, _I, _I, _P, _P, _I, _I, _P, C.c_size_t, _I, _I, _I, _I, _I, _S]),
}


class LibraryMissing(RuntimeError):
    pass


def load() -> C.CDLL:
    """Load (once) and type the shared library.  Raises LibraryMissing if it was never built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise LibraryMissing(
            f"{LIB_PATH} not found: the ptlflow_b200 hot path is hand-written CUDA and has no fallback. "
            "Build it with `python -m ptlflow_b200.csrc.build` (needs nvcc, no GPU required to compile)."
        )
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError here == header/library mismatch
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc: int, what: str = "") -> None:
    """Translate a negative pfb_status into RuntimeError (the reference plugin raises RuntimeError
    through TORCH_CHECK, ptlflow/utils/external/alt_cuda_corr/correlation.cpp:19-21)."""
    if rc != 0:
        msg = load().pfb_last_error().decode(errors="replace")
        raise RuntimeError(f"ptlflow_b200 {what} failed (status {rc}): {msg}")


def dtype_code(dt: torch.dtype) -> int:
    try:
        return _DTYPES[dt]
    except KeyError:
        raise RuntimeError(f"ptlflow_b200: unsupported dtype {dt}; use float32, float16 or bfloat16") from None


def stream_ptr(device=None) -> int:
    return torch.cuda.current_stream(device).cuda_stream


_private_streams: dict = {}
_private_lock = threading.Lock()
_private_tls = threading.local()


def _new_private_stream(idx: int) -> "torch.cuda.Stream":
    raw = C.c_void_p()
    with torch.cuda.device(idx):
        check(load().pfb_stream_create(C.byref(raw)), "stream_create")
    return torch.cuda.ExternalStream(raw.value, device=torch.device("cuda", idx))


def _device_index(device) -> int:
    dev = torch.device(device)
    return dev.index if dev.index is not None else torch.cuda.current_device()


def private_stream(device) -> "torch.cuda.Stream":
    """One stream per device that no other code can be handed: ``torch.cuda.Stream()`` draws from a pool of 32 and two
    callers can hold the same underlying stream (a pipeline slot launching eagerly on the stream another thread is capturing
    puts its kernels into that capture and fails its own allocations).  CUDA-graph captures run here, one at a time."""
    idx = _device_index(device)
    with _private_lock:
        st = _private_streams.get(idx)
        if st is None:
            st = _private_streams[idx] = _new_private_stream(idx)
        return st


def thread_stream(device, tag: str = "aux") -> "torch.cuda.Stream":
    """A private stream of THIS host thread (and device): the second lane of a forward's fork / join sections (the two
    encoders side by side).  Forwards of different host threads run concurrently, so each brings its own."""
    idx = _device_index(device)
    streams = getattr(_private_tls, "streams", None)
    if streams is None:
        streams = _private_tls.streams = {}
    st = streams.get((idx, tag))
    if st is None:
        st = streams[(idx, tag)] = _new_private_stream(idx)
    return st


def require_cuda(t: torch.Tensor, name: str) -> None:
    """Mirror of CHECK_INPUT (correlation.cpp:19-21): CUDA + contiguous, else RuntimeError."""
    if not t.is_cuda:
        raise RuntimeError(f"{name} must be a CUDA tensor")
    if not t.is_contiguous():
        raise RuntimeError(f"{name} must be contiguous")


def ptr_array(tensors) -> "C.Array":
    arr = (C.c_void_p * len(tensors))()
    for i, t in enumerate(tensors):
        arr[i] = t.data_ptr()
    return arr
