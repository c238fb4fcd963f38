"""ctypes binding of libmas_b200.so (the C-ABI declared in include/mas_b200.h).

The product path has NO fallback: if the shared library is missing or a call fails, a RuntimeError is
raised. Tensors are owned by torch (device memory, streams); only raw pointers, extents and the current
CUDA stream cross the boundary.
"""
from __future__ import annotations

import contextlib
import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(os.path.dirname(_HERE), "lib", "libmas_b200.so")

IMPL_AUTO, IMPL_SIMT, IMPL_TC, IMPL_TC3 = 0, 1, 2, 3
CONV_S1, CONV_S2, CONV_UP, CONV_ZS = 0, 1, 2, 3
CONV_UP_PHASE, CONV_S2_PHASE = 4, 5   # phase-decomposed Upsample / Downsample (mas_conv3x3_phase_tc16h)


class Tensor4(ctypes.Structure):
    _fields_ = [(k, ctypes.c_int64) for k in ("n", "h", "w", "c", "sn", "sh", "sw", "sc")]


_P, _I, _L, _F, _D, _Z, _T = (ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_float, ctypes.c_double,
                              ctypes.c_size_t, Tensor4)

# name -> (restype, argtypes); mirrors include/mas_b200.h one to one
_SPEC = {
    "mas_version": (_I, []),
    "mas_last_error": (ctypes.c_char_p, []),
    "mas_launch_count": (_L, []),
    "mas_tc_launch_count": (_L, []),
    "mas_launch_trace": (_I, [_I]),
    "mas_launch_trace_read": (_L, [_P, _L]),
    "mas_ffma_probe": (_I, [_P, _I, _P, _P]),
    "mas_copy_strided": (_I, [_P, _T, _P, _T, _P]),
    "mas_nchw_to_nhwc_pad": (_I, [_P, _P, _I, _I, _I, _I, _I, _P]),
    "mas_scale_by": (_I, [_P, _P, _P, _L, _P]),
    "mas_gn_ws_bytes": (_Z, [_I, _I, _I, _I]),
    "mas_gn_stats": (_I, [_P, _I, _I, _I, _I, _F, _P, _P, _P, _Z, _P]),
    "mas_gn_apply": (_I, [_P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _P]),
    "mas_gn_backward": (_I, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _I, _P, _P, _P, _P, _I, _I, _I, _I, _I, _P, _Z, _P]),
    "mas_add": (_I, [_P, _P, _P, _L, _P]),
    "mas_silu_forward": (_I, [_P, _P, _L, _P]),
    "mas_silu_backward": (_I, [_P, _P, _P, _L, _P]),
    "mas_pack_conv3x3": (_I, [_P, _P, _I, _I, _I, _I, _P]),
    "mas_conv3x3_fprop": (_I, [_P, _T, _P, _P, _P, _P, _T, _I, _I, _P]),
    "mas_tc_probe": (_I, [_P, _P, _P, _I, _I, ctypes.c_uint64, ctypes.c_uint32, _I, _P]),
    "mas_tc_probe16": (_I, [_P, ctypes.c_uint64, ctypes.c_uint32, _I, _P]),
    "mas_conv3x3_tc_eligible": (_I, [_T, _T, _I]),
    "mas_pack_conv3x3_tc": (_I, [_P, _P, _I, _I, _I, _P]),
    "mas_pack_conv3x3_tc_pair": (_I, [_P, _P, _P, _I, _I, _P]),
    "mas_conv3x3_fprop_tc": (_I, [_P, _T, _P, _P, _P, _P, _T, _I, _P, _I, _P, _P]),
    "mas_amax": (_I, [_P, _L, _P, _P]),
    "mas_pack_conv3x3_tc16": (_I, [_P, _P, _P, _I, _I, _I, _P]),
    "mas_conv3x3_fprop_tc16": (_I, [_P, _T, _P, _P, _P, _P, _T, _I, _P, _I, _P, _P, _P]),
    "mas_conv3x3_tc16h_eligible": (_I, [_T, _T]),
    "mas_conv3x3_fprop_tc16h": (_I, [_P, _T, _P, _P, _P, _P, _T, _P, _P, _P]),
    "mas_to_half": (_I, [_P, _P, _L, _P, _P]),
    "mas_pack_conv3x3_phase16": (_I, [_P, _P, _I, _I, _I, _I, _P]),
    "mas_conv3x3_phase_tc16h": (_I, [_P, _T, _P, _P, _P, _T, _I, _I, _P, _P]),
    "mas_conv3x3_phase_wgrad_tc16_ws_bytes": (_Z, [_T, _T, _I]),
    "mas_conv3x3_phase_wgrad_tc16": (_I, [_P, _T, _P, _P, _T, _P, _P, _P, _I, _P, _Z, _P]),
    "mas_gn_finalize_partials": (_I, [_P, _I, _I, _I, _I, _L, _F, _P, _P, _P]),
    "mas_gn_table": (_I, [_P, _P, _P, _P, _I, _I, _I, _P, _P]),
    "mas_pack_gemm_tc": (_I, [_P, _P, _I, _I, _I, _P]),
    "mas_gemm_rows_packed": (_I, [_P, _L, _P, _P, _L, _L, _I, _I, _F, _P, _P, _P, _P]),
    "mas_conv3x3_wgrad_ws_bytes": (_Z, [_T, _T, _I]),
    "mas_conv3x3_wgrad": (_I, [_P, _T, _P, _T, _P, _P, _I, _I, _P, _I, _P, _Z, _P]),
    "mas_conv3x3_wgrad_tc_eligible": (_I, [_T, _T, _I]),
    "mas_conv3x3_wgrad_tc16": (_I, [_P, _I, _T, _P, _T, _P, _P, _I, _P, _I, _P, _I, _P, _Z, _P]),
    "mas_conv1x1_wgrad_ws_bytes": (_Z, [_L, _I, _I]),
    "mas_conv1x1_wgrad": (_I, [_P, _L, _P, _L, _L, _I, _I, _P, _P, _I, _P, _Z, _P]),
    "mas_edge_small_cin_fprop": (_I, [_P, _T, _P, _P, _P, _T, _I, _P]),
    "mas_edge_small_cout_fprop": (_I, [_P, _T, _P, _P, _P, _T, _P]),
    "mas_edge_wgrad_ws_bytes": (_Z, [_I]),
    "mas_edge_small_cin_wgrad": (_I, [_P, _T, _P, _T, _P, _P, _P, _Z, _P]),
    "mas_edge_small_cout_wgrad": (_I, [_P, _T, _P, _T, _P, _P, _P, _Z, _P]),
    "mas_space_to_depth": (_I, [_P, _P, _I, _I, _I, _I, _P]),
    "mas_s2d_pack_weights": (_I, [_P, _P, _I, _I, _P]),
    "mas_s2d_unpack_wgrad": (_I, [_P, _P, _I, _I, _P]),
    "mas_sumpool2x2": (_I, [_P, _P, _I, _I, _I, _I, _P]),
    "mas_gemm": (_I, [_P, _P, _P, _I, _I, _I, _I, _L, _L, _L, _L, _L, _L, _I, _I, _F, _P, _P, _I, _P]),
    "mas_colsum_ws_bytes": (_Z, [_T]),
    "mas_colsum": (_I, [_P, _T, _P, _P, _Z, _P]),
    "mas_attnblock_ws_bytes": (_Z, [_I, _I, _I, _I]),
    "mas_attnblock_forward": (_I, [_P, _I, _I, _I, _I] + [_P] * 18 + [_I, _P, _Z, _P]),
    "mas_attnblock_backward": (_I, [_P, _P, _I, _I, _I, _I] + [_P] * 20 + [_I, _P, _Z, _P]),
    "mas_softmax_forward": (_I, [_P, _P, _L, _I, _P]),
    "mas_softmax_backward": (_I, [_P, _P, _P, _L, _I, _F, _P]),
    "mas_bn_stats": (_I, [_P, _L, _I, _P, _P]),
    "mas_bn_finalize": (_I, [_P, _D, _I, _F, _F, _P, _P, _P, _P, _P]),
    "mas_bn_invstd": (_I, [_P, _F, _P, _I, _P]),
    "mas_bn_apply": (_I, [_P, _P, _P, _P, _P, _P, _L, _I, _P]),
    "mas_bn_backward_reduce": (_I, [_P, _P, _P, _P, _L, _I, _P, _P]),
    "mas_bn_backward_apply": (_I, [_P, _P, _P, _P, _P, _P, _P, _D, _P, _P, _P, _L, _I, _P]),
    "mas_pack_conv4x4": (_I, [_P, _P, _I, _I, _I, _P]),
    "mas_conv4x4": (_I, [_P, _T, _P, _P, _P, _T, _I, _F, _I, _P]),
    "mas_conv4x4_dgrad": (_I, [_P, _T, _P, _P, _T, _I, _P]),
    "mas_conv4x4_wgrad_ws_bytes": (_Z, [_T, _T]),
    "mas_conv4x4_wgrad": (_I, [_P, _T, _P, _T, _P, _I, _P, _Z, _P]),
    "mas_lrelu_backward": (_I, [_P, _P, _F, _P, _L, _P]),
    "mas_bn_apply_lrelu": (_I, [_P, _P, _P, _P, _P, _F, _P, _L, _I, _P]),
    "mas_bn_backward_reduce_lrelu_ws_bytes": (_Z, [_L, _I]),
    "mas_bn_backward_reduce_lrelu": (_I, [_P, _P, _F, _P, _P, _P, _L, _I, _P, _P, _Z, _P]),
    "mas_conv4x4_shift_map": (_I, [_P, _T, _P, _I, _P]),
    "mas_conv4x4_shift_map_adjoint": (_I, [_P, _P, _T, _I, _P]),
    "mas_conv4x4_remap_weight": (_I, [_P, _P, _I, _I, _I, _I, _P]),
    "mas_bn_backward_apply_lrelu": (_I, [_P, _P, _F, _P, _P, _P, _P, _P, _P, _P, _P, _L, _I, _P]),
    "mas_vq_select_path": (_I, [_I]),
    "mas_vq_ws_bytes": (_Z, [_L, _I, _I]),
    "mas_vq_forward": (_I, [_P, _P, _L, _I, _I, _F, _P, _P, _P, _P, _Z, _P]),
    "mas_vq_forward_given": (_I, [_P, _P, _P, _L, _I, _I, _F, _P, _P, _P, _Z, _P]),
    "mas_kmeans_ws_bytes": (_Z, [_I, _I]),
    "mas_kmeans_update": (_I, [_P, _P, _L, _I, _I, _P, _P, _P, _P, _Z, _P]),
    "mas_vq_backward": (_I, [_P, _P, _P, _P, _P, _L, _I, _I, _F, _P, _P, _P]),
    "mas_vq_gather": (_I, [_P, _P, _L, _I, _I, _P, _P]),
    "mas_layernorm_forward": (_I, [_P, _P, _P, _P, _P, _P, _P, _L, _I, _F, _P]),
    "mas_layernorm_ws_bytes": (_Z, [_L, _I]),
    "mas_layernorm_backward": (_I, [_P, _P, _P, _P, _P, _P, _P, _P, _L, _I, _P, _Z, _P]),
    "mas_gelu_forward": (_I, [_P, _P, _L, _P]),
    "mas_gelu_backward": (_I, [_P, _P, _P, _L, _P]),
    "mas_softmax_causal_forward": (_I, [_P, _P, _L, _I, _I, _P]),
    "mas_embed3_forward": (_I, [_P, _P, _P, _P, _P, _P, _P, _L, _I, _I, _I, _I, _P]),
    "mas_embed3_backward": (_I, [_P, _P, _P, _P, _P, _P, _P, _L, _I, _I, _I, _I, _P]),
    "mas_linear_small": (_I, [_P, _L, _P, _P, _P, _L, _I, _I, _I, _I, _P]),
    "mas_kv_append": (_I, [_P, _I, _I, _I, _I, _P, _P, _I, _I, _P]),
    "mas_attn_decode": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _P]),
    "mas_cfg_mix": (_I, [_P, _P, _P, _L, _F, _P]),
    "mas_cfg_mix_rows": (_I, [_P, _P, _P, _I, _L, _P, _P]),
    "mas_attn_decode_append": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _P]),
    "mas_kv_append_f16": (_I, [_P, _I, _I, _I, _I, _P, _P, _I, _I, _P]),
    "mas_attn_decode_f16": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _P]),
    "mas_attn_decode_append_f16": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _P]),
    "mas_attn_decode_shared_append": (_I, [_P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _P]),
    "mas_attn_decode_shared_append_f16": (_I, [_P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _P]),
    "mas_attn_decode_shared": (_I, [_P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _P]),
    "mas_attn_decode_shared_f16": (_I, [_P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _P]),
    "mas_layernorm2_forward": (_I, [_P, _P, _P, _P, _P, _P, _P, _P, _L, _I, _F, _F, _P]),
    "mas_sample_topk": (_I, [_P, _L, _I, _I, _F, _I, _P, _P, _P]),
    "mas_sample_filtered": (_I, [_P, _L, _I, _I, _F, _I, _F, _P, _P, _P, _L, _P, _P]),
    "mas_sample_filtered_logp": (_I, [_P, _L, _I, _I, _F, _I, _F, _P, _P, _P, _L, _P, _P, _L, _P]),
    "mas_sample_rows": (_I, [_P, _L, _I, _I, _P, _P, _P, _P, _P, _L, _P, _P, _L, _P, _P, _L, _P]),
    "mas_pack_gemm_tc16": (_I, [_P, _P, _I, _I, _I, _P]),
    "mas_gemm_rows_f16": (_I, [_P, _L, _I, _P, _P, _L, _I, _P, _P, _P, _F, _P]),
    "mas_linear_rows_f16_ws_bytes": (_Z, [_L, _I, _I]),
    "mas_linear_rows_f16": (_I, [_P, _L, _I, _P, _P, _L, _I, _P, _P, _I, _P, _Z, _P]),
    "mas_wgrad_rows_f16_ws_bytes": (_Z, [_L, _I, _I]),
    "mas_wgrad_rows_f16": (_I, [_P, _P, _L, _I, _I, _P, _P, _P, _P, _P, _Z, _P]),
    "mas_to_fp8_ws_bytes": (_Z, [_L, _I]),
    "mas_to_fp8": (_I, [_P, _L, _I, _I, _P, _P, _P, _P, _P, _Z, _P]),
    "mas_pack_gemm_f8": (_I, [_P, _I, _I, _P, _P, _P, _P]),
    "mas_gemm_rows_f8": (_I, [_P, _L, _I, _I, _P, _P, _I, _P, _P, _P, _L, _P]),
    "mas_wgrad_rows_f8_ws_bytes": (_Z, [_L, _I, _I]),
    "mas_wgrad_rows_f8": (_I, [_P, _P, _L, _I, _I, _P, _P, _P, _P, _Z, _P]),
    "mas_attn_causal_forward": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _F, _P]),
    "mas_attn_causal_forward_stats": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _F, _D, _P, _P]),
    "mas_attn_causal_backward": (_I, [_P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _F, _D, _P, _P]),
    "mas_attn_causal_prefix_forward": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _F, _P]),
    "mas_dropout": (_I, [_P, _P, _P, _L, _D, _F, _P, _P]),
    "mas_attn_causal_dropout_forward": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _F, _D, _P, _P]),
    "mas_softmax_causal_dropout_backward": (_I, [_P, _P, _P, _L, _I, _I, _F, _D, _P, _P]),
    "mas_layernorm_dropout_forward": (_I, [_P, _P, _P, _P, _P, _P, _P, _L, _I, _F, _D, _P, _P]),
    "mas_layernorm_dropout_backward": (_I, [_P, _P, _P, _P, _P, _P, _P, _P, _L, _I, _D, _P, _P, _Z, _P]),
    "mas_ce_forward": (_I, [_P, _L, _P, _P, _P, _P, _L, _I, _P]),
    "mas_ce_backward": (_I, [_P, _L, _P, _P, _P, _P, _P, _L, _L, _I, _P]),
    "mas_gemm_batched2": (_I, [_P, _P, _P, _I, _I, _I, _I, _I, _L, _L, _L, _L, _L, _L, _L, _L, _L, _I, _I, _F, _I, _I, _P]),
    "mas_softmax_causal_backward": (_I, [_P, _P, _P, _L, _I, _I, _F, _P]),
    "mas_bce_ws_bytes": (_Z, [_T]),
    "mas_bce_cl_ws_bytes": (_Z, [_I, _I, _I]),
    "mas_bce_cl_forward": (_I, [_P, _P, _P, _I, _I, _I, _I, _I, _P, _P, _Z, _P]),
    "mas_bce_cl_backward": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _P, _P]),
    "mas_bce_logits": (_I, [_P, _T, _P, _T, _P, _P, _P, _T, _F, _P, _Z, _P]),
    "mas_scene_expand": (_I, [_P, _I, _I, _I, _P, _T, _P]),
    "mas_scene_decode": (_I, [_P, _T, _P, _P]),
    "mas_scene_confusion_ws_bytes": (_Z, [_L, _I]),
    "mas_scene_confusion": (_I, [_P, _P, _L, _I, _P, _P, _Z, _P]),
    "mas_image_quality_ws_bytes": (_Z, [_I, _I, _L, _L]),
    "mas_image_quality": (_I, [_P, _T, _P, _T, _P, _P, _P, _Z, _P]),
    "mas_bce_scene_forward": (_I, [_P, _P, _P, _I, _I, _I, _I, _P, _P, _Z, _P]),
    "mas_bce_scene_backward": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _P, _P]),
    "mas_bce_mse_cl_forward": (_I, [_P, _P, _P, _I, _I, _I, _I, _I, _P, _P, _Z, _P]),
    "mas_bce_mse_cl_backward": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _P, _P]),
    "mas_bce_mse_scene_forward": (_I, [_P, _P, _P, _I, _I, _I, _I, _P, _P, _Z, _P]),
    "mas_bce_mse_scene_backward": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _P, _P]),
    "mas_bce_mse_logits": (_I, [_P, _T, _P, _T, _P, _P, _P, _T, _F, _P, _Z, _P]),
    "mas_lpips_prep": (_I, [_P, _P, _P, _P, _P, _I, _I, _I, _P]),
    "mas_lpips_relu": (_I, [_P, _L, _P, _P]),
    "mas_lpips_maxpool": (_I, [_P, _P, _I, _I, _I, _I, _P, _P]),
    "mas_lpips_head_blocks": (_I, []),
    "mas_lpips_head_forward": (_I, [_P, _P, _I, _I, _I, _I, _P, _P]),
    "mas_lpips_head_finalize": (_I, [_P, _I, _L, _L, _L, _L, _L, _P, _P]),
    "mas_lpips_tap_backward": (_I, [_P, _P, _I, _I, _I, _I, _I, _I, _P, _P, _P, _P]),
    "mas_lpips_relu_backward": (_I, [_P, _P, _P, _L, _P, _P]),
    "mas_lpips_prep_backward": (_I, [_P, _P, _P, _I, _I, _I, _P]),
    "mas_lpips_scale_jacobian": (_I, [_P, _P, _L, _P, _I, _L, _P]),
    "mas_object_gather": (_I, [_P, _I, _P, _P, _P, _P, _P, _I, _I, _I, _I, _P]),
    "mas_object_relu": (_I, [_P, _P, _I, _I, _I, _I, _I, _P, _P]),
    "mas_object_maxpool": (_I, [_P, _P, _P, _I, _I, _I, _I, _I, _P, _P]),
    "mas_object_head_forward": (_I, [_P, _P, _P, _I, _I, _I, _I, _I, _P, _P]),
    "mas_object_head_finalize": (_I, [_P, _P, _I, _P, _P]),
    "mas_object_tap_backward": (_I, [_P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _P, _P, _P, _P]),
    "mas_object_scatter": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _P, _I, _I, _I, _I, _P]),
    "mas_object_loss": (_I, [_P, _P, _I, _P, _P]),
    "mas_face_prepare": (_I, [_P, _P, _I, _P, _T, _P, _T, _P, _P]),
    "mas_face_prepare_backward": (_I, [_P, _P, _I, _I, _I, _P, _P, _I, _I, _I, _P]),
    "mas_face_stem_forward": (_I, [_P, _P, _P, _I, _I, _I, _P]),
    "mas_face_stem_backward": (_I, [_P, _P, _P, _I, _I, _I, _P]),
    "mas_face_pool_forward": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _P, _P]),
    "mas_face_pool_backward": (_I, [_P, _P, _P, _P, _P, _F, _I, _I, _I, _I, _I, _I, _P, _P]),
    "mas_face_l1_blocks": (_I, []),
    "mas_face_l1_forward": (_I, [_P, _L, _P, _P, _P]),
    "mas_face_l1_finalize": (_I, [_P, _D, _D, _D, _D, _D, _P, _P, _P]),
    "mas_face_subsample_half": (_I, [_P, _P, _I, _I, _I, _I, _P, _P]),
    "mas_face_relu_seed_backward": (_I, [_P, _P, _I, _P, _F, _I, _I, _I, _I, _I, _I, _P, _P, _P]),
}

_lib = None


def exported_symbols():
    return sorted(_SPEC)


def load():
    """Load the shared library (once). Raises RuntimeError if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"libmas_b200.so not found at {LIB_PATH}: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a). There is no CPU/PyTorch fallback for this path.")
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in _SPEC.items():
        fn = getattr(lib, name)  # AttributeError here = header/library drift, which must be loud
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def _ptr(t):
    if t is None:
        return None
    if isinstance(t, torch.Tensor):
        return ctypes.c_void_p(t.data_ptr())
    return t


def stream_ptr():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


_prof = None   # when a list: (name, start_event, end_event) per call — see profile_start/profile_report


def _device_of(args):
    for a in args:
        if isinstance(a, torch.Tensor) and a.is_cuda:
            return a.device
    return None


def call(name, *args):
    """Invoke an int-returning entry on the current CUDA stream of the tensors' device; non-zero status -> RuntimeError.
    A model living on a device other than torch.cuda.current_device() is served by switching to it for the call."""
    dev = _device_of(args)
    if dev is not None and dev.index != torch.cuda.current_device():
        with torch.cuda.device(dev):
            return call(name, *args)
    lib = load()
    fn = getattr(lib, name)
    conv = [_ptr(a) for a in args]
    conv.append(stream_ptr())
    if _prof is not None:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        rc = fn(*conv)
        e1.record()
        shp = ",".join("%dc%d" % (a.c, a.h) for a in args if isinstance(a, Tensor4))
        if not shp and name.startswith("mas_gn_"):   # (N, HW, C) travel as plain ints there
            ints = [a for a in args if isinstance(a, int) and not isinstance(a, bool)]
            shp = "x".join(str(v) for v in ints[:3])
        _prof.append((name + ("|" + shp if shp else ""), e0, e1))
    else:
        rc = fn(*conv)
    if rc != 0:
        raise RuntimeError(f"{name} failed ({rc}): {lib.mas_last_error().decode(errors='replace')}")


def profile_start():
    """Measurement aid: time every C-ABI call with CUDA events (no profiler attached, kernels run at full speed)."""
    global _prof
    _prof = []


def profile_report(tag=None):
    """Returns {entry name: (calls, total ms)} since profile_start() and stops profiling."""
    global _prof
    torch.cuda.synchronize()
    agg = {}
    for name, e0, e1 in _prof or []:
        key = name if tag is None else tag(name)
        c, t = agg.get(key, (0, 0.0))
        agg[key] = (c + 1, t + e0.elapsed_time(e1))
    _prof = None
    return agg


def query(name, *args):
    """Invoke a size-returning helper (no stream argument)."""
    return getattr(load(), name)(*[_ptr(a) for a in args])


def launch_count() -> int:
    return int(load().mas_launch_count())


def tc_launch_count() -> int:
    """Launches of kernels that issue tensor-core (wgmma) MMAs (subset of launch_count)."""
    return int(load().mas_tc_launch_count())


@contextlib.contextmanager
def launch_trace():
    """Yields a list that, when the block ends, holds the name of every kernel the library launched inside it, in launch
    order (mas_launch_trace: recorded on the host at launch, so no profiler is needed and none can drop an entry)."""
    lib = load()
    names = []
    lib.mas_launch_trace(1)
    try:
        yield names
    finally:
        n = int(lib.mas_launch_trace_read(None, 0))
        buf = ctypes.create_string_buffer(n + 1)
        lib.mas_launch_trace_read(buf, n + 1)
        lib.mas_launch_trace(0)
        names.extend(buf.value.decode().splitlines())


def t4(x: torch.Tensor) -> Tensor4:
    """Describe a logical [N,C,H,W] tensor (any strides) as extents + element strides."""
    n, c, h, w = x.shape
    sn, sc, sh, sw = x.stride()
    return Tensor4(n, h, w, c, sn, sh, sw, sc)


def rows4(m: int, c: int) -> Tensor4:
    return Tensor4(1, 1, m, c, m * c, m * c, c, 1)


_ws = {}


def workspace(nbytes: int, device) -> torch.Tensor:
    """Grow-only per-device scratch buffer (all kernels of this library run on the current stream, so a
    single buffer is race-free)."""
    key = (device.type, device.index)
    buf = _ws.get(key)
    if buf is None or buf.numel() < nbytes:
        buf = torch.empty(max(int(nbytes), 1 << 20), dtype=torch.uint8, device=device)
        _ws[key] = buf
    return buf


def pin_workspaces():
    """References to the current scratch buffers (a CUDA graph that recorded their addresses keeps them alive through
    this list; workspace() replaces — never resizes in place — a buffer that is too small)."""
    return list(_ws.values())
