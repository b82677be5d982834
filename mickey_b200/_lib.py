"""ctypes binding of libmickey_b200.so (the C ABI declared in include/mickey_b200.h), and the rules every caller follows
at that boundary: the stream argument, workspace allocation, the row pitch of N x N arguments and the handle's lifetime.

There is no fallback: if the shared library is missing or does not load, importing the binding
raises with the build command — the product path never routes around the CUDA extension.
"""
from __future__ import annotations

import ctypes as C
import math
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_C", "libmickey_b200.so")


class MkConfig(C.Structure):
    _fields_ = [
        ("embed_dim", C.c_int), ("depth", C.c_int), ("heads", C.c_int),
        ("down_factor", C.c_int),
        ("block_dims", C.c_int * 4),
        ("desc_dim", C.c_int),
        ("use_softmax", C.c_int), ("depth_sigmoid", C.c_int), ("max_depth", C.c_float),
        ("kp_pos_enc", C.c_int), ("dsc_pos_enc", C.c_int), ("norm_dsc", C.c_int),
        ("temperature", C.c_float), ("use_dustbin", C.c_int),
        ("it_matches", C.c_int), ("it_ransac", C.c_int),
        ("num_sampled", C.c_int), ("num_corr", C.c_int), ("num_refine", C.c_int),
        ("th_inlier", C.c_float), ("th_soft_inlier", C.c_float),
    ]


class MkGemmArgs(C.Structure):
    _fields_ = [
        ("epi", C.c_int), ("impl", C.c_int),
        ("a", C.c_void_p), ("a_rows", C.c_longlong), ("a_cols", C.c_longlong), ("a_ld", C.c_longlong),
        ("b", C.c_void_p), ("b_rows", C.c_longlong), ("b_cols", C.c_longlong), ("b_ld", C.c_longlong),
        ("M", C.c_int), ("N", C.c_int), ("k_chunks", C.c_int), ("chunks_per_tap", C.c_int), ("num_taps", C.c_int),
        ("tap_shift", C.c_int * 9),
        ("groups", C.c_int), ("a_row_group_off", C.c_int), ("a_col_group_off", C.c_int), ("a_col_base", C.c_int),
        ("b_row_group_off", C.c_int),
        ("act", C.c_int),
        ("bias", C.c_void_p), ("bias_group_off", C.c_int),
        ("gamma", C.c_void_p), ("beta", C.c_void_p), ("ln_group_off", C.c_int),
        ("out_f", C.c_void_p), ("out_f_ld", C.c_longlong), ("out_f_group_off", C.c_longlong),
        ("out_h", C.c_void_p), ("out_h_ld", C.c_longlong), ("out_h_group_off", C.c_longlong),
        ("res_h", C.c_void_p), ("res_h_ld", C.c_longlong), ("res_h_group_off", C.c_longlong),
        ("aux", C.c_void_p), ("aux_group_mask", C.c_int),
        ("pad_h2", C.c_int), ("pad_w2", C.c_int), ("tok_per_img", C.c_int),
        ("eps", C.c_float),
        ("n_valid", C.c_int), ("inv_temp", C.c_float),
        ("dustbin", C.c_void_p),
        ("part_row", C.c_void_p), ("part_col", C.c_void_p), ("part_ld", C.c_int),
        ("lse_r", C.c_void_p), ("lse_c", C.c_void_p), ("scr0", C.c_void_p), ("scr1", C.c_void_p),
        ("scores", C.c_void_p), ("kp_scores", C.c_void_p), ("final_scores", C.c_void_p),
        ("lse_bound", C.c_float),
        ("out_pitch", C.c_longlong),
    ]


class MkHtrLayer(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("q_proj", "k_proj", "v_proj", "merge", "mlp0", "mlp2",
                                          "norm1_w", "norm1_b", "norm2_w", "norm2_b")]


MkHtrLayerGrads = MkHtrLayer     # the same ten pointers, written instead of read


class MkResblockParams(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("w1", "w2", "wsc", "bn1_w", "bn1_b", "bn1_mean", "bn1_var",
                                          "bn2_w", "bn2_b", "bn2_mean", "bn2_var")] + \
               [(n, C.c_float) for n in ("eps1", "eps2", "momentum1", "momentum2")]


class MkResblockGrads(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("dx", "w1", "w2", "wsc", "bn1_w", "bn1_b", "bn2_w", "bn2_b")]


EXPORTS = {
    # name: (restype, argtypes)
    "mk_create": (C.c_int, [C.c_int, C.POINTER(MkConfig), C.POINTER(C.c_void_p)]),
    "mk_destroy": (C.c_int, [C.c_void_p]),
    "mk_last_error": (C.c_char_p, []),
    "mk_version": (C.c_char_p, []),
    "mk_sizeof": (C.c_int, [C.c_char_p]),
    "mk_set_tensor": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int, C.c_longlong]),
    "mk_finalize": (C.c_int, [C.c_void_p, C.c_int, C.c_int]),
    "mk_workspace_bytes": (C.c_longlong, [C.c_void_p, C.c_int, C.c_int, C.c_int]),
    "mk_workspace_offset": (C.c_longlong, [C.c_void_p, C.c_char_p, C.c_int, C.c_int, C.c_int]),
    "mk_extract": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                             C.c_void_p, C.c_void_p, C.c_longlong, C.c_void_p]),
    "mk_extract_u8": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                C.c_void_p, C.c_void_p, C.c_longlong, C.c_void_p]),
    "mk_workspace_bytes_for": (C.c_longlong, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int]),
    "mk_extract_images": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                    C.c_void_p, C.c_void_p, C.c_longlong, C.c_void_p]),
    "mk_extract_images_u8": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.c_void_p, C.c_longlong, C.c_void_p]),
    "mk_forward_pairs": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                   C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                   C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_ulonglong,
                                   C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_longlong,
                                   C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_longlong,
                                   C.c_void_p]),
    "mk_localize": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                              C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_ulonglong,
                              C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_longlong,
                              C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_longlong,
                              C.c_void_p]),
    "mk_localize_u8": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                 C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_ulonglong,
                                 C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                 C.c_longlong, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                 C.c_longlong, C.c_void_p]),
    "mk_backbone_ws_bytes": (C.c_longlong, [C.c_void_p, C.c_int, C.c_int, C.c_int]),
    "mk_backbone_features": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                       C.c_longlong, C.c_void_p]),
    "mk_match": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_longlong, C.c_void_p, C.c_longlong, C.c_void_p]),
    "mk_solve_pose": (C.c_int, [C.c_void_p, C.c_void_p, C.c_longlong, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                C.c_ulonglong, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                C.c_void_p, C.c_void_p, C.c_void_p, C.c_longlong, C.c_void_p]),
    "mk_procrustes_ws_bytes": (C.c_longlong, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]),
    "mk_procrustes_solve": (C.c_int, [C.c_void_p, C.c_longlong, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                      C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float,
                                      C.c_ulonglong, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_longlong, C.c_void_p]),
    "mk_mapfree_frame_metrics": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                           C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "mk_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_ulonglong,
                             C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_longlong,
                             C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_longlong,
                             C.c_void_p]),
    "mk_forward_u8": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_ulonglong,
                                C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_longlong,
                                C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_longlong,
                                C.c_void_p]),
    "mk_mutual_matches": (C.c_int, [C.c_void_p, C.c_longlong, C.c_int, C.c_int, C.c_float, C.c_void_p, C.c_void_p,
                                    C.c_void_p, C.c_void_p, C.c_longlong, C.c_void_p]),
    "mk_mutual_matches_ws_bytes": (C.c_longlong, [C.c_int, C.c_int]),
    "mk_loss_search": (C.c_int, [C.c_void_p, C.c_longlong, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                 C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float,
                                 C.c_ulonglong, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                 C.c_void_p, C.c_longlong, C.c_void_p]),
    "mk_loss_search_ws_bytes": (C.c_longlong, [C.c_int, C.c_int]),
    "mk_loss_gradient": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                   C.c_void_p, C.c_void_p, C.c_longlong, C.c_void_p]),
    "mk_loss_gradient_ws_bytes": (C.c_longlong, [C.c_int, C.c_int, C.c_int]),
    "mk_loss_tail_ws_bytes": (C.c_longlong, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]),
    "mk_loss_tail_forward": (C.c_int, [C.c_void_p] * 12 + [C.c_int] * 8 + [C.c_float] * 4 + [C.c_void_p] * 5
                             + [C.c_longlong, C.c_void_p]),
    "mk_loss_tail_backward": (C.c_int, [C.c_void_p] * 12 + [C.c_int] * 8 + [C.c_float] * 2 + [C.c_void_p] * 8
                              + [C.c_longlong, C.c_void_p]),
    "mk_dual_softmax_ws_bytes": (C.c_longlong, [C.c_int, C.c_int]),
    "mk_dual_softmax_backward_ws_bytes": (C.c_longlong, [C.c_int, C.c_int]),
    "mk_dual_softmax": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_int, C.c_int,
                                  C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_longlong, C.c_void_p, C.c_void_p,
                                  C.c_void_p, C.c_longlong, C.c_void_p]),
    "mk_dual_softmax_backward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_int,
                                           C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_longlong, C.c_void_p,
                                           C.c_longlong, C.c_void_p, C.c_longlong, C.c_void_p, C.c_void_p, C.c_void_p,
                                           C.c_void_p, C.c_void_p, C.c_void_p, C.c_longlong, C.c_void_p]),
    "mk_head_transformer_ws_bytes": (C.c_longlong, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]),
    "mk_head_transformer_backward_ws_bytes": (C.c_longlong, [C.c_int, C.c_int, C.c_int, C.c_int]),
    "mk_head_transformer": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.POINTER(MkHtrLayer), C.c_int,
                                      C.c_void_p, C.c_int, C.c_void_p, C.c_longlong, C.c_void_p]),
    "mk_head_transformer_backward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.POINTER(MkHtrLayer),
                                               C.c_int, C.c_void_p, C.POINTER(MkHtrLayerGrads), C.c_void_p, C.c_longlong,
                                               C.c_void_p]),
    "mk_resblock_ws_bytes": (C.c_longlong, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]),
    "mk_resblock_saved_bytes": (C.c_longlong, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]),
    "mk_resblock_backward_ws_bytes": (C.c_longlong, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]),
    "mk_resblock_forward": (C.c_int, [C.c_void_p, C.POINTER(C.c_longlong), C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                      C.POINTER(MkResblockParams), C.c_int, C.c_void_p, C.c_void_p, C.c_longlong,
                                      C.c_void_p, C.c_longlong, C.c_void_p]),
    "mk_resblock_layout": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_longlong),
                                     C.POINTER(C.c_longlong)]),
    "mk_resblock_backward": (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(C.c_longlong), C.c_void_p, C.c_int, C.c_int,
                                       C.c_int, C.c_int, C.c_int, C.POINTER(MkResblockParams), C.c_int, C.c_int,
                                       C.POINTER(MkResblockGrads), C.c_void_p, C.c_longlong, C.c_void_p]),
    "mk_head_out_backward_ws_bytes": (C.c_longlong, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]),
    "mk_head_out_forward": (C.c_int, [C.c_int, C.c_void_p, C.POINTER(C.c_longlong), C.c_int, C.c_int, C.c_int, C.c_int,
                                      C.c_void_p, C.c_void_p, C.c_float, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p]),
    "mk_head_out_backward": (C.c_int, [C.c_int, C.c_void_p, C.POINTER(C.c_longlong), C.c_int, C.c_int, C.c_int, C.c_int,
                                       C.c_void_p, C.c_float, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.c_void_p, C.c_longlong, C.c_void_p]),
    "mk_pose_to_submission": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "mk_launch_count": (C.c_longlong, [C.c_void_p]),
    "mk_pdl_enabled": (C.c_int, []),
    "mk_set_seed": (C.c_int, [C.c_void_p, C.c_ulonglong, C.c_void_p]),
    "mk_profile_enable": (C.c_int, [C.c_void_p, C.c_int]),
    "mk_profile_read": (C.c_int, [C.c_void_p, C.c_char_p, C.c_int]),
    "mk_op_gemm": (C.c_int, [C.POINTER(MkGemmArgs), C.c_void_p]),
    "mk_op_patch_gather": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                     C.c_int, C.c_void_p]),
    "mk_op_ingest_u8": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                  C.c_int, C.c_void_p]),
    "mk_op_layernorm": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_int,
                                  C.c_int, C.c_int, C.c_void_p]),
    "mk_op_attention": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "mk_op_linattn": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_void_p]),
    "mk_op_matcher_reduce": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "mk_op_sample": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_longlong, C.c_int, C.c_int, C.c_ulonglong, C.c_void_p, C.c_longlong,
                               C.c_void_p, C.c_void_p, C.c_void_p]),
    "mk_op_sample_workspace_bytes": (C.c_longlong, [C.c_int, C.c_int]),
    "mk_op_kabsch": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    "mk_op_conv_tf32_ws_bytes": (C.c_longlong, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]),
    "mk_op_conv_tf32": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                  C.c_int, C.c_void_p, C.c_longlong, C.c_void_p]),
}

# every struct the binding passes, by its C name: load() checks each size against the library's
STRUCTS = {"mk_config": MkConfig, "mk_gemm_args": MkGemmArgs, "mk_htr_layer": MkHtrLayer,
           "mk_htr_layer_grads": MkHtrLayerGrads, "mk_resblock_params": MkResblockParams,
           "mk_resblock_grads": MkResblockGrads}

_lib = None


class MickeyB200Error(RuntimeError):
    pass


def load():
    """Load the shared library (once) and declare every exported signature."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise MickeyB200Error(
            f"{LIB_PATH} not found. Build it with `python -m mickey_b200.build` (needs nvcc; sm_90a only). "
            "mickey_b200 has no CPU or PyTorch fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in EXPORTS.items():
        fn = getattr(lib, name)          # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    sizes = {name: (lib.mk_sizeof(name.encode()), C.sizeof(st)) for name, st in STRUCTS.items()}
    bad = [f"{name} {lib_size} vs {py_size}" for name, (lib_size, py_size) in sizes.items() if lib_size != py_size]
    if bad:
        raise MickeyB200Error("ctypes struct layout does not match the library (stale build?): " + ", ".join(bad))
    _lib = lib
    return lib


def check(rc: int, what: str = ""):
    if rc != 0:
        msg = load().mk_last_error().decode(errors="replace")
        raise MickeyB200Error(f"{what} failed (code {rc}): {msg}")


def ptr(t):
    """Device (or host) address of a torch tensor, or None."""
    return None if t is None else C.c_void_p(t.data_ptr())


def stream(dev=None):
    """The current CUDA stream of `dev` (None: the current device), as the library's `stream` argument."""
    return C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def workspace(nbytes, dev, what: str):
    """A uint8 buffer on `dev` for the byte count `nbytes` that the library's `what` (a mk_*_ws_bytes function) returned.
    A negative count is the library rejecting the arguments, and raises; a zero count still gets one byte, so the
    workspace pointer is never NULL."""
    nbytes = int(nbytes)
    if nbytes < 0:
        raise MickeyB200Error(f"{what} returned {nbytes}: {load().mk_last_error().decode(errors='replace')}")
    return torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)


def pitched(t):
    """(tensor, row pitch in floats) for an fp32 [B, N, N] argument of the library.  t itself when its rows are contiguous,
    at least N floats apart, and its matrices N row pitches apart (contiguous tensors, the engine's [B, N, pitch][:, :, :N]
    views); any other layout (transposed, expanded, ...) becomes a contiguous copy with pitch N."""
    B, N, _ = t.shape
    s0, s1, s2 = t.stride()
    if s2 == 1 and s1 >= N and (B == 1 or s0 == N * s1):
        return t, s1
    return t.contiguous(), N


class Handle:
    """An mk_handle of the library, created on `device` (a CUDA torch.device) for `cfg` (MkConfig) and destroyed with this
    object: the tensors registered with it and the named buffers of its workspaces."""

    def __init__(self, device, cfg: MkConfig):
        self.lib = load()
        self.device = device
        h = C.c_void_p()
        check(self.lib.mk_create(device.index or 0, C.byref(cfg), C.byref(h)), "mk_create")
        self.h = h

    def __del__(self):
        try:
            if getattr(self, "h", None):
                self.lib.mk_destroy(self.h)
        except Exception:
            pass

    def register(self, name: str, t):
        """mk_set_tensor: the handle reads t (contiguous fp32 or fp16 on the handle's device) as `name` from now on."""
        assert t.is_contiguous() and t.device == self.device
        dt = {torch.float32: 0, torch.float16: 1}[t.dtype]
        check(self.lib.mk_set_tensor(self.h, name.encode(), ptr(t), dt, t.numel()), f"mk_set_tensor({name})")

    def workspace_view(self, ws, n_pairs: int, H: int, W: int, name: str, dtype, shape):
        """Typed view of the named buffer of `ws`, a workspace laid out for n_pairs pairs of H x W images."""
        off = self.lib.mk_workspace_offset(self.h, name.encode(), n_pairs, H, W)
        if off < 0:
            raise MickeyB200Error(self.lib.mk_last_error().decode())
        nbytes = math.prod(shape) * torch.empty((), dtype=dtype).element_size()
        return ws[off:off + nbytes].view(dtype).reshape(shape)
