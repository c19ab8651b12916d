"""ctypes binding of the C-ABI declared in ``include/b200reco.h``.

There is NO fallback: if the shared library is missing or fails to load the
import raises.  Device memory and streams come from torch (plumbing only).
"""
from __future__ import annotations

import ctypes
import os
from ctypes import (c_char_p, c_double, c_float, c_int, c_int32, c_int64, c_size_t, c_uint32, c_uint64, c_ulonglong,
                    c_void_p, POINTER)

_PKG_DIR = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_PKG_DIR, "libb200reco.so")

if not os.path.exists(LIB_PATH):
    raise ImportError(
        f"{LIB_PATH} is missing: build it with `python -m librecommender_b200.build` "
        "(nvcc, sm_90a).  librecommender_b200 has no CPU fallback."
    )

lib = ctypes.CDLL(LIB_PATH)

# name -> (restype, argtypes); must list every symbol of include/b200reco.h
_P = c_void_p
SIGNATURES = {
    "b200_version": (c_int, []),
    "b200_last_error": (c_char_p, []),
    "b200_launch_count": (c_ulonglong, []),
    "b200_build_consumed_csr_host": (c_int, [_P, _P, c_int64, c_int64, _P, _P, POINTER(c_int64)]),
    "b200_mask_consumed": (c_int, [_P, c_int64, _P, c_int64, c_int64, c_int32, _P, _P, c_int64, _P]),
    "b200_topk_rows_workspace_bytes": (c_int, [c_int64, c_int64, c_int32, POINTER(c_size_t)]),
    "b200_topk_rows": (c_int, [_P, c_int64, c_int64, c_int64, c_int32, _P, _P, _P, c_size_t, _P]),
    "b200_score_rows_f32": (c_int, [_P, c_int64, _P, c_int64, _P, c_int64, c_int64, c_int32, _P, c_int64, _P]),
    "b200_embed_catalog_bytes": (c_int, [c_int64, c_int32, POINTER(c_size_t)]),
    "b200_embed_catalog_prepare": (c_int, [_P, c_int64, c_int64, c_int32, _P, c_size_t, _P]),
    "b200_recommend_embed_tune": (c_int, [c_int32, c_float]),
    "b200_recommend_embed_speculation": (c_int, [c_int32, c_float]),
    "b200_recommend_embed_debug": (c_int, [c_int32]),
    "b200_recommend_embed_plan": (c_int, [c_int64, c_int64, c_int32, c_int32, _P, c_int32]),
    "b200_recommend_embed_workspace_bytes": (c_int, [c_int64, c_int64, c_int32, c_int32, POINTER(c_size_t)]),
    "b200_recommend_embed": (c_int, [_P, c_int64, _P, c_int64, _P, c_int64, c_int64, c_int32, _P, _P, _P,
                                     c_int64, c_int32, c_int32, _P, _P, _P, _P, c_size_t, _P, _P, _P, _P]),
    "b200_spmm_long_row_threshold": (c_int, []),
    "b200_spmm_chunk": (c_int, []),
    "b200_spmm_csr": (c_int, [_P, _P, _P, c_int64, _P, c_int64, c_int32, _P, c_int64, _P, c_int64, c_int32,
                              c_float, _P, _P, c_int64, _P, _P, c_int64, _P, _P]),
    "b200_als_long_row_threshold": (c_int, []),
    "b200_als_chunk": (c_int, []),
    "b200_als_stage_rows": (c_int, [c_int32]),
    "b200_als_workspace_bytes": (c_int, [c_int32, c_int32, c_int64, c_int64, POINTER(c_size_t)]),
    "b200_als_cg": (c_int, [_P, _P, _P, c_int64, _P, _P, c_int64, c_int32, _P, c_int32, c_int32, _P, c_int64, _P, _P,
                            c_int64, _P, _P, c_int64, _P, c_size_t, _P]),
    "b200_als_direct": (c_int, [_P, _P, _P, c_int64, _P, _P, c_int64, c_int32, _P, c_int32, _P, c_int64, _P, _P,
                                c_int64, _P, _P, c_int64, _P, c_size_t, POINTER(c_int64), POINTER(c_int32), _P]),
    "b200_bpr_default_inflight": (c_int64, [c_int32]),
    "b200_bpr_update": (c_int, [c_int32, _P, _P, c_int64, _P, _P, c_int64, c_int64, _P, _P, c_int32, _P, _P, _P, _P,
                                c_float, c_float, c_float, c_float, c_float, c_int32, c_uint64, _P, _P, c_int64, _P]),
    "b200_skipgram_default_inflight": (c_int64, [c_int32]),
    "b200_skipgram_subsample": (c_int, [_P, _P, c_int64, c_int64, _P, c_uint64, c_int64, _P, _P, _P, _P, _P]),
    "b200_skipgram_epoch": (c_int, [_P, c_int64, _P, _P, _P, c_int64, c_int64, _P, _P, _P, c_int32, c_int32, _P, _P,
                                    _P, _P, _P, c_int64, c_uint32, _P, c_int64, c_int32, c_int32, c_double, c_double,
                                    c_double, c_double, c_uint64, c_int64, _P, _P, c_int64, _P]),
    "b200_item_walks": (c_int, [_P, _P, c_int64, c_int32, c_int32, c_uint64, c_int64, _P, _P, _P, _P]),
    "b200_sage_neighbors": (c_int, [_P, _P, _P, _P, _P, _P, c_int64, c_int64, c_int32, c_int32, c_uint64, _P, _P]),
    "b200_pinsage_neighbors": (c_int, [_P, _P, _P, _P, _P, _P, c_int64, c_int64, c_int32, c_int32, c_int32, c_int32,
                                       c_uint64, c_uint64, _P, _P, _P, _P]),
    "b200_sage_aggregate": (c_int, [_P, c_int64, _P, c_int64, _P, c_int64, _P, _P, _P, c_int32, _P, c_int32, _P,
                                    c_int64, _P]),
    "b200_sage_aggregate_backward": (c_int, [_P, c_int64, _P, c_int64, _P, c_int64, _P, _P, _P, c_int32, c_int32, _P,
                                             c_int64, _P]),
    "b200_sage_walk_pairs": (c_int, [_P, _P, _P, _P, c_int64, c_int64, c_int32, c_int32, c_int32, c_uint64, c_uint64,
                                     _P, _P, _P, _P, _P, _P]),
    "b200_sage_i2i_negatives": (c_int, [_P, _P, c_int64, c_int32, c_int64, c_int32, c_uint64, c_uint64, _P, _P]),
    "b200_swing_scores_workspace_bytes": (c_int, [c_int64, c_int64, c_int32, POINTER(c_size_t)]),
    "b200_swing_scores": (c_int, [_P, _P, c_int64, _P, _P, c_int64, c_float, c_int32, _P, _P, _P, _P, c_size_t, _P]),
    "b200_swing_plan": (c_int, [c_int64, c_int32, POINTER(c_int32), POINTER(c_int32)]),
    "b200_swing_recommend": (c_int, [_P, _P, _P, c_int64, _P, _P, _P, c_int64, c_int32, _P, _P, c_int32, _P, c_int64,
                                     _P, c_int64, _P, _P]),
    "b200_swing_random_keys": (c_int, [_P, c_int64, c_int64, c_int64, _P, _P, c_int32, c_uint64, _P]),
    "b200_swing_predict": (c_int, [_P, _P, c_int64, _P, _P, _P, c_int64, c_int32, _P, _P, c_int64, c_float, _P, _P]),
    "b200_cf_cosine_workspace_bytes": (c_int, [c_int64, c_int32, POINTER(c_size_t)]),
    "b200_cf_plan": (c_int, [c_int64, c_int32, POINTER(c_int32), POINTER(c_int32)]),
    "b200_cf_cosine": (c_int, [_P, _P, _P, c_int64, _P, _P, _P, c_int64, c_int64, c_int32, _P, _P, _P, _P, c_size_t,
                               _P]),
    "b200_user_cf_recommend": (c_int, [_P, _P, _P, c_int64, _P, _P, _P, c_int64, c_int32, _P, _P, c_int32, _P,
                                       c_int64, _P, c_int64, _P, _P]),
    "b200_cf_predict": (c_int, [_P, _P, _P, c_int64, _P, _P, _P, c_int64, c_int32, _P, _P, c_int64, c_int32, c_float,
                                _P, _P]),
    "b200_feat_forward_tune": (c_int, [c_int32]),
    "b200_feat_forward": (c_int, [_P, _P, _P, _P, c_int64, c_int64, c_int64, _P, c_int64, _P, c_int64, _P, _P, _P, c_float,
                                  _P, _P, _P, c_float, _P, _P, c_int64, _P]),
    "b200_fm_pair_scores": (c_int, [_P, _P, _P, c_int64, _P, _P, _P, c_int64, c_int32, c_float, _P, _P, _P, c_float,
                                    _P, c_int64, _P]),
    "b200_deepfm_pair_scores": (c_int, [_P, _P, _P, _P, c_int64, _P, _P, _P, _P, c_int64, c_int32, c_int32, c_int32,
                                        c_int32, c_float, _P, _P, _P, _P, _P, c_float, _P, c_int64, _P]),
    "b200_multi_sparse_combine": (c_int, [_P, c_int64, c_int32, _P, c_int64, c_int32, c_int64, c_int32, c_int32, _P,
                                          c_int64, _P]),
    "b200_gather_rows": (c_int, [_P, c_int64, c_int32, _P, c_int64, _P, c_int64, _P]),
    "b200_peer_gather_rows": (c_int, [_P, c_int32, c_int64, c_int32, _P, c_int64, _P, c_int64, _P]),
    "b200_peer_scatter_add_rows": (c_int, [_P, c_int32, c_int64, c_int32, _P, c_int64, _P, c_int64, _P]),
    "b200_scatter_add_rows": (c_int, [_P, c_int64, c_int32, _P, c_int64, _P, c_int64, _P]),
    "b200_linear_f32": (c_int, [_P, c_int64, c_int64, _P, c_int64, _P, c_int32, c_int32, c_int32, _P, c_int64, _P]),
    "b200_linear_tf32x3_split_ld": (c_int64, [c_int32]),
    "b200_linear_tf32x3_split_weights": (c_int, [_P, c_int64, c_int32, c_int32, _P, _P]),
    "b200_linear_tf32x3": (c_int, [_P, c_int64, c_int64, _P, c_int64, _P, _P, c_int32, c_int32, c_int32, _P, c_int64,
                                   _P]),
    "b200_linear_tf32x3_splitk": (c_int, [_P, c_int64, c_int64, _P, c_int64, _P, c_int32, c_int32, c_int32, c_int32, _P,
                                          c_size_t, _P, c_int64, _P]),
    "b200_bn_train_forward": (c_int, [_P, c_int64, c_int64, c_int32, _P, _P, c_float, c_float, _P, c_int64, _P, _P, _P,
                                      _P, _P]),
    "b200_fm_head_forward": (c_int, [_P, c_int64, c_int64, c_int32, _P, _P, _P, _P, _P, _P, _P]),
    "b200_fm_head_backward_workspace_bytes": (c_size_t, [c_int64, c_int32]),
    "b200_fm_head_backward": (c_int, [_P, _P, _P, c_int64, c_int64, c_int32, _P, _P, _P, _P, c_float, _P, _P, c_int64,
                                      _P, _P, _P, _P, _P, _P, c_size_t, _P]),
    "b200_feat_backward": (c_int, [_P, _P, _P, _P, c_int64, _P, c_int64, _P, c_int64, _P, c_int64, _P, _P, _P, _P, _P,
                                   _P, _P, _P, _P, _P, _P, _P]),
    "b200_col_reduce": (c_int, [_P, c_int64, c_int64, c_int32, _P, _P, c_int64, _P, _P]),
    "b200_bn_train_backward": (c_int, [_P, c_int64, _P, c_int64, c_int64, c_int32, _P, _P, _P, c_float, c_int32, _P,
                                       c_int64, _P, _P, _P, c_size_t, _P]),
    "b200_relu_backward": (c_int, [_P, _P, c_int64, _P, _P]),
    "b200_deepfm_head_forward": (c_int, [_P, _P, _P, c_int64, c_int32, _P, c_int64, c_int32, _P, _P, c_int64, _P, _P]),
    "b200_deepfm_head_backward": (c_int, [_P, _P, c_int32, c_int32, c_int64, _P, _P, c_int64, _P, c_int64, _P]),
    "b200_adam_dense": (c_int, [_P, _P, _P, _P, c_int64, c_float, c_float, c_float, c_float, c_int64, _P]),
    "b200_adam_begin_step": (c_int, [_P, c_float, c_float, c_float, c_float, c_int64, _P, _P]),
    "b200_axpy": (c_int, [_P, _P, c_float, c_int64, _P]),
    "b200_adam_dense_dev": (c_int, [_P, _P, _P, _P, c_int64, _P, c_float, c_float, c_float, _P]),
    "b200_loss_workspace_bytes": (c_size_t, []),
    "b200_pointwise_loss": (c_int, [_P, _P, c_int64, c_int32, c_float, c_float, _P, _P, _P, c_size_t, _P]),
    "b200_pairwise_loss": (c_int, [_P, c_int64, _P, c_int64, c_int32, c_float, c_float, c_float, c_int32, _P, _P, _P,
                                   _P, c_size_t, _P]),
    "b200_softmax_inbatch_loss": (c_int, [_P, c_int64, c_int32, c_float, _P, _P, c_int32, _P, _P, c_size_t, _P]),
    "b200_sampled_class_loss_workspace_bytes": (c_size_t, [c_int32, c_int32]),
    "b200_sampled_class_loss": (c_int, [c_int32, _P, c_int64, c_int32, c_int32, _P, _P, _P, _P, c_int32, c_int64, _P,
                                        _P, _P, _P, c_size_t, _P]),
    "b200_unique_candidates_workspace_bytes": (c_size_t, [c_int64]),
    "b200_unique_candidates": (c_int, [c_int32, c_int64, c_int32, c_uint64, _P, _P, c_size_t, _P, _P, _P]),
    "b200_concat_dense": (c_int, [_P, c_int64, c_int32, _P, c_int64, c_int32, _P, c_int64, c_int32, _P, c_float,
                                  c_int64, _P, _P]),
    "b200_l2_normalize_rows": (c_int, [_P, c_int64, c_int64, c_int32, _P]),
    "b200_l2_normalize_backward": (c_int, [_P, c_int64, _P, c_int64, c_int64, c_int32, _P, c_int64, _P]),
    "b200_seq_pool": (c_int, [_P, c_int64, c_int32, c_int64, _P, c_int64, _P, c_int32, _P, c_int64, c_int64, c_int64,
                              _P, c_int64, _P]),
    "b200_seq_pool_backward": (c_int, [_P, c_int64, c_int32, c_int64, _P, c_int64, _P, c_int32, _P, c_int64, _P, c_int64,
                                       _P]),
    "b200_din_attention_tune": (c_int, [c_int32]),
    "b200_din_attention_backward": (c_int, [_P, c_int64, c_int32, _P, _P, c_int64, _P, c_int32, _P, c_int64, _P, _P, _P,
                                            c_float, _P, c_int64, _P, c_int64, _P, _P, _P, _P, _P]),
    "b200_din_attention": (c_int, [_P, c_int64, c_int32, _P, _P, c_int64, _P, c_int32, _P, c_int64, c_int64, c_int64,
                                   _P, _P, _P, c_float, _P, c_int64, _P]),
    "b200_mul_elementwise": (c_int, [_P, _P, c_int64, _P, _P]),
    "b200_ngcf_combine": (c_int, [_P, c_int64, _P, c_int64, c_int64, c_int32, c_float, _P, c_int64, _P]),
    "b200_din_user_weights": (c_int, [_P, c_int64, c_int32, _P, c_int32, _P, _P, _P, c_int64, _P, _P]),
    "b200_linear_tf32x3_sigmoid_dot": (c_int, [_P, c_int64, c_int64, _P, c_int64, _P, _P, c_int32, c_int32, _P, _P, c_int64,
                                               _P]),
    "b200_din_attention_from_logits": (c_int, [_P, c_int64, c_int64, _P, c_int64, c_int32, _P, c_int32, c_float, _P,
                                               c_int64, _P]),
    "b200_din_attention_hoisted": (c_int, [_P, c_int64, c_int64, _P, c_int64, c_int32, _P, c_int32, _P, c_float, _P,
                                           c_int64, _P]),
    "b200_sample_negatives": (c_int, [_P, _P, c_int64, c_int32, c_int64, c_int32, c_int32, c_uint64, c_uint64,
                                      _P, _P, c_int64, _P, _P, _P]),
    "b200_interacted_seqs": (c_int, [_P, _P, c_int64, _P, _P, c_int64, c_int32, c_int32, _P, c_uint64, c_uint64,
                                     _P, _P, _P]),
    "b200_interacted_dual_seqs": (c_int, [_P, _P, c_int64, _P, _P, c_int64, c_int32, c_int32, c_int32, _P, c_uint64,
                                          c_uint64, _P, _P, _P, _P, _P]),
    "b200_gather_dot": (c_int, [_P, c_int64, _P, _P, c_int64, _P, c_int64, c_int32, c_int32, c_float, c_float, _P, _P]),
    "b200_autoint_rows": (c_int, [_P, c_int64, c_int64, c_int32, c_int32, c_int32, c_int32, _P, _P, _P, c_float, c_int32,
                                  _P, _P]),
    "b200_autoint_grid": (c_int, [_P, c_int64, c_int64, _P, c_int64, c_int64, _P, c_int32, c_int32, c_int32, c_int32, _P,
                                  _P, _P, c_float, c_int32, _P, c_int64, _P]),
    "b200_transformer_encode": (c_int, [_P, c_int64, _P, _P, c_int64, _P, c_int64, c_int32, _P, c_int32, c_int32,
                                        c_int32, c_int32, c_int32, _P, _P, _P, _P]),
    "b200_transformer_pair_smem_bytes": (c_int64, [c_int32, c_int32, c_int32]),
    "b200_transformer_pair_scores": (c_int, [_P, c_int64, c_int64, _P, _P, _P, _P, c_int64, _P, c_int64, c_int32,
                                             c_int32, c_int32, c_int32, c_int32, _P, _P, _P, _P, _P, c_float, _P,
                                             c_int64, _P]),
    "b200_transformer_target_attention": (c_int, [_P, c_int64, _P, c_int32, c_int32, _P, _P, _P, c_int64, c_int64,
                                                  c_int64, _P, c_int64, _P]),
    "b200_sim_attention": (c_int, [_P, c_int64, _P, c_int64, c_int32, c_int32, _P, c_int64, _P, _P, _P, c_int32, _P,
                                   c_int64, _P, c_int32, c_int32, _P, _P, _P, c_int64, c_int64, c_int64, _P, c_int64,
                                   _P, _P]),
    "b200_sim_pair_smem_bytes": (c_int64, [c_int32] * 7),
    "b200_sim_pair_scores": (c_int, [_P, _P, c_int64, c_int64, _P, c_int64, _P, c_int64, _P, _P, c_int64, _P, _P, _P,
                                     _P, c_int64, _P, c_int64, c_int32, c_int32, c_int32, c_int32, c_int32, c_int32,
                                     c_int32, c_int32, _P, _P, _P, _P, _P, _P, c_float, _P, c_int64, _P]),
    "b200_sim_gsu_forward": (c_int, [_P, c_int64, c_int32, _P, _P, c_int64, _P, c_int32, c_int32, c_int64, _P, _P,
                                     c_int64, _P]),
    "b200_sim_esu_forward": (c_int, [_P, c_int64, _P, _P, c_int64, _P, _P, c_int64, c_int32, c_int32, c_int32, _P,
                                     c_int64, _P, _P]),
    "b200_sim_esu_backward": (c_int, [_P, c_int64, _P, _P, c_int64, _P, _P, c_int64, c_int32, c_int32, c_int32, _P,
                                      _P, c_int64, _P, c_int64, _P, _P, c_int64, _P]),
    "b200_sim_long_backward": (c_int, [_P, c_int64, _P, c_int32, _P, c_int32, c_int64, c_int32, _P, c_int64, _P,
                                       c_int64, _P, c_int64, _P]),
    "b200_autoint_attention_forward":(c_int, [_P, c_int64, _P, c_int64, _P, c_int64, c_int64, c_int32, c_int32,
                                               c_int32, c_float, _P, c_int64, _P, _P]),
    "b200_autoint_attention_backward": (c_int, [_P, c_int64, _P, c_int64, _P, c_int64, _P, c_int64, _P, _P, c_int64,
                                                c_int64, c_int32, c_int32, c_int32, c_float, _P, _P, _P, c_int64, _P]),
    "b200_transformer_attention_forward": (c_int, [_P, c_int64, _P, c_int64, _P, c_int64, _P, c_int64, c_int32,
                                                   c_int32, c_int32, c_int32, c_float, _P, c_int64, _P, _P]),
    "b200_transformer_attention_backward": (c_int, [_P, c_int64, _P, c_int64, _P, c_int64, _P, c_int64, _P, _P,
                                                    c_int64, _P, c_int64, c_int32, c_int32, c_int32, c_int32, c_float,
                                                    _P, _P, _P, c_int64, _P]),
    "b200_rms_norm_forward": (c_int, [_P, c_int64, c_int64, c_int32, _P, _P, c_int64, _P, _P]),
    "b200_rms_norm_backward": (c_int, [_P, c_int64, _P, c_int64, _P, c_int64, c_int32, _P, _P, c_int64, _P]),
    "b200_activation_forward": (c_int, [_P, c_int64, c_int32, _P, _P]),
    "b200_activation_backward": (c_int, [_P, _P, c_int64, c_int32, _P, _P]),
    "b200_transformer_target_attention_backward": (c_int, [_P, c_int64, _P, c_int32, c_int32, _P, _P, c_int64,
                                                           c_int64, _P, c_int64, _P, _P]),
    "b200_rnn_layer_floats": (c_int64, [c_int32, c_int32, c_int32]),
    "b200_rnn_encode": (c_int, [_P, c_int64, _P, _P, c_int64, c_int32, _P, c_int64, c_int32, c_int32, _P, _P, _P, _P,
                                _P, c_int64, _P]),
    "b200_rnn_train_forward": (c_int, [_P, c_int64, _P, _P, c_int64, c_int32, _P, c_int64, c_int32, c_int32, _P, _P,
                                       _P, _P, _P, c_int64, _P, _P]),
    "b200_rnn_backward": (c_int, [_P, c_int64, _P, c_int32, c_int32, c_int32, c_int32, c_int32, _P, _P, c_int64, _P,
                                  _P, _P, _P, _P, _P, _P]),
    "b200_caser_weight_floats": (c_int64, [c_int32, c_int32, c_int32, c_int32]),
    "b200_wavenet_weight_floats": (c_int64, [c_int32, c_int32, c_int32]),
    "b200_caser_encode": (c_int, [_P, c_int64, _P, c_int64, c_int32, _P, c_int64, c_int32, c_int32, c_int32, _P, _P,
                                  c_int64, _P]),
    "b200_wavenet_encode": (c_int, [_P, c_int64, _P, c_int64, c_int32, _P, c_int64, c_int32, c_int32, c_int32, _P, _P,
                                    _P, c_int64, _P]),
    "b200_caser_train_forward": (c_int, [_P, c_int64, _P, c_int64, c_int32, _P, c_int64, c_int32, c_int32, c_int32, _P,
                                         _P, c_int64, _P, _P]),
    "b200_wavenet_train_forward": (c_int, [_P, c_int64, _P, c_int64, c_int32, _P, c_int64, c_int32, c_int32, c_int32,
                                           _P, _P, _P, c_int64, _P, _P, _P]),
    "b200_caser_backward_workspace_floats": (c_int64, [c_int64, c_int32, c_int32, c_int32, c_int32]),
    "b200_caser_backward": (c_int, [c_int64, c_int32, c_int32, c_int32, c_int32, _P, c_int64, _P, c_int64, _P, _P,
                                    c_int64, _P, _P, c_int64, _P, _P, c_int64, _P]),
    "b200_wavenet_pool_backward": (c_int, [c_int64, c_int32, c_int32, _P, c_int64, _P, _P, _P]),
    "b200_wavenet_layer_inputs": (c_int, [_P, c_int64, c_int64, c_int32, c_int32, c_int32, _P, _P]),
    "b200_wavenet_layer_dx": (c_int, [_P, c_int64, c_int32, c_int32, c_int32, _P, c_int64, _P]),
}

for _name, (_res, _args) in SIGNATURES.items():
    _fn = getattr(lib, _name)  # AttributeError here == header/library mismatch
    _fn.restype = _res
    _fn.argtypes = _args


# float32 bit pattern, as an int32, of a REMOVED score (a consumed item, an empty candidate slot): the NaN 0xffffffff,
# which b200_topk_rows ranks below every score (csrc/common.cuh kRemovedBits).  Write it through an int32 view.
REMOVED_BITS = -1


class B200Error(RuntimeError):
    pass


def check(rc: int) -> None:
    if rc != 0:
        msg = lib.b200_last_error().decode("utf-8", "replace")
        if "exceeds num of items" in msg:
            raise ValueError(msg)
        raise B200Error(f"[b200reco rc={rc}] {msg}")


def ptr(t) -> c_void_p:
    """Raw data pointer of a torch tensor / numpy array (None -> NULL)."""
    if t is None:
        return c_void_p(0)
    if hasattr(t, "data_ptr"):
        return c_void_p(t.data_ptr())
    return c_void_p(t.ctypes.data)


def current_stream() -> c_void_p:
    import torch

    return c_void_p(torch.cuda.current_stream().cuda_stream)


def launch_count() -> int:
    return int(lib.b200_launch_count())


def require_cuda():
    import torch

    if not torch.cuda.is_available():
        raise B200Error("librecommender_b200 needs a CUDA device (sm_90a); there is no CPU fallback")
    return torch.device("cuda", torch.cuda.current_device())
