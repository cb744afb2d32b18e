"""ctypes binding of include/hnh_b200.h (the C ABI of libhnh_b200.so)."""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


class LibraryMissing(RuntimeError):
    pass


def library_path() -> str:
    return os.path.join(_HERE, "libhnh_b200.so")


# name -> (restype, argtypes); every symbol declared in include/hnh_b200.h
_P = C.c_void_p
_I64 = C.c_int64
ABI = {
    "hnh_abi_version": (C.c_int, []),
    "hnh_build_info": (C.c_char_p, []),
    "hnh_last_error_string": (C.c_char_p, []),
    "hnh_launch_count": (C.c_uint64, []),
    "hnh_sddmm_f64": (C.c_int, [_P, _P, _P, _I64, _I64, _P, _P, C.c_int, C.c_int, _P]),
    "hnh_sddmm_scaled_f64": (C.c_int, [_P, _P, _P, _I64, _I64, _P, _P, C.c_int, C.c_int, _P, _P, _P]),
    "hnh_sddmm_coo_f64": (C.c_int, [_P, _P, _P, _I64, _P, _P, C.c_int, C.c_int, _P]),
    "hnh_spmm_f64": (C.c_int, [_P, _P, _P, _I64, _I64, _P, _P, C.c_int, C.c_int, _P]),
    "hnh_fused_f64": (C.c_int, [_P, _P, _P, _I64, _I64, _P, _P, _P, C.c_int, C.c_int, _P]),
    "hnh_fused_scaled_f64": (C.c_int, [_P, _P, _P, _I64, _I64, _P, _P, _P, C.c_int, C.c_int, _P, _P, _P]),
    "hnh_fill_f64": (C.c_int, [_P, _I64, C.c_double, _P]),
    "hnh_random_uniform_f64": (C.c_int, [_P, _I64, C.c_uint64, _P]),
    "hnh_hadamard_f64": (C.c_int, [_P, _P, _P, _I64, _P]),
    "hnh_expand_row_idx": (C.c_int, [_P, _I64, _I64, _P, _P]),
    "hnh_batch_dot_f64": (C.c_int, [_P, _P, _P, _I64, C.c_int, _P]),
    "hnh_row_axpy_f64": (C.c_int, [_P, _P, C.c_double, _P, _P, _I64, C.c_int, _P]),
    "hnh_vec_quotient_f64": (C.c_int, [_P, _P, C.c_double, _P, C.c_double, _I64, _P]),
    "hnh_axpby_f64": (C.c_int, [_P, C.c_double, _P, C.c_double, _P, _I64, _P]),
    "hnh_squared_norm_f64": (C.c_int, [_P, _P, _I64, _P]),
    "hnh_leaky_relu_f64": (C.c_int, [_P, _P, _I64, C.c_double, _P]),
    "hnh_relu_cols_f64": (C.c_int, [_P, _I64, _I64, _P, _I64, _I64, _P]),
    "hnh_dgemm_f64": (C.c_int, [_P, _P, _P, _I64, _I64, _I64, _P]),
    "hnh_leaky_relu_grad_f64": (C.c_int, [_P, _P, _I64, C.c_double, _P]),
    "hnh_relu_cols_backward_f64": (C.c_int, [_P, _P, _P, _I64, _I64, _I64, _I64, _P]),
    "hnh_dgemm_tn_workspace_bytes": (C.c_int64, [_I64, _I64, _I64]),
    "hnh_dgemm_tn_f64": (C.c_int, [_P, _P, _P, _I64, _I64, _I64, _P, C.c_size_t, _P]),
    "hnh_dgemm_nt_f64": (C.c_int, [_P, _P, _P, _I64, _I64, _I64, C.c_int, _P]),
    "hnh_edge_keys_from_index": (C.c_int, [_P, _P, _I64, _I64, _P]),
    "hnh_edge_softmax_piece_bound": (C.c_int64, [_I64, _I64]),
    "hnh_edge_softmax_plan": (C.c_int, [_P, _I64, _I64, _P, _P, _P, _P, _I64, C.POINTER(C.c_int64), _P]),
    "hnh_edge_softmax_stats_f64": (C.c_int, [_P, _P, _P, _P, _P, _I64, _I64, _P, _P, _P, _P, _P]),
    "hnh_edge_softmax_rescale_f64": (C.c_int, [_P, _P, _P, _I64, _P]),
    "hnh_edge_softmax_apply_f64": (C.c_int, [_P, _P, _P, _I64, _P, _P, _P]),
    "hnh_edge_softmax_dot_f64": (C.c_int, [_P, _P, _P, _P, _P, _P, _I64, _I64, _P, _P, _P]),
    "hnh_edge_softmax_backward_f64": (C.c_int, [_P, _P, _P, _P, _I64, _P, _P]),
    "hnh_edge_sum_f64": (C.c_int, [_P, _P, _P, _P, _P, _I64, _I64, _P, _P, _P]),
    "hnh_gat_node_scalars_f64": (C.c_int, [_P, _P, _P, _P, _P, _I64, _I64, _P]),
    "hnh_gat_edge_scores_f64": (C.c_int, [_P, _P, _P, _P, _P, _I64, C.c_double, C.c_int, _P]),
    "hnh_gat_rank2_update_f64": (C.c_int, [_P, _P, _P, _P, _P, _I64, _I64, _P]),
    "hnh_gatv2_scores_f64": (C.c_int, [_P, _P, _I64, _I64, _P, _I64, _P, _I64, _P, C.c_int, C.c_double, _P, _P]),
    "hnh_gatv2_grad_workspace_bytes": (C.c_int64, [_I64, C.c_int]),
    "hnh_gatv2_grad_f64": (C.c_int, [_P, _P, _P, _I64, _I64, _P, _I64, _P, _I64, _P, C.c_int, C.c_double, _P, _I64, _P, _P,
                                     C.c_size_t, _P]),
    "hnh_sparse_attention_step_f64": (C.c_int, [_P, _P, _I64, _I64, C.c_int, _P, _I64, _P, _I64, _P, _I64, C.c_double, _P, _I64,
                                                _P, _I64, _P, _I64, _P]),
    "hnh_sparse_attention_finish_f64": (C.c_int, [_I64, C.c_int, _P, _I64, _P, _I64, _P, _I64, _P, _I64, _P, _I64, _P]),
    "hnh_sparse_attention_grad_q_f64": (C.c_int, [_P, _P, _I64, _I64, C.c_int, _P, _I64, _P, _I64, _P, _I64, _P, _I64, _P, _I64,
                                                  _P, _I64, C.c_double, _P, _I64, _P]),
    "hnh_sparse_attention_grad_kv_f64": (C.c_int, [_P, _P, _I64, _I64, C.c_int, _P, _I64, _P, _I64, _P, _I64, _P, _I64, _P, _I64,
                                                   _P, _I64, C.c_double, _P, _I64, _P, _I64, _P]),
    "hnh_sparse_attention_step_dropout_f64": (C.c_int, [_P, _P, _I64, _I64, C.c_int, _P, _I64, _P, _I64, _P, _I64, C.c_double,
                                                        _P, _I64, _P, _I64, _P, _I64, C.c_double, C.c_uint64, _I64, _I64, _P]),
    "hnh_sparse_attention_grad_q_dropout_f64": (C.c_int, [_P, _P, _I64, _I64, C.c_int, _P, _I64, _P, _I64, _P, _I64, _P, _I64,
                                                          _P, _I64, _P, _I64, C.c_double, _P, _I64, C.c_double, C.c_uint64,
                                                          _I64, _I64, _P]),
    "hnh_sparse_attention_grad_kv_dropout_f64": (C.c_int, [_P, _P, _I64, _I64, C.c_int, _P, _I64, _P, _I64, _P, _I64, _P, _I64,
                                                           _P, _I64, _P, _I64, C.c_double, _P, _I64, _P, _I64, C.c_double,
                                                           C.c_uint64, _I64, _I64, _P]),
    "hnh_sparse_attention_step_bias_f64": (C.c_int, [_P, _P, _I64, _I64, C.c_int, _P, _I64, _P, _I64, _P, _I64, C.c_double,
                                                     _P, _I64, _P, _I64, _P, _I64, C.c_double, C.c_uint64, _I64, _I64, _P,
                                                     _P]),
    "hnh_sparse_attention_grad_q_bias_f64": (C.c_int, [_P, _P, _I64, _I64, C.c_int, _P, _I64, _P, _I64, _P, _I64, _P, _I64,
                                                       _P, _I64, _P, _I64, C.c_double, _P, _I64, C.c_double, C.c_uint64,
                                                       _I64, _I64, _P, _P, _P]),
    "hnh_sparse_attention_grad_kv_bias_f64": (C.c_int, [_P, _P, _I64, _I64, C.c_int, _P, _I64, _P, _I64, _P, _I64, _P, _I64,
                                                        _P, _I64, _P, _I64, C.c_double, _P, _I64, _P, _I64, C.c_double,
                                                        C.c_uint64, _I64, _I64, _P, _P, _P]),
    "hnh_sparse_attention_step_edge_f64": (C.c_int, [_P, _P, _I64, _I64, C.c_int, _P, _I64, _P, _I64, _P, _I64, C.c_double,
                                                     _P, _I64, _P, _I64, _P, _I64, C.c_double, C.c_uint64, _I64, _I64, _P,
                                                     _P, _I64, _P]),
    "hnh_sparse_attention_grad_q_edge_f64": (C.c_int, [_P, _P, _I64, _I64, C.c_int, _P, _I64, _P, _I64, _P, _I64, _P, _I64,
                                                       _P, _I64, _P, _I64, C.c_double, _P, _I64, C.c_double, C.c_uint64,
                                                       _I64, _I64, _P, _P, _P, _I64, _P, _I64, _P]),
    "hnh_sparse_attention_grad_kv_edge_f64": (C.c_int, [_P, _P, _I64, _I64, C.c_int, _P, _I64, _P, _I64, _P, _I64, _P, _I64,
                                                        _P, _I64, _P, _I64, C.c_double, _P, _I64, _P, _I64, C.c_double,
                                                        C.c_uint64, _I64, _I64, _P, _P, _P, _I64, _P]),
    "hnh_row_bias_add_f64": (C.c_int, [_P, _P, _I64, _I64, _P]),
    "hnh_gt_gate_f64": (C.c_int, [_P, _P, _P, _P, _I64, _I64, C.c_int, _P]),
    "hnh_gt_gate_backward_workspace_bytes": (C.c_int64, [_I64, _I64]),
    "hnh_gt_gate_backward_f64": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _I64, _I64, C.c_int, _P, C.c_size_t, _P]),
    "hnh_row_bias_relu_f64": (C.c_int, [_P, _P, _P, _I64, _I64, _P]),
    "hnh_layer_norm_f64": (C.c_int, [_P, _P, _P, _P, _P, _P, _I64, _I64, C.c_double, _P]),
    "hnh_layer_norm_backward_workspace_bytes": (C.c_int64, [_I64, _I64]),
    "hnh_layer_norm_backward_f64": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _I64, _I64, C.c_int, _P, C.c_size_t, _P]),
    "hnh_cross_entropy_workspace_bytes": (C.c_int64, [_I64]),
    "hnh_cross_entropy_f64": (C.c_int, [_P, _P, _P, _P, _I64, _I64, _I64, C.c_double, _P, C.c_size_t, _P]),
    "hnh_adamw_f64": (C.c_int, [_P, _P, _P, _P, _I64, C.c_double, C.c_double, C.c_double, C.c_double, C.c_double,
                                C.c_double, C.c_double, _P, _P]),
    "hnh_clip_coef_f64": (C.c_int, [_P, _P, _I64, C.c_double, _P]),
    "hnh_pair_sums_workspace_bytes": (C.c_int64, [_I64]),
    "hnh_pair_sums_f64": (C.c_int, [_P, _P, _I64, _P, C.c_size_t, _P]),
    "hnh_link_bce_f64": (C.c_int, [_P, _P, _P, _I64, _I64, _P, _I64, _P, _I64, C.c_int, C.c_double, _P, _I64, _P, _I64, _P, _P]),
    "hnh_link_target_check_f64": (C.c_int, [_P, _P, _I64, _P]),
    "hnh_distmult_bce_f64": (C.c_int, [_P, _P, _P, _I64, _I64, C.c_int, _P, _I64, _P, _I64, _P, _I64, C.c_int, C.c_double,
                                       C.c_double, _P, _I64, _P, _I64, _P, _P, _P]),
    "hnh_distmult_bce_grad_f64": (C.c_int, [_P, _P, _P, _I64, _I64, C.c_int, _P, _I64, _P, _I64, _P, _I64, C.c_int, C.c_double,
                                            C.c_double, _P, _I64, _P]),
    "hnh_distmult_relation_grad_f64": (C.c_int, [_P, _P, _P, _P, _I64, C.c_int, _P, _P, _P, _P, _I64, _P, _I64, C.c_int, _P, _P,
                                                 _I64, _P]),
    "hnh_rank_count_f64": (C.c_int, [_P, _I64, _I64, _P, _I64, _I64, C.c_int, _P, _P, _P, _P]),
    "hnh_rank_queries_f64": (C.c_int, [_P, _I64, _I64, _P, _I64, _I64, _I64, _P, _P, _P, _I64, C.c_int, C.c_int, _P]),
    "hnh_rank_pairs_f64": (C.c_int, [_P, _I64, _I64, _P, _I64, _I64, C.c_int, _P, _P, _I64, _P, _P, _P, _P, _P]),
    "hnh_entry_coords_from_index_f64":(C.c_int, [_P, _P, _I64, _I64, _P]),
    "hnh_max_aggregate_step_f64": (C.c_int, [_P, _P, _I64, _I64, _P, _I64, C.c_int, _P, _I64, _P, _I64, _P]),
    "hnh_max_aggregate_finish_f64": (C.c_int, [_P, _P, _I64, _P]),
    "hnh_max_aggregate_grad_scale_f64": (C.c_int, [_P, _P, _P, _I64, _P]),
    "hnh_max_aggregate_grad_f64": (C.c_int, [_P, _P, _I64, _I64, _P, _I64, _P, _I64, _P, _I64, C.c_int, _P, _I64, _P]),
    "hnh_segment_pool_workspace_bytes": (C.c_int64, [_I64, C.c_int, C.c_int]),
    "hnh_segment_pool_f64": (C.c_int, [_P, _P, _P, _P, _I64, _I64, _P, _I64, C.c_int, _P, _I64, _P, _I64, _P, C.c_size_t, _P]),
    "hnh_segment_max_count_merge_f64": (C.c_int, [_P, _P, _P, _I64, _P]),
    "hnh_segment_pool_grad_f64": (C.c_int, [_P, _I64, _I64, _P, _I64, _P, _P, _I64, _P, _I64, _P, _I64, C.c_int, _P, _I64, _P]),
    "hnh_multi_aggregate_step_f64": (C.c_int, [_P, _P, _I64, _I64, _P, _I64, C.c_int, C.c_int, _P, _I64, _P]),
    "hnh_multi_aggregate_finish_f64": (C.c_int, [_P, _I64, _I64, C.c_int, C.c_int, _P]),
    "hnh_multi_aggregate_grad_prep_f64": (C.c_int, [_P, _I64, _P, _I64, _I64, C.c_int, C.c_int, _P, _I64, _P]),
    "hnh_multi_aggregate_grad_f64": (C.c_int, [_P, _P, _I64, _I64, _P, _I64, _P, _I64, C.c_int, C.c_int, _P, _I64, _P]),
    "hnh_pna_combine_f64": (C.c_int, [_P, _I64, _P, _I64, _P, _I64, C.c_int, _P, _I64, _I64, C.c_int, C.c_uint, C.c_int, C.c_uint,
                                      C.c_int, C.c_double, C.c_double, _P, _I64, _P]),
    "hnh_pna_combine_grad_f64": (C.c_int, [_P, _I64, _P, _I64, C.c_int, _P, _I64, _I64, C.c_int, C.c_uint, C.c_int, C.c_uint,
                                           C.c_int, C.c_double, C.c_double, _P, _I64, _P, _I64, _P]),
    "hnh_edge_relu_aggregate_step_f64": (C.c_int, [_P, _P, _I64, _I64, _P, _I64, _P, _I64, C.c_int, _P, _I64, _P]),
    "hnh_edge_relu_aggregate_grad_f64": (C.c_int, [_P, _P, _I64, _I64, _P, _I64, _P, _I64, _P, _I64, C.c_int, _P, _I64, _P]),
    "hnh_edge_relu_aggregate_edge_grad_f64": (C.c_int, [_P, _P, _I64, _I64, _P, _I64, _P, _I64, _P, _I64, C.c_int, _P, _I64, _P]),
    "hnh_gin_combine_f64": (C.c_int, [_P, _P, _P, _P, _I64, _P]),
    "hnh_gin_combine_grad_f64": (C.c_int, [_P, _P, _P, _P, _P, _I64, _P]),
    "hnh_relational_aggregate_f64": (C.c_int, [_P, _P, _P, _I64, _I64, _P, _I64, C.c_int, C.c_int, _P, _I64, _P]),
    "hnh_relational_aggregate_grad_f64": (C.c_int, [_P, _P, _P, _I64, _I64, _P, _I64, C.c_int, C.c_int, _P, _I64, _P]),
    "hnh_window_scale_f64": (C.c_int, [_P, _I64, _P, _I64, _I64, C.c_int, C.c_int, _P]),
    "hnh_relation_check_f64": (C.c_int, [_P, _P, _I64, C.c_int, _P]),
    "hnh_basis_aggregate_f64": (C.c_int, [_P, _P, _P, _I64, _I64, _P, _I64, C.c_int, _P, _I64, _P, C.c_int, C.c_int, _P, _I64,
                                          _P]),
    "hnh_basis_aggregate_grad_f64": (C.c_int, [_P, _P, _P, _I64, _I64, _P, _I64, _P, _I64, _P, C.c_int, C.c_int, _P, _I64,
                                               C.c_int, _P, _I64, _P, _I64, _P]),
    "hnh_relation_keys": (C.c_int, [_P, _P, _I64, C.c_int, _P]),
    "hnh_block_create_host": (C.c_int, [_P, _P, _I64, _I64, _I64, C.c_int, C.POINTER(_P)]),
    "hnh_block_destroy": (None, [_P]),
    "hnh_block_run_host": (C.c_int, [_P, C.c_int, _P, _P, _P, _P, C.c_int, C.c_int, _P]),
    "hnh_er_generate_host": (C.c_int64, [C.c_int, C.c_int, C.c_uint64, _I64, _I64, _P, _P, _P, _I64]),
    "hnh_coo_to_csr_host": (C.c_int, [_I64, _I64, _I64, _P, _P, _P, C.c_int, _P, _P, _P, _P]),
    "hnh_sddmm_coo_host": (C.c_int, [_P, _P, _P, _I64, _P, _I64, _P, _I64, C.c_int]),
    "hnh_spmm_host": (C.c_int, [_P, _P, _P, _I64, _I64, _P, _I64, _P, C.c_int]),
    "hnh_er_generate_device": (C.c_int64, [C.c_int, C.c_int, C.c_uint64, _I64, _I64, _P, _P, _P, _I64, _P]),
    "hnh_coo_to_csr_device": (C.c_int, [_I64, _I64, _I64, _P, _P, _P, C.c_int, _P, _P, _P, _P, _P]),
    "hnh_tuples_bucket_by_owner_device": (C.c_int, [_P, _P, _P, _I64, C.c_int, _I64, _I64, _P, _I64, _I64, C.c_int, _P, _P, _P, _P, _P]),
    "hnh_tuples_sort_colmajor_device": (C.c_int, [_P, _P, _P, _I64, C.c_uint64, C.c_uint64, _P]),
    "hnh_tuples_mod_device": (C.c_int, [_P, _P, _I64, C.c_uint64, C.c_uint64, _P]),
    "hnh_tuples_block_starts_device": (C.c_int, [_P, _I64, C.c_uint64, C.c_int, _P, _P]),
}


def _preload_bundled_nccl():
    """libhnh_b200.so needs `libnccl.so.2`.  When PyTorch shares the process it brings its own, newer
    NCCL under the same soname; whichever copy is mapped first serves both.  Map PyTorch's copy first
    (when there is one) so that a later `import torch` still finds every symbol it was built against."""
    import sys
    for base in sys.path:
        cand = os.path.join(base, "nvidia", "nccl", "lib", "libnccl.so.2")
        if os.path.exists(cand):
            try:
                C.CDLL(cand, mode=C.RTLD_GLOBAL)
            except OSError:
                pass
            return


def lib():
    """Load libhnh_b200.so (built in-tree by build.py).  Raises LibraryMissing loudly when it
    has not been built -- the product has no fallback path."""
    global _LIB
    if _LIB is None:
        path = library_path()
        if not os.path.exists(path):
            raise LibraryMissing(
                f"{path} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'`"
                " (nvcc, sm_90a).  distributed_sddmm_b200 has no CPU fallback.")
        _preload_bundled_nccl()
        L = C.CDLL(path)
        for name, (res, args) in ABI.items():
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _LIB = L
    return _LIB


def check(rc: int, what: str = "hnh call") -> None:
    if rc != 0:
        msg = lib().hnh_last_error_string().decode()
        raise RuntimeError(f"{what} failed with code {rc}: {msg}")


# ---- driver ABI (include/hnh_b200_driver.h) --------------------------------------------------
class AlgDims(C.Structure):
    _fields_ = [("M", C.c_int64), ("N", C.c_int64), ("R", C.c_int64), ("p", C.c_int), ("c", C.c_int),
                ("localArows", C.c_int), ("localAcols", C.c_int), ("localBrows", C.c_int),
                ("localBcols", C.c_int), ("s_values", C.c_int64), ("st_values", C.c_int64),
                ("r_split", C.c_int), ("grid_i", C.c_int), ("grid_j", C.c_int), ("grid_k", C.c_int),
                ("n_a_submatrices", C.c_int), ("n_b_submatrices", C.c_int)]


_SZ = C.c_size_t
_PSZ = C.POINTER(C.c_size_t)
CB_SENDRECV = C.CFUNCTYPE(C.c_int, _P, C.c_int, _P, _SZ, C.c_int, _P, _SZ, C.c_int)
CB_ALLGATHER = C.CFUNCTYPE(C.c_int, _P, C.c_int, _P, _P, _SZ)
CB_REDUCE_SCATTER = C.CFUNCTYPE(C.c_int, _P, C.c_int, _P, _P, _SZ)
CB_ALLREDUCE = C.CFUNCTYPE(C.c_int, _P, C.c_int, _P, _SZ)
CB_ALLTOALLV = C.CFUNCTYPE(C.c_int, _P, C.c_int, _P, _PSZ, _PSZ, _P, _PSZ, _PSZ)
CB_BARRIER = C.CFUNCTYPE(C.c_int, _P, C.c_int)
CB_SPLIT = C.CFUNCTYPE(C.c_int, _P, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int),
                       C.POINTER(C.c_int))


class ExternalTransport(C.Structure):
    _fields_ = [("ctx", _P), ("sendrecv", CB_SENDRECV), ("allgather", CB_ALLGATHER),
                ("reduce_scatter_f64", CB_REDUCE_SCATTER), ("allreduce_f64", CB_ALLREDUCE),
                ("alltoallv", CB_ALLTOALLV), ("barrier", CB_BARRIER), ("split", CB_SPLIT)]


_PP = C.POINTER(_P)
ABI.update({
    "hnhd_init_self": (C.c_int, []),
    "hnhd_nccl_unique_id": (C.c_int, [C.c_char_p]),
    "hnhd_init_nccl": (C.c_int, [C.c_int, C.c_int, C.c_char_p]),
    "hnhd_init_external": (C.c_int, [C.c_int, C.c_int, C.POINTER(ExternalTransport)]),
    "hnhd_finalize": (C.c_int, []),
    "hnhd_world_rank": (C.c_int, []),
    "hnhd_world_size": (C.c_int, []),
    "hnhd_barrier": (C.c_int, []),
    "hnhd_device_synchronize": (C.c_int, []),
    "hnhd_spmat_load_er": (C.c_int, [C.c_int, C.c_int, C.c_uint64, _PP]),
    "hnhd_spmat_load_file": (C.c_int, [C.c_char_p, _PP]),
    "hnhd_spmat_from_tuples": (C.c_int, [C.c_uint64, C.c_uint64, _P, _P, _P, _I64, _PP]),
    "hnhd_spmat_info": (C.c_int, [_P, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64),
                                  C.POINTER(C.c_int64)]),
    "hnhd_spmat_tuples": (C.c_int, [_P, _P, _P, _P, _I64]),
    "hnhd_spmat_destroy": (None, [_P]),
    "hnhd_alg_create": (C.c_int, [C.c_char_p, _P, C.c_int, C.c_int, _PP]),
    "hnhd_alg_destroy": (None, [_P]),
    "hnhd_alg_dims": (C.c_int, [_P, C.POINTER(AlgDims)]),
    "hnhd_alg_submatrices": (C.c_int, [_P, C.c_int, _P, C.c_int]),
    "hnhd_setup_times_json": (C.c_int, [C.c_char_p, _SZ, C.c_int]),
    "hnhd_alg_info_json": (C.c_int, [_P, C.c_char_p, _SZ]),
    "hnhd_alg_perf_json": (C.c_int, [_P, C.c_char_p, _SZ]),
    "hnhd_alg_reset_timers": (C.c_int, [_P]),
    "hnhd_alg_block_count": (C.c_int, [_P, C.c_int]),
    "hnhd_alg_block_meta": (C.c_int, [_P, C.c_int, C.c_int, C.POINTER(C.c_int64), C.POINTER(C.c_int64),
                                      C.POINTER(C.c_int64), C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "hnhd_alg_block_arrays": (C.c_int, [_P, C.c_int, C.c_int, _P, _P, _P, _P]),
    "hnhd_dense_create": (C.c_int, [_I64, _I64, C.c_double, _PP]),
    "hnhd_dense_like": (C.c_int, [_P, C.c_int, C.c_double, _PP]),
    "hnhd_dense_fill": (C.c_int, [_P, C.c_double]),
    "hnhd_dense_dummy_initialize": (C.c_int, [_P, _P, C.c_int]),
    "hnhd_dense_from_host": (C.c_int, [_P, _P]),
    "hnhd_dense_to_host": (C.c_int, [_P, _P]),
    "hnhd_dense_shape": (C.c_int, [_P, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "hnhd_dense_data": (_P, [_P]),
    "hnhd_dense_destroy": (None, [_P]),
    "hnhd_vec_create": (C.c_int, [_I64, C.c_double, _PP]),
    "hnhd_vec_like": (C.c_int, [_P, C.c_int, C.c_double, _PP]),
    "hnhd_vec_fill": (C.c_int, [_P, C.c_double]),
    "hnhd_vec_from_host": (C.c_int, [_P, _P]),
    "hnhd_vec_to_host": (C.c_int, [_P, _P]),
    "hnhd_vec_size": (C.c_int64, [_P]),
    "hnhd_vec_destroy": (None, [_P]),
    "hnhd_alg_op": (C.c_int, [_P, C.c_int, _P, _P, _P, _P, C.c_int]),
    "hnhd_alg_fused_host": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _P, C.c_int, C.c_int64]),
    "hnhd_als_run": (C.c_int, [_P, _P, _P, _P, _P, C.c_int, C.c_int, _P, _P, _P]),
    "hnhd_gat_create": (C.c_int, [_P, C.c_int, C.POINTER(C.c_int), C.c_double, _PP]),
    "hnhd_gat_weight_shape": (C.c_int, [_P, C.c_int, C.c_int, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "hnhd_gat_set_weight": (C.c_int, [_P, C.c_int, C.c_int, _P]),
    "hnhd_gat_get_weight": (C.c_int, [_P, C.c_int, C.c_int, _P]),
    "hnhd_gat_get_attention_vectors": (C.c_int, [_P, C.c_int, C.c_int, _P, _P]),
    "hnhd_gat_get_weight_grad": (C.c_int, [_P, C.c_int, C.c_int, _P]),
    "hnhd_gat_set_attention": (C.c_int, [_P, C.c_char_p]),
    "hnhd_gat_set_attention_vectors": (C.c_int, [_P, C.c_int, C.c_int, _P, _P]),
    "hnhd_gat_get_attention_grads": (C.c_int, [_P, C.c_int, C.c_int, _P, _P]),
    "hnhd_alg_edge_softmax": (C.c_int, [_P, _P, C.c_int]),
    "hnhd_alg_edge_softmax_backward": (C.c_int, [_P, _P, _P, C.c_int]),
    "hnhd_alg_additive_scores": (C.c_int, [_P, _P, _P, _P, C.c_int, C.c_double, C.c_int]),
    "hnhd_alg_edge_sums": (C.c_int, [_P, _P, _P, _P]),
    "hnhd_alg_gatv2_scores": (C.c_int, [_P, _P, _P, _P, _P, C.c_int, C.c_double]),
    "hnhd_alg_gatv2_backward": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _P, C.c_double]),
    "hnhd_alg_sparse_attention": (C.c_int, [_P, _P, _P, _P, _P, _P, C.c_int, C.c_double]),
    "hnhd_alg_sparse_attention_backward": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, C.c_int, C.c_double]),
    "hnhd_alg_sparse_attention_dropout": (C.c_int, [_P, _P, _P, _P, _P, _P, C.c_int, C.c_double, C.c_double, C.c_uint64]),
    "hnhd_alg_sparse_attention_backward_dropout": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, C.c_int, C.c_double,
                                                             C.c_double, C.c_uint64]),
    "hnhd_alg_sparse_attention_bias": (C.c_int, [_P, _P, _P, _P, _P, _P, C.c_int, C.c_double, C.c_double, C.c_uint64, _P]),
    "hnhd_alg_sparse_attention_backward_bias": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, C.c_int, C.c_double,
                                                          C.c_double, C.c_uint64, _P, _P, _P, _P]),
    "hnhd_alg_sparse_attention_edge": (C.c_int, [_P, _P, _P, _P, _P, _P, C.c_int, C.c_double, C.c_double, C.c_uint64, _P,
                                                 _P]),
    "hnhd_alg_sparse_attention_backward_edge": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, C.c_int, C.c_double,
                                                          C.c_double, C.c_uint64, _P, _P, _P, _P, _P, _P, _P]),
    "hnhd_alg_entry_coordinates": (C.c_int, [_P, C.c_int, _P, _P]),
    "hnhd_gt_create": (C.c_int, [_P, C.c_int, C.POINTER(C.c_int), C.c_int, C.c_int, _PP]),
    "hnhd_gt_create_block": (C.c_int, [_P, C.c_int, C.POINTER(C.c_int), C.c_int, C.c_int, C.c_int, C.c_double, _PP]),
    "hnhd_gt_set_edge_attributes": (C.c_int, [_P, _P, _I64, _P, _I64]),
    "hnhd_labels_create": (C.c_int, [_P, _P, _I64, C.c_int, _PP]),
    "hnhd_labels_destroy": (None, [_P]),
    "hnhd_adamw_create": (C.c_int, [C.c_double, C.c_double, C.c_double, C.c_double, C.c_double, C.c_double, _PP]),
    "hnhd_adamw_set_lr": (C.c_int, [_P, C.c_double]),
    "hnhd_adamw_destroy": (None, [_P]),
    "hnhd_alg_link_loss": (C.c_int, [_P, _P, _P, _P, _P, _P, _P]),
    "hnhd_link_targets_create": (C.c_int, [_P, _P, _PP]),
    "hnhd_link_targets_destroy": (None, [_P]),
    "hnhd_alg_distmult_loss": (C.c_int, [_P, _P, _P, _P, C.c_int, C.c_double, C.c_double, _P, _P, _P, _P, C.c_int, _P]),
    "hnhd_distmult_create": (C.c_int, [_P, C.c_int, C.c_int, _PP]),
    "hnhd_distmult_destroy": (None, [_P]),
    "hnhd_distmult_param_shape": (C.c_int, [_P, C.c_char_p, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "hnhd_distmult_set_param": (C.c_int, [_P, C.c_char_p, _P]),
    "hnhd_distmult_get_param": (C.c_int, [_P, C.c_char_p, _P]),
    "hnhd_distmult_get_param_grad": (C.c_int, [_P, C.c_char_p, _P]),
    "hnhd_relational_link_targets_create": (C.c_int, [_P, _P, _P, C.c_int, _PP]),
    "hnhd_relational_link_targets_destroy": (None, [_P]),
    "hnhd_model_relational_link_train_step": (C.c_int, [_P, _P, _P, _P, C.c_double, C.c_uint64, _P]),
    "hnhd_model_relational_link_evaluate": (C.c_int, [_P, _P, _P, _P, _P, _P]),
    "hnhd_link_ranking_create": (C.c_int, [_P, _P, _P, _P, _I64, C.c_int, _PP]),
    "hnhd_link_ranking_destroy": (None, [_P]),
    "hnhd_model_link_rank": (C.c_int, [_P, _P, _P, _P, _P, _P, _I64, _P, _P, C.POINTER(C.c_double)]),
    "hnhd_alg_max_aggregate": (C.c_int, [_P, _P, _P, _P]),
    "hnhd_alg_max_aggregate_backward": (C.c_int, [_P, _P, _P, _P, _P, _P, C.c_int]),
    "hnhd_sage_create": (C.c_int, [_P, C.c_int, C.POINTER(C.c_int), C.c_char_p, _PP]),
    "hnhd_alg_relational_aggregate": (C.c_int, [_P, _P, _P, C.c_int]),
    "hnhd_alg_relational_aggregate_backward": (C.c_int, [_P, _P, _P, C.c_int, C.c_int]),
    "hnhd_alg_multi_aggregate": (C.c_int, [_P, _P, _P, C.c_int]),
    "hnhd_alg_multi_aggregate_backward": (C.c_int, [_P, _P, _P, _P, _P, C.c_int, C.c_int]),
    "hnhd_alg_edge_relu_aggregate": (C.c_int, [_P, _P, _P, _P]),
    "hnhd_alg_edge_relu_aggregate_backward": (C.c_int, [_P, _P, _P, _P, _P, _P, _P, C.c_int]),
    "hnhd_gin_create": (C.c_int, [_P, C.c_int, C.POINTER(C.c_int), C.c_int, C.c_double, C.c_int, _PP]),
    "hnhd_gin_set_edge_attributes": (C.c_int, [_P, _P, _I64, _P, _I64]),
    "hnhd_pna_create": (C.c_int, [_P, C.c_int, C.POINTER(C.c_int), C.c_char_p, C.c_char_p, C.c_double, C.c_double, _PP]),
    "hnhd_rgcn_create": (C.c_int, [_P, C.c_int, C.POINTER(C.c_int), C.c_int, C.c_char_p, _PP]),
    "hnhd_rgcn_create_bases": (C.c_int, [_P, C.c_int, C.POINTER(C.c_int), C.c_int, C.c_int, C.c_char_p, _PP]),
    "hnhd_alg_basis_aggregate": (C.c_int, [_P, _P, _P, _P, C.c_int, _P]),
    "hnhd_alg_basis_aggregate_backward": (C.c_int, [_P, _P, _P, _P, _P, _P, C.c_int, _P, C.c_int]),
    "hnhd_model_buffer_shape": (C.c_int, [_P, C.c_int, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "hnhd_model_set_input": (C.c_int, [_P, _P]),
    "hnhd_model_get_buffer": (C.c_int, [_P, C.c_int, _P]),
    "hnhd_model_forward": (C.c_int, [_P, C.c_double, C.c_uint64]),
    "hnhd_model_backward": (C.c_int, [_P, _P]),
    "hnhd_model_get_input_grad": (C.c_int, [_P, _P]),
    "hnhd_model_param_shape": (C.c_int, [_P, C.c_int, C.c_char_p, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "hnhd_model_set_param": (C.c_int, [_P, C.c_int, C.c_char_p, _P]),
    "hnhd_model_get_param": (C.c_int, [_P, C.c_int, C.c_char_p, _P]),
    "hnhd_model_get_param_grad": (C.c_int, [_P, C.c_int, C.c_char_p, _P]),
    "hnhd_model_train_step": (C.c_int, [_P, _P, _P, C.c_double, C.c_uint64, _P]),
    "hnhd_model_link_train_step": (C.c_int, [_P, _P, _P, C.c_double, C.c_uint64, _P]),
    "hnhd_model_link_evaluate": (C.c_int, [_P, _P, _P, _P]),
    "hnhd_model_destroy": (None, [_P]),
    "hnhd_readout_create": (C.c_int, [_P, _P, _I64, _I64, C.c_char_p, C.c_int, _PP]),
    "hnhd_readout_destroy": (None, [_P]),
    "hnhd_readout_pool": (C.c_int, [_P, _P, _P]),
    "hnhd_readout_pool_backward": (C.c_int, [_P, _P, _P, _P]),
    "hnhd_readout_param_shape": (C.c_int, [_P, C.c_char_p, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "hnhd_readout_set_param": (C.c_int, [_P, C.c_char_p, _P]),
    "hnhd_readout_get_param": (C.c_int, [_P, C.c_char_p, _P]),
    "hnhd_readout_get_param_grad": (C.c_int, [_P, C.c_char_p, _P]),
    "hnhd_graph_labels_create": (C.c_int, [_P, _P, _I64, C.c_int, _PP]),
    "hnhd_graph_labels_destroy": (None, [_P]),
    "hnhd_model_graph_train_step": (C.c_int, [_P, _P, _P, _P, C.c_double, C.c_uint64, _P]),
    "hnhd_model_graph_evaluate": (C.c_int, [_P, _P, _P, _P, _P]),
    "hnhd_timer_start": (C.c_int, []),
    "hnhd_timer_stop": (C.c_int, [C.POINTER(C.c_double)]),
    "hnhd_als_residuals": (C.c_int, [_P, C.c_int, _P]),
    "hnhd_benchmark_algorithm": (C.c_int, [_P, C.c_char_p, C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_char_p,
                                           C.c_int, C.c_int, C.c_char_p, _SZ]),
})
