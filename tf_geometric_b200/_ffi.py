# coding=utf-8
"""ctypes binding of include/tfgk.h (libtfgk.so, sm_90a).

There is deliberately NO fallback: if the shared library is missing, or a call fails, an exception is raised.
PyTorch is only the owner of device memory and streams; every pointer handed to the library is `tensor.data_ptr()`.
"""
import ctypes
import os
import threading

_LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "lib", "libtfgk.so")
_lock = threading.Lock()
_lib = None

ABI_VERSION = 7

OK = 0
ERR_INVALID_ARGUMENT, ERR_CUDA, ERR_WORKSPACE, ERR_UNSUPPORTED, ERR_INDEX_OUT_OF_RANGE = 1, 2, 3, 4, 5
REDUCE_SUM, REDUCE_MEAN, REDUCE_MAX = 0, 1, 2
ACT_NONE, ACT_RELU = 0, 1
POW_INV_SQRT, POW_INV = 0, 1
HEADS_SPLIT, HEADS_BROADCAST, HEADS_REDUCE = 0, 1, 2
FLAG_ALL, FLAG_UPPER, FLAG_MAPPED = 0, 1, 2
BERNOULLI_NONE, BERNOULLI_DROPOUT, BERNOULLI_KEEP = 0, 1, 2
SAMPLE_NO_PADDING, SAMPLE_PADDING, SAMPLE_HEAD = 0, 1, 2
GCN_NORM_BOTH, GCN_NORM_LEFT, GCN_NORM_RIGHT = 0, 1, 2
GCN_LOOP_NONE, GCN_LOOP_NORMED, GCN_LOOP_FILL = 0, 1, 2
NEG_UPPER, NEG_START = 0, 1
PAD_ROW_MAJOR, PAD_STEP_MAJOR = 0, 1
SPGEMM_GRAD_LEFT, SPGEMM_GRAD_RIGHT = 0, 1
DTYPE_F32, DTYPE_BF16, DTYPE_FP8_E4M3, DTYPE_F16 = 0, 1, 2, 3

_i32, _i64, _f32, _int = ctypes.c_int32, ctypes.c_int64, ctypes.c_float, ctypes.c_int
_ptr, _size = ctypes.c_void_p, ctypes.c_size_t
_u64, _u32, _f64 = ctypes.c_uint64, ctypes.c_uint32, ctypes.c_double

# name -> argtypes, exactly as declared in include/tfgk.h (tests check every symbol is exported)
SIGNATURES = {
    "tfgk_version": [],
    "tfgk_device_info": [ctypes.POINTER(_int)] * 3,
    "tfgk_self_loops_i32": [_ptr, _i64, _i32, _ptr, _ptr],
    "tfgk_self_loop_weights_f32": [_ptr, _i64, _i32, _f32, _ptr, _ptr],
    "tfgk_segment_count_i32": [_ptr, _i64, _i32, _ptr, _ptr],
    "tfgk_csr_workspace_bytes": [_i64, _i32, ctypes.POINTER(_size)],
    "tfgk_csr_build": [_ptr, _ptr, _i64, _i32, _i32, _ptr, _ptr, _ptr, _ptr, _size, _ptr],
    "tfgk_csr_build_in_range": [_ptr, _ptr, _i64, _i32, _i32, _ptr, _ptr, _ptr, _ptr, _size, _ptr],
    "tfgk_edge_unique_workspace_bytes": [_i64, _i32, ctypes.POINTER(_size)],
    "tfgk_edge_unique": [_ptr, _ptr, _i64, _i32, _ptr, _ptr, ctypes.POINTER(_i32), _ptr, _size, _ptr],
    "tfgk_directed_workspace_bytes": [_i64, ctypes.POINTER(_size)],
    "tfgk_directed_edges": [_ptr, _i64, _i64, _ptr, _i64, _ptr, ctypes.POINTER(_i32), _ptr, _size, _ptr],
    "tfgk_plan_capacity": [_i64, _i32, _i32, _i32, _i32, ctypes.POINTER(_i64), ctypes.POINTER(_i64)],
    "tfgk_plan_workspace_bytes": [_i32, ctypes.POINTER(_size)],
    "tfgk_plan_build": [_ptr, _i32, _i32, _i32, _i32, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _i64, _i64,
                        ctypes.POINTER(_i32), _ptr, _size, _ptr],
    "tfgk_permute_f32": [_ptr, _ptr, _i64, _i32, _ptr, _ptr],
    "tfgk_unpermute_f32": [_ptr, _ptr, _i64, _i32, _ptr, _ptr],
    "tfgk_host_register": [_ptr, _size, ctypes.POINTER(_ptr)],
    "tfgk_host_unregister": [_ptr],
    "tfgk_gather_rows_mapped_f32": [_ptr, _i64, _i64, _i32, _ptr, _i64, _ptr, _i64, _ptr],
    "tfgk_gather_rows_cached_f32": [_ptr, _i64, _i64, _i32, _ptr, _i64, _ptr, _ptr, _i64, _ptr, _i64, _ptr],
    "tfgk_gather_rows_mapped_16": [_ptr, _i32, _i64, _i64, _i32, _ptr, _i64, _ptr, _i32, _i64, _ptr],
    "tfgk_gather_rows_cached_16": [_ptr, _i32, _i64, _i64, _i32, _ptr, _i64, _ptr, _ptr, _i64, _ptr, _i64, _ptr],
    "tfgk_mapped_id_range_i32": [_ptr, _ptr, _i64, _ptr, _ptr, _size, _ptr],
    "tfgk_mapped_rowptr_workspace_bytes": [_i32, ctypes.POINTER(_size)],
    "tfgk_mapped_rowptr_i32": [_ptr, _i64, _i32, _ptr, _ptr, _size, _ptr],
    "tfgk_mapped_select_rows_workspace_bytes": [_i64, ctypes.POINTER(_size)],
    "tfgk_mapped_select_rows_i32": [_ptr, _ptr, _ptr, _i64, _i32, _i32, _ptr, _ptr, _ptr, _i64, _ptr, _size, _ptr],
    "tfgk_csr_rowsum_f32": [_ptr, _ptr, _i32, _ptr, _ptr],
    "tfgk_deg_inv_f32": [_ptr, _i32, _int, _ptr, _ptr],
    "tfgk_scale_edges_f32": [_ptr, _ptr, _ptr, _i64, _ptr, _ptr, _ptr, _ptr],
    "tfgk_spmm_f32": [_ptr, _ptr, _ptr, _ptr, _i64, _i32, _i32, _int, _f32, _ptr, _i64, _f32, _ptr, _int, _ptr, _i64,
                      _ptr, _ptr],
    "tfgk_spmm_proj_f32": [_ptr, _ptr, _ptr, _ptr, _i64, _i32, _i32, _ptr, _i32, _ptr, _int, _ptr, _i64, _ptr, _ptr],
    "tfgk_spmm_bf16": [_ptr, _ptr, _ptr, _ptr, _i64, _i32, _i32, _int, _f32, _ptr, _i64, _f32, _ptr, _int, _ptr, _i64,
                       _ptr, _ptr],
    "tfgk_spmm_bf16_dual": [_ptr, _ptr, _ptr, _ptr, _i64, _i32, _i32, _int, _f32, _ptr, _i64, _f32, _ptr, _int, _ptr,
                            _i64, _ptr, _i64, _ptr, _ptr],
    "tfgk_spmm_fp8": [_ptr, _ptr, _ptr, _ptr, _i64, _ptr, _i32, _i32, _int, _f32, _ptr, _i64, _f32, _ptr, _int, _ptr,
                      _i64, _ptr, _ptr],
    "tfgk_segment_softmax_f32": [_ptr, _ptr, _i32, _i32, _ptr, _ptr],
    "tfgk_gat_fused_f32": [_ptr, _ptr, _ptr, _i64, _ptr, _i64, _ptr, _i64, _i32, _i32, _i32, _i32, _f32, _int, _ptr,
                           _int, _ptr, _int, _ptr, _i64, _ptr, _ptr],
    "tfgk_gat_fused_bf16": [_ptr, _ptr, _ptr, _i64, _ptr, _i64, _ptr, _i64, _i32, _i32, _i32, _i32, _f32, _int, _ptr,
                            _int, _ptr, _int, _ptr, _i64, _ptr, _ptr],
    "tfgk_gat_fused_fp8": [_ptr, _ptr, _ptr, _i64, _ptr, _i64, _ptr, _i32, _i32, _i32, _f32, _ptr, _int, _ptr, _i64, _ptr,
                           _ptr],
    "tfgk_gat_pack_keys_f32": [_ptr, _i64, _i32, _i32, _ptr, _i64, _ptr, _ptr],
    "tfgk_gat_fused_packed_f32": [_ptr, _ptr, _ptr, _i64, _ptr, _i64, _ptr, _i32, _i32, _i32, _f32, _ptr, _int, _ptr, _i64,
                                  _ptr, _ptr],
    "tfgk_gemm_workspace_bytes": [_i32, _i32, _i32, ctypes.POINTER(_size)],
    "tfgk_gemm_f32": [_ptr, _i64, _int, _ptr, _i64, _int, _ptr, _int, _f32, _i32, _i32, _i32, _ptr, _i64, _ptr, _size,
                      _ptr],
    "tfgk_gemm_proj_f32": [_ptr, _i32, _i64, _i64, _i32, _i32, _ptr, _i32, _i32, _i32, _ptr],
    "tfgk_gemm_proj_mixed": [_ptr, _i32, _i64, _i64, _i32, _i32, _ptr, _i32, _i32, _i32, _ptr],
    "tfgk_round_bf16": [_ptr, _i64, _i32, _i32, _ptr, _i64, _ptr],
    "tfgk_gemm_proj_fp8": [_ptr, _i32, _i64, _i64, _i32, _i32, _ptr, _i32, _i32, _i32, _ptr],
    "tfgk_quantize_fp8": [_ptr, _i64, _i32, _i32, _ptr, _i64, _ptr, _i64, _ptr],
    "tfgk_peer_alloc": [_size, ctypes.POINTER(_ptr)],
    "tfgk_peer_free": [_ptr],
    "tfgk_peer_export": [_ptr, _ptr],
    "tfgk_peer_open": [_ptr, ctypes.POINTER(_ptr)],
    "tfgk_peer_close": [_ptr],
    "tfgk_peer_barrier": [_ptr, _i32, _i32, _u32, _i32, _ptr],
    "tfgk_peer_pull": [_ptr, _ptr, _i64, _i32, _ptr],
    "tfgk_colsum_workspace_bytes": [_i64, _i32, ctypes.POINTER(_size)],
    "tfgk_colsum_f32": [_ptr, _i64, _i64, _i32, _ptr, _ptr, _size, _ptr],
    "tfgk_l2_normalize_f32": [_ptr, _i64, _i32, _i32, _ptr, _i64, _ptr],
    "tfgk_dropout_f32": [_ptr, _i64, _f32, _u64, _u32, _ptr, _ptr],
    "tfgk_spmm_heads_f32": [_ptr, _ptr, _ptr, _ptr, _ptr, _i64, _i32, _i32, _i32, _int, _f32, _u64, _u32, _f32, _ptr,
                            _int, _ptr, _i64, _ptr],
    "tfgk_gat_softmax_bwd_f32": [_ptr, _ptr, _ptr, _ptr, _i64, _ptr, _i64, _i32, _i32, _i32, _int, _f32, _u64, _u32,
                                 _ptr, _ptr],
    "tfgk_dropout_devkey_f32": [_ptr, _i64, _f32, _ptr, _u64, _u32, _ptr, _ptr],
    "tfgk_spmm_heads_devkey_f32": [_ptr, _ptr, _ptr, _ptr, _ptr, _i64, _i32, _i32, _i32, _int, _f32, _ptr, _u64, _u32, _f32,
                                   _ptr, _int, _ptr, _i64, _ptr],
    "tfgk_gat_softmax_bwd_devkey_f32": [_ptr, _ptr, _ptr, _ptr, _i64, _ptr, _i64, _i32, _i32, _i32, _int, _f32, _ptr, _u64,
                                        _u32, _ptr, _ptr],
    "tfgk_rng_advance": [_ptr, _ptr, _ptr],
    "tfgk_capture_id": [_ptr, ctypes.POINTER(_u64)],
    "tfgk_gat_fused_stats_f32": [_ptr, _ptr, _ptr, _i64, _ptr, _i64, _ptr, _i64, _i32, _i32, _i32, _i32, _f32, _ptr, _int,
                                 _ptr, _i64, _ptr, _ptr, _ptr],
    "tfgk_gat_bwd_prepare_f32": [_ptr, _i64, _ptr, _i64, _ptr, _int, _ptr, _i32, _i32, _i32, _ptr, _i64, _ptr],
    "tfgk_gat_bwd_dst_f32": [_ptr, _ptr, _ptr, _i64, _ptr, _i64, _ptr, _i64, _ptr, _i64, _i32, _i32, _i32, _f32, _ptr, _i64,
                             _ptr],
    "tfgk_gat_bwd_src_f32": [_ptr, _ptr, _ptr, _i64, _ptr, _i64, _ptr, _i64, _ptr, _i64, _i32, _i32, _i32, _f32, _ptr, _i64,
                             _ptr, _i64, _ptr],
    "tfgk_edge_flags_i32": [_ptr, _ptr, _i64, _int, _ptr, _ptr, _int, _f32, _u64, _u32, _ptr, _ptr],
    "tfgk_select_workspace_bytes": [_i64, ctypes.POINTER(_size)],
    "tfgk_select_flagged_i32": [_ptr, _i64, _ptr, ctypes.POINTER(_i64), _ptr, _size, _ptr],
    "tfgk_sort_keys_f32": [_ptr, _i64, _int, _ptr, _ptr],
    "tfgk_argsort_workspace_bytes": [_i64, ctypes.POINTER(_size)],
    "tfgk_stable_argsort_u32": [_ptr, _i64, _int, _ptr, _ptr, _size, _ptr],
    "tfgk_neighbor_sample_workspace_bytes": [_i32, ctypes.POINTER(_size)],
    "tfgk_neighbor_sample_count": [_ptr, _i32, _i32, _f64, _int, _ptr, ctypes.POINTER(_i64), _ptr, _size, _ptr],
    "tfgk_neighbor_sample_fill": [_ptr, _i32, _i32, _f64, _int, _u64, _u32, _ptr, _ptr, _ptr, _ptr],
    "tfgk_neighbor_sample_rows_count": [_ptr, _i32, _ptr, _i32, _i32, _f64, _int, _ptr, ctypes.POINTER(_i64), _ptr, _size,
                                        _ptr],
    "tfgk_neighbor_sample_rows_fill": [_ptr, _i32, _ptr, _i32, _i32, _f64, _int, _u64, _u32, _ptr, _ptr, _ptr, _ptr],
    "tfgk_relabel_workspace_bytes": [_i64, ctypes.POINTER(_size)],
    "tfgk_reindex_i32": [_ptr, _i32, _ptr, _i64, _i32, _ptr, _ptr, ctypes.POINTER(_i32), _ptr, _size, _ptr],
    "tfgk_frontier_i32": [_ptr, _i64, _i32, _ptr, _i32, _ptr, _ptr, ctypes.POINTER(_i32), ctypes.POINTER(_i32), _ptr, _size,
                          _ptr],
    "tfgk_block_sample_workspace_bytes": [_i32, _i64, ctypes.POINTER(_size)],
    "tfgk_block_sample_begin": [_ptr, _i32, _i32, _ptr, _ptr, _ptr, _i32, _ptr],
    "tfgk_block_sample_count": [_ptr, _i32, _ptr, _ptr, _i32, _i32, _i32, _i32, _int, _ptr, _ptr, _size, _ptr],
    "tfgk_block_sample_read_total": [_ptr, _i32, _ptr, _i32, ctypes.POINTER(_i32), ctypes.POINTER(_i64), _ptr],
    "tfgk_block_sample_fill": [_ptr, _i32, _ptr, _ptr, _i32, _ptr, _ptr, _ptr, _i32, _i32, _i32, _i64, _i32, _int, _u64,
                               _u32, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _size, _ptr],
    "tfgk_block_sample_end": [_ptr, _i32, _i32, _ptr, _ptr, _i32, _ptr, _ptr],
    "tfgk_block_sample_mapped_workspace_bytes": [_i32, _i64, ctypes.POINTER(_size)],
    "tfgk_block_sample_fill_mapped": [_ptr, _i32, _ptr, _ptr, _i32, _ptr, _ptr, _ptr, _i32, _i32, _i32, _i64, _i32, _int,
                                      _u64, _u32, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _size, _ptr],
    "tfgk_block_self_loops_i32": [_ptr, _ptr, _ptr, _i64, _i32, _ptr, _ptr, _ptr, _ptr],
    "tfgk_block_gcn_values_f32": [_ptr, _ptr, _ptr, _i64, _ptr, _i32, _ptr, _ptr, _int, _int, _f32, _f32, _ptr, _ptr],
    "tfgk_block_pairs_workspace_bytes": [_i32, ctypes.POINTER(_size)],
    "tfgk_block_sample_begin_pairs": [_ptr, _ptr, _i32, _i32, _ptr, _ptr, _ptr, _i32, _ptr, _ptr, _size, _ptr],
    "tfgk_link_tail_negatives_i32": [_ptr, _i32, _i32, _i32, _u64, _u32, _ptr, _ptr, _ptr],
    "tfgk_block_exclusion_workspace_bytes": [_i32, ctypes.POINTER(_size)],
    "tfgk_block_exclusion_count": [_ptr, _i32, _ptr, _ptr, _i32, _ptr, _ptr, _i64, _ptr, ctypes.POINTER(_i64), _ptr, _size,
                                   _ptr],
    "tfgk_block_exclusion_fill": [_ptr, _i32, _ptr, _ptr, _i32, _ptr, _ptr, _ptr, _ptr, _size, _ptr],
    "tfgk_block_exclusion_fill_mapped": [_ptr, _i32, _ptr, _ptr, _i32, _ptr, _ptr, _ptr, _ptr, _size, _ptr],
    "tfgk_block_sample_count_excl": [_ptr, _i32, _ptr, _ptr, _i32, _i32, _i32, _i32, _int, _ptr, _i32, _ptr, _ptr, _size,
                                     _ptr],
    "tfgk_block_sample_fill_excl": [_ptr, _i32, _ptr, _ptr, _i32, _ptr, _ptr, _ptr, _i32, _i32, _i32, _i64, _i32, _int,
                                    _u64, _u32, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _i32, _ptr, _size, _ptr],
    "tfgk_block_sample_fill_mapped_excl": [_ptr, _i32, _ptr, _ptr, _i32, _ptr, _ptr, _ptr, _i32, _i32, _i32, _i64, _i32,
                                           _int, _u64, _u32, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _i32, _ptr, _size,
                                           _ptr],
    "tfgk_block_gcn_values_excl_f32": [_ptr, _ptr, _ptr, _i64, _ptr, _i32, _ptr, _ptr, _int, _int, _f32, _f32, _ptr, _i32,
                                       _ptr, _ptr],
    "tfgk_csr_positive_degree_f32": [_ptr, _i32, _ptr, _i64, _ptr, _ptr, _ptr],
    "tfgk_neighbor_sample_rows_count_weighted": [_ptr, _i32, _ptr, _i32, _i32, _int, _ptr, _ptr, _ptr,
                                                 ctypes.POINTER(_i64), _ptr, _size, _ptr],
    "tfgk_neighbor_sample_rows_fill_weighted": [_ptr, _i32, _ptr, _i32, _i32, _int, _ptr, _ptr, _u64, _u32, _ptr, _ptr,
                                                _ptr, _ptr],
    "tfgk_block_sample_count_weighted": [_ptr, _i32, _ptr, _ptr, _i32, _i32, _i32, _i32, _int, _ptr, _ptr, _ptr, _ptr,
                                         _size, _ptr],
    "tfgk_block_sample_count_weighted_excl": [_ptr, _i32, _ptr, _ptr, _i32, _i32, _i32, _i32, _int, _ptr, _ptr, _ptr,
                                              _ptr, _i32, _ptr, _ptr, _size, _ptr],
    "tfgk_block_sample_count_weighted_mapped_excl": [_ptr, _i32, _ptr, _ptr, _i32, _i32, _i32, _i32, _int, _ptr, _ptr,
                                                     _ptr, _ptr, _i32, _ptr, _ptr, _size, _ptr],
    "tfgk_block_sample_fill_weighted": [_ptr, _i32, _ptr, _ptr, _ptr, _i32, _ptr, _ptr, _ptr, _i32, _i32, _i32, _i64,
                                        _i32, _int, _u64, _u32, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _size, _ptr],
    "tfgk_block_sample_fill_weighted_excl": [_ptr, _i32, _ptr, _ptr, _ptr, _i32, _ptr, _ptr, _ptr, _i32, _i32, _i32,
                                             _i64, _i32, _int, _u64, _u32, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr,
                                             _i32, _ptr, _size, _ptr],
    "tfgk_block_sample_fill_weighted_mapped": [_ptr, _i32, _ptr, _ptr, _ptr, _i32, _ptr, _ptr, _ptr, _i32, _i32, _i32,
                                               _i64, _i32, _int, _u64, _u32, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _size,
                                               _ptr],
    "tfgk_block_sample_fill_weighted_mapped_excl": [_ptr, _i32, _ptr, _ptr, _ptr, _i32, _ptr, _ptr, _ptr, _i32, _i32,
                                                    _i32, _i64, _i32, _int, _u64, _u32, _ptr, _ptr, _ptr, _ptr, _ptr,
                                                    _ptr, _ptr, _i32, _ptr, _size, _ptr],
    "tfgk_block_sample_count_labor": [_ptr, _i32, _ptr, _ptr, _ptr, _i32, _i32, _i32, _i32, _u64, _u32, _ptr, _ptr, _size,
                                      _ptr],
    "tfgk_block_sample_count_labor_excl": [_ptr, _i32, _ptr, _ptr, _ptr, _i32, _i32, _i32, _i32, _u64, _u32, _ptr, _ptr,
                                           _i32, _ptr, _ptr, _size, _ptr],
    "tfgk_block_sample_count_labor_mapped_excl": [_ptr, _i32, _ptr, _ptr, _ptr, _i32, _i32, _i32, _i32, _u64, _u32, _ptr,
                                                  _ptr, _i32, _ptr, _ptr, _size, _ptr],
    "tfgk_block_sample_fill_labor": [_ptr, _i32, _ptr, _ptr, _i32, _ptr, _ptr, _ptr, _i32, _i32, _i32, _i64, _i32, _u64,
                                     _u32, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _size, _ptr],
    "tfgk_block_sample_fill_labor_excl": [_ptr, _i32, _ptr, _ptr, _i32, _ptr, _ptr, _ptr, _i32, _i32, _i32, _i64, _i32,
                                          _u64, _u32, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _i32, _ptr, _size, _ptr],
    "tfgk_block_sample_fill_labor_mapped": [_ptr, _i32, _ptr, _ptr, _i32, _ptr, _ptr, _ptr, _i32, _i32, _i32, _i64, _i32,
                                            _u64, _u32, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _size, _ptr],
    "tfgk_block_sample_fill_labor_mapped_excl": [_ptr, _i32, _ptr, _ptr, _i32, _ptr, _ptr, _ptr, _i32, _i32, _i32, _i64,
                                                 _i32, _u64, _u32, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _i32, _ptr,
                                                 _size, _ptr],
    "tfgk_row_block_i32": [_ptr, _i32, _i32, _i32, _ptr, _i64, _ptr, _ptr, _ptr, _ptr, _ptr, ctypes.POINTER(_i32), _ptr,
                           _size, _ptr],
    "tfgk_copy_async": [_ptr, _ptr, _size, _ptr],
    "tfgk_edge_dot_f32": [_ptr, _i64, _i32, _ptr, _ptr, _i64, _i32, _ptr, _ptr],
    "tfgk_neg_offsets_workspace_bytes": [_i32, ctypes.POINTER(_size)],
    "tfgk_neg_offsets": [_ptr, _i32, _int, _ptr, ctypes.POINTER(_i64), _ptr, _size, _ptr],
    "tfgk_neg_draw": [_i64, _ptr, _i64, _u64, _u32, _i32, _ptr, _ptr],
    "tfgk_neg_dup_flags": [_ptr, _ptr, _i64, _ptr, _ptr],
    "tfgk_neg_decode": [_ptr, _ptr, _ptr, _i32, _int, _ptr, _i64, _ptr, _ptr, _ptr],
    "tfgk_neg_sample_start": [_ptr, _ptr, _i32, _ptr, _i64, _u64, _u32, _ptr, _ptr],
    "tfgk_random_pairs_i32": [_i32, _i64, _u64, _u32, _ptr, _ptr],
    "tfgk_sddmm_csr_f32": [_ptr, _ptr, _ptr, _i32, _ptr, _i64, _ptr, _i64, _i32, _ptr, _f32, _ptr, _ptr],
    "tfgk_graph_tmm_workspace_bytes": [_i32, _i32, _i32, _i32, ctypes.POINTER(_size)],
    "tfgk_graph_tmm_f32": [_ptr, _i64, _ptr, _i64, _i32, _i32, _i32, _ptr, _ptr, _i32, _ptr, _i64, _ptr, _size, _ptr],
    "tfgk_graph_rmm_f32": [_ptr, _i64, _ptr, _i32, _ptr, _i64, _i32, _i32, _i32, _int, _f32, _ptr, _i64, _ptr],
    "tfgk_pad_rows_f32": [_ptr, _ptr, _i32, _i32, _int, _ptr, _i64, _i32, _i32, _ptr, _ptr, _ptr],
    "tfgk_unpad_rows_f32": [_ptr, _ptr, _i32, _i32, _ptr, _i32, _ptr, _i64, _ptr],
    "tfgk_spgemm_plan_workspace_bytes": [_i32, ctypes.POINTER(_size)],
    "tfgk_spgemm_plan": [_ptr, _ptr, _i32, _i32, _ptr, _ptr, _i32, _ptr, _ptr, _ptr, _ptr, _ptr, _size, _ptr],
    "tfgk_spgemm_rows_workspace_bytes": [_i64, ctypes.POINTER(_size)],
    "tfgk_spgemm_count": [_ptr, _ptr, _ptr, _ptr, _i32, _i32, _ptr, _ptr, _i64, _ptr, _ptr, _size, _ptr],
    "tfgk_spgemm_rowptr": [_ptr, _i32, _ptr, ctypes.POINTER(_i64), _ptr, _size, _ptr],
    "tfgk_spgemm_fill_f32": [_ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _i32, _i32, _ptr, _ptr, _i64, _ptr, _ptr, _ptr, _ptr, _size,
                             _ptr],
    "tfgk_spgemm_grad_workspace_bytes": [_i64, ctypes.POINTER(_size)],
    "tfgk_spgemm_grad_plan": [_int, _ptr, _ptr, _i64, _ptr, _ptr, _i32, _i32, _i32, _ptr, ctypes.POINTER(_i64), _ptr, _size,
                              _ptr],
    "tfgk_spgemm_grad_f32": [_int, _ptr, _ptr, _ptr, _i64, _ptr, _ptr, _ptr, _i32, _i32, _i32, _ptr, _ptr, _ptr, _ptr, _i64,
                             _ptr, _ptr, _ptr],
    "tfgk_spmm_max_f32":[_ptr, _ptr, _ptr, _ptr, _i64, _i32, _i32, _ptr, _i64, _ptr, _i64, _ptr, _ptr],
    "tfgk_spmm_max_bwd_f32": [_ptr, _ptr, _ptr, _ptr, _i64, _i32, _i32, _i32, _ptr, _i64, _ptr, _i64, _ptr, _i64, _ptr,
                              _ptr, _i64, _ptr, _ptr],
}


class PlanStruct(ctypes.Structure):
    """struct tfgk_plan of include/tfgk.h."""
    _fields_ = [("n_tasks", _i32), ("n_hubs", _i32), ("n_slots", _i32), ("chunk", _i32),
                ("task_row", _ptr), ("task_nrows", _ptr), ("task_e0", _ptr), ("task_e1", _ptr), ("task_slot", _ptr),
                ("hub_row", _ptr), ("hub_slot0", _ptr), ("hub_nslots", _ptr), ("scratch", _ptr), ("scratch_bytes", _size)]


class ProjBlock(ctypes.Structure):
    """struct tfgk_proj_block of include/tfgk.h."""
    _fields_ = [("B", _ptr), ("ldb", _i64), ("ncols", _i32), ("transB", _i32), ("bias", _ptr), ("act", _int), ("C", _ptr),
                ("ldc", _i64)]


class ProjBlockOut(ctypes.Structure):
    """struct tfgk_proj_block_out of include/tfgk.h."""
    _fields_ = ProjBlock._fields_ + [("c_dtype", _i32)]


class ProjBlockFp8(ctypes.Structure):
    """struct tfgk_proj_block_fp8 of include/tfgk.h."""
    _fields_ = ProjBlockOut._fields_ + [("E", _ptr), ("lde", _i64)]


PEER_HANDLE_BYTES = 64


class TfgkError(RuntimeError):
    """A tfgk_* entry point returned a non-zero status."""

    def __init__(self, fn, code, message):
        super().__init__("{} failed with status {}: {}".format(fn, code, message))
        self.code = code


def library_path():
    return _LIB_PATH


def lib():
    """Load libtfgk.so once.  Raises ImportError (never falls back) when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is None:
            if not os.path.exists(_LIB_PATH):
                raise ImportError(
                    "tf_geometric_b200: {} is missing - build it with `python -c 'import __graft_entry__ as g; "
                    "g.build()'` or `make -C tf_geometric_b200/csrc`. There is no CPU/PyTorch fallback.".format(_LIB_PATH))
            handle = ctypes.CDLL(_LIB_PATH)
            for name, argtypes in SIGNATURES.items():
                fn = getattr(handle, name)
                fn.argtypes = argtypes
                fn.restype = _int
            handle.tfgk_last_error.argtypes = []
            handle.tfgk_last_error.restype = ctypes.c_char_p
            if handle.tfgk_version() != ABI_VERSION:
                raise ImportError("libtfgk.so ABI version {} != expected {}".format(handle.tfgk_version(), ABI_VERSION))
            _lib = handle
    return _lib


class CallTrace(object):
    """Optional instrumentation used by bench.py: counts ABI calls by name and, for the names in `timed`, brackets the
    call with CUDA events on the launching stream (torch.cuda.Event on torch's current stream, which is the stream
    handed to the library)."""

    def __init__(self, timed=()):
        self.counts = {}
        self.timed = set(timed)
        self.events = {name: [] for name in self.timed}

    def elapsed_ms(self, name):
        """Per-call device durations (ms); call after synchronising."""
        return [a.elapsed_time(b) for a, b in self.events.get(name, [])]


_trace = None


def set_trace(trace):
    """Install (or remove, with None) a CallTrace; returns the previous one."""
    global _trace
    prev, _trace = _trace, trace
    return prev


# Entries that cannot be recorded in a CUDA graph, with the op that reaches them and why: they read a result back on the
# host (a size, a count, an id check), or they take a host-side random key that a graph would replay unchanged.
NOT_CAPTURABLE = {
    "tfgk_csr_build": ("the CSR build of an edge list without a cached structure", "it checks the node ids on the host"),
    "tfgk_plan_build": ("the work-plan build of a CSR", "it returns the task counts to the host"),
    "tfgk_edge_unique": ("the edge merge", "it returns the number of unique edges to the host"),
    "tfgk_directed_edges": ("the undirected-to-directed edge conversion", "it returns the edge count to the host"),
    "tfgk_edge_flags_i32": ("edge filtering (drop_edge, the edge samplers, convert_edge_to_upper)", "its flags are "
                            "compacted by select_flagged, which returns the number of kept edges to the host"),
    "tfgk_select_flagged_i32": ("select_flagged", "it returns the number of selected entries to the host"),
    "tfgk_neighbor_sample_count": ("the neighbour sampler", "it returns the number of sampled edges to the host"),
    "tfgk_neighbor_sample_fill": ("the neighbour sampler", "it takes a host-side key"),
    "tfgk_neighbor_sample_rows_count": ("the mini-batch neighbourhood sampler", "it returns the number of sampled edges "
                                        "to the host"),
    "tfgk_neighbor_sample_rows_fill": ("the mini-batch neighbourhood sampler", "it takes a host-side key"),
    "tfgk_reindex_i32": ("reindex_sampled_edge_index", "it returns the number of duplicate node ids to the host"),
    "tfgk_frontier_i32": ("the mini-batch neighbourhood sampler", "it returns the number of new nodes to the host"),
    "tfgk_block_sample_read_total": ("the block sampler", "it returns a hop's edge total to the host"),
    "tfgk_block_sample_fill": ("the block sampler", "it takes a host-side key"),
    "tfgk_block_sample_end": ("the block sampler", "it returns the batch's sizes to the host"),
    "tfgk_block_sample_fill_mapped": ("the host-memory block sampler", "it takes a host-side key"),
    "tfgk_block_sample_fill_excl": ("the link block sampler", "it takes a host-side key"),
    "tfgk_block_sample_fill_mapped_excl": ("the host-memory link block sampler", "it takes a host-side key"),
    "tfgk_link_tail_negatives_i32": ("the link block sampler's negatives", "it takes a host-side key"),
    "tfgk_neighbor_sample_rows_count_weighted": ("the weighted mini-batch neighbourhood sampler", "it returns the "
                                                 "number of sampled edges to the host"),
    "tfgk_neighbor_sample_rows_fill_weighted": ("the weighted mini-batch neighbourhood sampler", "it takes a host-side key"),
    "tfgk_block_sample_fill_weighted": ("the weighted block sampler", "it takes a host-side key"),
    "tfgk_block_sample_fill_weighted_excl": ("the weighted link block sampler", "it takes a host-side key"),
    "tfgk_block_sample_fill_weighted_mapped": ("the weighted host-memory block sampler", "it takes a host-side key"),
    "tfgk_block_sample_fill_weighted_mapped_excl": ("the weighted host-memory link block sampler",
                                                    "it takes a host-side key"),
    "tfgk_block_sample_count_labor": ("the LABOR block sampler", "it takes a host-side key"),
    "tfgk_block_sample_count_labor_excl": ("the LABOR link block sampler", "it takes a host-side key"),
    "tfgk_block_sample_count_labor_mapped_excl": ("the LABOR host-memory link block sampler", "it takes a host-side key"),
    "tfgk_block_sample_fill_labor": ("the LABOR block sampler", "it takes a host-side key"),
    "tfgk_block_sample_fill_labor_excl": ("the LABOR link block sampler", "it takes a host-side key"),
    "tfgk_block_sample_fill_labor_mapped": ("the LABOR host-memory block sampler", "it takes a host-side key"),
    "tfgk_block_sample_fill_labor_mapped_excl": ("the LABOR host-memory link block sampler", "it takes a host-side key"),
    "tfgk_block_exclusion_count": ("the link block sampler's exclusion lists", "it returns their total to the host"),
    "tfgk_row_block_i32": ("the row blocks of layer-wise inference", "it returns the number of source rows to the host"),
    "tfgk_host_register": ("HostFeatureTable", "it page-locks host memory, which a graph cannot record"),
    "tfgk_mapped_id_range_i32": ("the CSR build of HostNeighborSampler", "it returns the id range to the host"),
    "tfgk_neg_offsets": ("negative sampling", "it returns the number of candidate pairs to the host"),
    "tfgk_neg_draw": ("negative sampling", "it takes a host-side key"),
    "tfgk_neg_sample_start": ("negative sampling", "it takes a host-side key"),
    "tfgk_random_pairs_i32": ("negative sampling", "it takes a host-side key"),
    "tfgk_spgemm_plan": ("SparseMatrix @ SparseMatrix (K10's plan)", "it returns the product counts to the host"),
    "tfgk_spgemm_rowptr": ("SparseMatrix @ SparseMatrix (K10's row pointers)", "it returns the number of entries to the host"),
    "tfgk_spgemm_grad_plan": ("the SparseMatrix @ SparseMatrix gradient (K12's plan)", "it returns the slice count to the "
                              "host"),
}


def capturing():
    """Whether the current CUDA stream is recording a graph (torch.cuda.graph, make_graphed_callables)."""
    import torch
    return torch.cuda.is_initialized() and torch.cuda.is_current_stream_capturing()


def refuse_capture(op, reason):
    """Raise before any device work when `op` is called while the current stream records a CUDA graph."""
    if capturing():
        raise RuntimeError("{} cannot be captured in a CUDA graph: {}. Run it eagerly, outside the capture (a warm-up "
                           "step builds and caches the structures a captured step needs).".format(op, reason))


def call(name, *args):
    refusal = NOT_CAPTURABLE.get(name)
    if refusal is not None:
        refuse_capture(*refusal)
    handle = lib()
    trace = _trace
    if trace is None:
        rc = getattr(handle, name)(*args)
    else:
        trace.counts[name] = trace.counts.get(name, 0) + 1
        if name in trace.timed:
            import torch
            start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record()
            rc = getattr(handle, name)(*args)
            end.record()
            trace.events[name].append((start, end))
        else:
            rc = getattr(handle, name)(*args)
    if rc != OK:
        raise TfgkError(name, rc, handle.tfgk_last_error().decode("utf-8", "replace"))
    return rc
