"""ctypes loader for libvecb200.so (the C ABI declared in include/vecb200.h).

The library is the product; this module only binds it.  There is no Python or
CPU implementation behind any call: if the shared object is missing or no
sm_90 device is usable every entry point raises.
"""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libvecb200.so")

OK, EINVAL, ENODEVICE, ECUDA, ENOMEM, ESTATE = 0, -1, -2, -3, -4, -5

ALLREDUCE_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int64, C.c_int, C.c_void_p)

# name -> (restype, argtypes); keep in step with include/vecb200.h (tests/test_abi.py checks the header)
_vp, _i, _i64, _u64 = C.c_void_p, C.c_int, C.c_int64, C.c_uint64
SIGNATURES = {
    "vb_init": (_i, [_i]),
    "vb_shutdown": (_i, []),
    "vb_last_error": (C.c_char_p, []),
    "vb_last_error_detail": (C.c_char_p, []),
    "vb_abi_version": (_i, []),
    "vb_stream": (_vp, []),
    "vb_launch_count": (_i64, []),
    "vb_synchronize": (_i, []),
    "vb_stream_wait_event": (_i, [_vp]),
    "vb_prof_enable": (_i, [_i]),
    "vb_prof_read": (_i, [_i, C.POINTER(C.c_double), C.POINTER(_i64)]),
    "vb_distance_batch": (_i, [_i, _i, _i, _vp, _vp, _i64, _vp]),
    "vb_norm_batch": (_i, [_i, _i, _vp, _i64, _vp]),
    "vb_l2_normalize_batch": (_i, [_i, _i, _vp, _i64, _vp]),
    "vb_binary_quantize_batch": (_i, [_i, _i, _vp, _i64, _vp]),
    "vb_vector_to_halfvec_batch": (_i, [_i, _vp, _i64, _vp]),
    "vb_halfvec_to_vector_batch": (_i, [_i, _vp, _i64, _vp]),
    "vb_subvector_batch": (_i, [_i, _i, _vp, _i64, C.c_int32, C.c_int32, _vp, C.POINTER(_i)]),
    "vb_norm_batch_dev": (_i, [_i, _i, _vp, _i64, _vp]),
    "vb_l2_normalize_batch_dev": (_i, [_i, _i, _vp, _i64, _vp]),
    "vb_binary_quantize_batch_dev": (_i, [_i, _i, _vp, _i64, _vp]),
    "vb_vector_to_halfvec_batch_dev": (_i, [_i, _vp, _i64, _vp]),
    "vb_halfvec_to_vector_batch_dev": (_i, [_i, _vp, _i64, _vp]),
    "vb_subvector_batch_dev": (_i, [_i, _i, _vp, _i64, C.c_int32, C.c_int32, _vp, C.POINTER(_i)]),
    "vb_arith_batch": (_i, [_i, _i, _i, _vp, _i64, _i, _vp, _i64, _vp]),
    "vb_arith_batch_dev": (_i, [_i, _i, _i, _vp, _i64, _i, _vp, _i64, _vp]),
    "vb_concat_batch": (_i, [_i, _i, _vp, _i64, _i, _vp, _i64, _vp, C.POINTER(_i)]),
    "vb_concat_batch_dev": (_i, [_i, _i, _vp, _i64, _i, _vp, _i64, _vp, C.POINTER(_i)]),
    "vb_array_to_rows_batch": (_i, [_i, _i, _i, C.c_int32, _vp, _i64, _vp]),
    "vb_array_to_rows_batch_dev": (_i, [_i, _i, _i, C.c_int32, _vp, _i64, _vp]),
    "vb_numeric_array_to_rows_batch": (_i, [_i, _i, C.c_int32, _vp, _vp, _i64, _vp, C.POINTER(_i64)]),
    "vb_numeric_array_to_rows_batch_dev": (_i, [_i, _i, C.c_int32, _vp, _vp, _i64, _vp, C.POINTER(_i64)]),
    "vb_sparsevec_distance_batch": (_i, [_i, _i, _i, C.c_int32, _vp, _vp, _i64, _vp, _vp, _vp, _vp]),
    "vb_sparsevec_norm_batch": (_i, [_i64, _vp, _vp, _vp]),
    "vb_sparsevec_l2_normalize_batch": (_i, [_i64, _vp, _vp, _vp, _vp, _vp, _vp]),
    "vb_sparse_table_create": (_i, [_i, C.POINTER(_vp)]),
    "vb_sparse_table_append": (_i, [_vp, _i64, _vp, _vp, _vp]),
    "vb_sparse_table_rows": (_i64, [_vp]),
    "vb_sparse_table_nnz": (_i64, [_vp]),
    "vb_sparse_table_free": (_i, [_vp]),
    "vb_sparse_exact_topk": (_i, [_vp, _i, _i, _i64, _vp, _vp, _vp, _i, _vp, _vp]),
    "vb_sparse_table_filter_create": (_i, [_vp, _vp, _i64, C.POINTER(_vp)]),
    "vb_sparse_exact_topk_filtered": (_i, [_vp, _i, _i, _i64, _vp, _vp, _vp, _i, _vp, _i, _vp, _vp, _vp]),
    "vb_sparse_table_rerank": (_i, [_vp, _i, _i, _i64, _vp, _vp, _vp, _vp, _i, _i, _vp, _vp]),
    "vb_sparse_table_append_dev": (_i, [_vp, _i64, _vp, _vp, _vp]),
    "vb_sparse_exact_topk_dev": (_i, [_vp, _i, _i, _i64, _vp, _vp, _vp, _i, _vp, _vp]),
    "vb_sparse_table_filter_create_dev": (_i, [_vp, _vp, _i64, C.POINTER(_vp)]),
    "vb_sparse_exact_topk_filtered_dev": (_i, [_vp, _i, _i, _i64, _vp, _vp, _vp, _i, _vp, _i, _vp, _vp, _vp]),
    "vb_sparse_table_rerank_dev": (_i, [_vp, _i, _i, _i64, _vp, _vp, _vp, _vp, _i, _i, _vp, _vp]),
    "vb_array_to_sparsevec_batch": (_i, [_i, _i, C.c_int32, _vp, _vp, _i64, _i64, _vp, _vp, _vp, C.POINTER(_i64)]),
    "vb_array_to_sparsevec_batch_dev": (_i, [_i, _i, C.c_int32, _vp, _vp, _i64, _i64, _vp, _vp, _vp, C.POINTER(_i64)]),
    "vb_dense_to_sparsevec_batch": (_i, [_i, _i, _vp, _i64, _i64, _vp, _vp, _vp]),
    "vb_dense_to_sparsevec_batch_dev": (_i, [_i, _i, _vp, _i64, _i64, _vp, _vp, _vp]),
    "vb_sparsevec_to_dense_batch": (_i, [_i, _i, _i64, _vp, _vp, _vp, _vp]),
    "vb_sparsevec_to_dense_batch_dev": (_i, [_i, _i, _i64, _vp, _vp, _vp, _vp]),
    "vb_text_to_rows_batch": (_i, [_i, C.c_int32, _i64, _vp, _vp, _i64, _vp, _vp, C.POINTER(_i64)]),
    "vb_text_to_rows_batch_dev": (_i, [_i, C.c_int32, _i64, _vp, _vp, _i64, _vp, _vp, C.POINTER(_i64)]),
    "vb_text_to_sparsevec_batch": (_i, [C.c_int32, _i64, _vp, _vp, _i64, _vp, _vp, _vp, _vp, C.POINTER(_i64)]),
    "vb_text_to_sparsevec_batch_dev": (_i, [C.c_int32, _i64, _vp, _vp, _i64, _vp, _vp, _vp, _vp, C.POINTER(_i64)]),
    "vb_rows_to_text_batch": (_i, [_i, _i, _vp, _i64, _i64, _vp, _vp]),
    "vb_rows_to_text_batch_dev": (_i, [_i, _i, _vp, _i64, _i64, _vp, _vp]),
    "vb_sparsevec_to_text_batch": (_i, [_i, _i64, _vp, _vp, _vp, _i64, _vp, _vp]),
    "vb_sparsevec_to_text_batch_dev": (_i, [_i, _i64, _vp, _vp, _vp, _i64, _vp, _vp]),
    "vb_binary_to_rows_batch": (_i, [_i, C.c_int32, _i64, _vp, _vp, _i64, _vp, _vp, C.POINTER(_i64)]),
    "vb_binary_to_rows_batch_dev": (_i, [_i, C.c_int32, _i64, _vp, _vp, _i64, _vp, _vp, C.POINTER(_i64)]),
    "vb_binary_to_sparsevec_batch": (_i, [C.c_int32, _i64, _vp, _vp, _i64, _vp, _vp, _vp, _vp, C.POINTER(_i64)]),
    "vb_binary_to_sparsevec_batch_dev": (_i, [C.c_int32, _i64, _vp, _vp, _i64, _vp, _vp, _vp, _vp, C.POINTER(_i64)]),
    "vb_rows_to_binary_batch": (_i, [_i, _i, _vp, _i64, _i64, _vp, _vp]),
    "vb_rows_to_binary_batch_dev": (_i, [_i, _i, _vp, _i64, _i64, _vp, _vp]),
    "vb_sparsevec_to_binary_batch": (_i, [_i, _i64, _vp, _vp, _vp, _i64, _vp, _vp]),
    "vb_sparsevec_to_binary_batch_dev": (_i, [_i, _i64, _vp, _vp, _vp, _i64, _vp, _vp]),
    "vb_table_create": (_i, [_i, _i, C.POINTER(_vp)]),
    "vb_table_append": (_i, [_vp, _vp, _i64]),
    "vb_table_append_dev": (_i, [_vp, _vp, _i64]),
    "vb_table_rows": (_i64, [_vp]),
    "vb_table_device_rows": (_vp, [_vp, C.POINTER(C.c_size_t)]),
    "vb_table_free": (_i, [_vp]),
    "vb_exact_topk": (_i, [_vp, _i, _vp, _i64, _i, _vp, _vp]),
    "vb_exact_topk_dev": (_i, [_vp, _i, _vp, _i64, _i, _vp, _vp]),
    "vb_table_rerank": (_i, [_vp, _i, _vp, _i64, _vp, _i, _i, _vp, _vp]),
    "vb_table_rerank_dev": (_i, [_vp, _i, _vp, _i64, _vp, _i, _i, _vp, _vp]),
    "vb_table_filter_create": (_i, [_vp, _vp, _i64, C.POINTER(_vp)]),
    "vb_table_filter_create_dev": (_i, [_vp, _vp, _i64, C.POINTER(_vp)]),
    "vb_ivf_filter_create": (_i, [_vp, _vp, _i64, C.POINTER(_vp)]),
    "vb_ivf_filter_create_dev": (_i, [_vp, _vp, _i64, C.POINTER(_vp)]),
    "vb_filter_rows": (_i64, [_vp]),
    "vb_filter_free": (_i, [_vp]),
    "vb_exact_topk_filtered": (_i, [_vp, _i, _vp, _i64, _i, _vp, _i, _vp, _vp, _vp]),
    "vb_exact_topk_filtered_dev": (_i, [_vp, _i, _vp, _i64, _i, _vp, _i, _vp, _vp, _vp]),
    "vb_table_aggregate": (_i, [_vp, _i, _vp, _i, _i64, _vp, _vp, _vp]),
    "vb_table_aggregate_dev": (_i, [_vp, _i, _vp, _i, _i64, _vp, _vp, _vp]),
    "vb_table_order_create": (_i, [_vp, C.POINTER(_vp)]),
    "vb_sparse_table_order_create": (_i, [_vp, C.POINTER(_vp)]),
    "vb_order_rows": (_i64, [_vp]),
    "vb_order_groups": (_i64, [_vp]),
    "vb_order_passes": (_i64, [_vp]),
    "vb_order_read": (_i, [_vp, _vp, _vp, _vp]),
    "vb_order_read_dev": (_i, [_vp, _vp, _vp, _vp]),
    "vb_order_bounds": (_i, [_vp, _vp, _i64, _vp, _vp]),
    "vb_order_bounds_dev": (_i, [_vp, _vp, _i64, _vp, _vp]),
    "vb_sparse_order_bounds": (_i, [_vp, _i, _i64, _vp, _vp, _vp, _vp, _vp]),
    "vb_sparse_order_bounds_dev": (_i, [_vp, _i, _i64, _vp, _vp, _vp, _vp, _vp]),
    "vb_order_free": (_i, [_vp]),
    "vb_ivf_create": (_i, [_i, _i, _i, _i, C.POINTER(_vp)]),
    "vb_ivf_load": (_i, [_vp, _vp, _vp, _vp, _vp]),
    "vb_ivf_load_dev": (_i, [_vp, _vp, _vp, _vp, _vp]),
    "vb_ivf_rows": (_i64, [_vp]),
    "vb_ivf_begin_load": (_i, [_vp, _vp]),
    "vb_ivf_load_list": (_i, [_vp, _i, _vp, _vp, _i64]),
    "vb_ivf_end_load": (_i, [_vp]),
    "vb_ivf_replace_list": (_i, [_vp, _i, _vp, _vp, _i64]),
    "vb_ivf_insert": (_i, [_vp, _vp, _vp, _i64, _vp]),
    "vb_ivf_insert_dev": (_i, [_vp, _vp, _vp, _i64, _vp]),
    "vb_ivf_delete": (_i, [_vp, _vp, _i64, C.POINTER(_i64)]),
    "vb_ivf_list_offsets": (_i, [_vp, _vp]),
    "vb_ivf_build": (_i, [_vp, _vp, _vp, _i64, _i, _vp, _vp, _vp, C.POINTER(_i)]),
    "vb_ivf_build_dev": (_i, [_vp, _vp, _vp, _i64, _i, _vp, _vp, _vp, C.POINTER(_i)]),
    "vb_ivf_centers": (_i, [_vp, _vp]),
    "vb_ivf_free": (_i, [_vp]),
    "vb_ivf_scan_lists": (_i, [_vp, _vp, _i64, _i, _vp, _vp]),
    "vb_ivf_scan_items": (_i, [_vp, _vp, _vp, _i, _i64, _vp, _vp, _vp]),
    "vb_ivf_search": (_i, [_vp, _vp, _i64, _i, _i, _vp, _vp]),
    "vb_ivf_search_dev": (_i, [_vp, _vp, _i64, _i, _i, _vp, _vp]),
    "vb_ivf_search_filtered": (_i, [_vp, _vp, _i64, _i, _i, _vp, _i, _vp, _vp, _vp]),
    "vb_ivf_search_filtered_dev": (_i, [_vp, _vp, _i64, _i, _i, _vp, _i, _vp, _vp, _vp]),
    "vb_ivf_scan_begin": (_i, [_vp, _vp, _i64, _i, _i, _i, C.POINTER(_vp)]),
    "vb_ivf_scan_begin_filtered": (_i, [_vp, _vp, _i64, _i, _i, _i, _vp, _i, _vp, C.POINTER(_vp)]),
    "vb_ivf_scan_next": (_i, [_vp, _vp, _vp, _vp]),
    "vb_ivf_scan_lists_done": (_i, [_vp, _vp]),
    "vb_ivf_scan_end": (_i, [_vp]),
    "vb_ivf_prefetch_queries": (_i, [_vp, _vp, _i64, _i]),
    "vb_ivf_search_prefetched": (_i, [_vp, _i, _i, _i, _vp, _vp]),
    "vb_ivf_last_scan_bytes": (_i64, [_vp]),
    "vb_ivf_last_candidates": (_i64, [_vp]),
    "vb_ivf_tc_fallbacks": (_i64, [_vp]),
    "vb_ivf_tc_traffic": (_i, [_i, _vp]),
    "vb_ivf_tc_level0_rescored": (_i, [_vp]),
    "vb_ivf_search_sharded_dev": (_i, [_vp, _vp, _i64, _i, _i, _vp, _vp]),
    "vb_ivf_search_sharded": (_i, [_vp, _vp, _i64, _i, _i, _vp, _vp]),
    "vb_exact_topk_sharded_dev": (_i, [_vp, _i, _vp, _i64, _i, _i64, _vp, _vp]),
    "vb_comm_unique_id": (_i, [_vp, C.c_size_t]),
    "vb_comm_init": (_i, [_vp, _i, _i]),
    "vb_comm_free": (_i, []),
    "vb_comm_world": (_i, []),
    "vb_comm_rank": (_i, []),
    "vb_comm_allreduce": (_i, [_vp, _i64, _i]),
    "vb_comm_allgather": (_i, [_vp, _vp, _i64]),
    "vb_ivf_tc_level1_fallbacks": (_i64, [_vp]),
    "vb_ivf_tc_level0_fallbacks": (_i64, [_vp]),
    "vb_ivf_tc_levelp_fallbacks": (_i64, [_vp]),
    "vb_kmeans": (_i, [_vp, _i, _vp, _i, _i, _u64, _vp, _vp, _vp]),
    "vb_kmeans_pp_init": (_i, [_vp, _i, _vp, _i, _u64]),
    "vb_kmeans_pp_stats": (_i, [_vp]),
    "vb_kmeans_pp_init_draws": (_i, [_vp, _i, _vp, _i, _i64, _vp, _vp]),
    "vb_assign": (_i, [_vp, _i, _vp, _i, _vp]),
    "vb_assign_dev": (_i, [_vp, _i, _vp, _i, _vp]),
    "vb_set_tensor_cores": (_i, [_i]),
    "vb_last_assign_rechecked": (_i64, []),
    "vb_set_option": (_i, [C.c_char_p, _i64]),
    "vb_hnsw_create": (_i, [_i, _i, _i, _i, C.POINTER(_vp)]),
    "vb_hnsw_load": (_i, [_vp, _vp, _i64, _vp, _vp, _vp, _vp, _i64, _i64]),
    "vb_hnsw_free": (_i, [_vp]),
    "vb_hnsw_build": (_i, [_vp, _vp, _i64, _i, _u64, _vp]),
    "vb_hnsw_build_dev": (_i, [_vp, _vp, _i64, _i, _u64, _vp]),
    "vb_hnsw_insert": (_i, [_vp, _vp, _i64, _i, _u64, _vp, _vp, C.POINTER(_i64)]),
    "vb_hnsw_insert_dev": (_i, [_vp, _vp, _i64, _i, _u64, _vp, _vp, C.POINTER(_i64)]),
    "vb_hnsw_insert_changes": (_i, [_vp, _vp, _i64]),
    "vb_hnsw_set_heaptid_counts": (_i, [_vp, _vp]),
    "vb_hnsw_vacuum": (_i, [_vp, _vp, _i, C.POINTER(_i64), C.POINTER(_i64)]),
    "vb_hnsw_rows": (_i64, [_vp]),
    "vb_hnsw_upper_slots": (_i64, [_vp]),
    "vb_hnsw_export": (_i, [_vp, _vp, _vp, _vp, _vp, C.POINTER(_i64), _vp]),
    "vb_hnsw_search": (_i, [_vp, _vp, _i64, _i, _i, _vp, _vp, _vp]),
    "vb_hnsw_search_dev": (_i, [_vp, _vp, _i64, _i, _i, _vp, _vp, _vp]),
    "vb_hnsw_scan_begin": (_i, [_vp, _vp, _i64, _i, _i64, C.POINTER(_vp)]),
    "vb_hnsw_scan_next": (_i, [_vp, _vp, _vp, _vp]),
    "vb_hnsw_scan_tuples": (_i, [_vp, _vp]),
    "vb_hnsw_scan_end": (_i, [_vp]),
    "vb_hnsw_filter_create": (_i, [_vp, _vp, _i64, C.POINTER(_vp)]),
    "vb_hnsw_filter_create_dev": (_i, [_vp, _vp, _i64, C.POINTER(_vp)]),
    "vb_hnsw_scan_begin_filtered": (_i, [_vp, _vp, _i64, _i, _i64, _i, _vp, _i, _vp, C.POINTER(_vp)]),
}


class IvfBuildOpts(C.Structure):
    """vb_ivf_build_opts"""
    _fields_ = [("seed", _u64), ("max_iter", _i), ("sample_rows", _vp), ("n_samples", _i64), ("first_row", _i64), ("u", _vp),
                ("chunk_rows", _i64)]


class TextInputError(ValueError):
    """a type input error: the reference's errmsg, with its errdetail (.detail, "" when none) and the failing
    literal's index (.row)"""

    def __init__(self, msg, detail, row):
        super().__init__(msg)
        self.detail = detail
        self.row = row


class VecB200Error(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"libvecb200 error {code}: {msg}")
        self.code = code


_lib = None


def load() -> C.CDLL:
    """dlopen the in-tree library and declare every prototype.  Raises if it was not built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                f"{LIB_PATH} is missing: build it with `python -m pgvector_b200.build` "
                "(there is no CPU fallback for the distance hot path)")
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)      # AttributeError here = ABI mismatch, fail loudly
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


def check(rc: int):
    if rc != OK:
        msg = load().vb_last_error()
        raise VecB200Error(rc, msg.decode() if msg else "")
