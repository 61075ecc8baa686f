"""ctypes binding of librxgpu.so (C ABI: include/rxgpu.h).

Python is only the test / benchmark / multi-GPU driver here; the product is the C-ABI library plus the C++ adapter
(reindexer_b200/host/gpu_bruteforce.h).  Method names follow the reference's ``Map`` duck-type
(hnswlib::BruteforceSearch, cpp_src/core/index/float_vector/hnswlib/bruteforce.h).  There is no CPU fallback: every
compute call raises RxGpuError when the CUDA extension or a device is missing.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "librxgpu.so")

L2, IP, COS = 0, 1, 2
FLAG_HOST_MIRROR = 1

_f32p = C.POINTER(C.c_float)
_u64p = C.POINTER(C.c_uint64)
_u32p = C.POINTER(C.c_uint32)
_i32p = C.POINTER(C.c_int32)
_u8p = C.POINTER(C.c_uint8)


class RxGpuError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"[{code}] {msg}")
        self.code = code
        self.what = msg


class SelectParams(C.Structure):
    _fields_ = [("k", C.c_uint32), ("has_radius", C.c_int), ("radius", C.c_float), ("need_sort", C.c_int), ("is_array", C.c_int),
                ("raw", C.c_int)]


class HnswNodeUpdate(C.Structure):
    _fields_ = [("node", C.c_uint32), ("level", C.c_int32), ("level0", C.c_void_p), ("upper", C.c_void_p), ("vec", C.c_void_p),
                ("label", C.c_uint64), ("deleted", C.c_int)]


class HnswGraph(C.Structure):
    _fields_ = [("n", C.c_uint32), ("M", C.c_uint32), ("maxM0", C.c_uint32), ("maxlevel", C.c_int32), ("enterpoint", C.c_uint32),
                ("upper_slots", C.c_uint64), ("level0", C.c_void_p), ("levels", C.c_void_p), ("upper_offsets", C.c_void_p),
                ("upper", C.c_void_p)]


class FtPostings(C.Structure):
    _fields_ = [("ndocs", C.c_uint32), ("doc_ids", _u32p), ("pos_begin", _u32p), ("positions", _u32p)]


class FtFieldConfig(C.Structure):
    _fields_ = [("bm25_boost", C.c_double), ("bm25_weight", C.c_double), ("term_len_boost", C.c_double), ("term_len_weight", C.c_double),
                ("position_boost", C.c_double), ("position_weight", C.c_double)]


class FtConfig(C.Structure):
    _fields_ = [("merge_limit", C.c_uint32), ("min_rank", C.c_int32), ("bm25_k1", C.c_double), ("bm25_b", C.c_double),
                ("bm25_type", C.c_int32), ("distance_boost", C.c_double), ("distance_weight", C.c_double),
                ("full_match_boost", C.c_double), ("nfields", C.c_uint32), ("fields", C.POINTER(FtFieldConfig)),
                ("summation_ranks_by_fields_ratio", C.c_double)]


class FtTerm(C.Structure):
    _fields_ = [("op", C.c_int32), ("boost", C.c_float), ("term_len_boost", C.c_float), ("field_boosts", _f32p), ("nsubterms", C.c_uint32),
                ("postings", _u32p), ("procs", _f32p), ("need_sum_rank", _u8p), ("suppressed", _u8p), ("nsynonyms", C.c_uint32),
                ("synonym_ids", _u32p), ("phrase_num", C.c_int32), ("distance", C.c_int32)]


class FtSynonym(C.Structure):
    _fields_ = [("nterms", C.c_uint32), ("terms", C.POINTER(FtTerm))]


class FtQuery(C.Structure):
    _fields_ = [("nterms", C.c_uint32), ("terms", C.POINTER(FtTerm)), ("nsynonyms", C.c_uint32), ("synonyms", C.POINTER(FtSynonym))]


class Sq8Params(C.Structure):
    _fields_ = [("min_q", C.c_float), ("max_q", C.c_float), ("alpha", C.c_float), ("alpha_2", C.c_float), ("delta", C.c_float)]


class FtStats(C.Structure):
    _fields_ = [("launches", C.c_uint32), ("preselected", C.c_uint32), ("postings_scanned", C.c_uint64), ("algorithmic_bytes", C.c_uint64),
                ("device_ms", C.c_float)]


FT_MERGE_INFO_DTYPE = np.dtype([("id", np.int32), ("proc", np.float32), ("field", np.uint8), ("normalized_proc", np.uint8)], align=True)


class IvfTrainParams(C.Structure):
    _fields_ = [("niter", C.c_int32), ("seed", C.c_int32), ("max_points_per_centroid", C.c_int32)]


class IvfTrainStats(C.Structure):
    _fields_ = [("obj", C.c_double), ("nsplit", C.c_int32), ("assign_ms", C.c_float), ("update_ms", C.c_float), ("host_ms", C.c_float)]


class HnswBuildStats(C.Structure):
    _fields_ = [("batches", C.c_uint64), ("rows", C.c_uint64), ("distances", C.c_uint64), ("reverse_links", C.c_uint64),
                ("lists_pruned", C.c_uint64), ("search_select_ms", C.c_float), ("sort_ms", C.c_float), ("link_ms", C.c_float)]


class SearchStats(C.Structure):
    _fields_ = [("launches", C.c_uint32), ("passes", C.c_uint32), ("query_tile", C.c_uint32), ("tie_replays", C.c_uint32), ("tie_from_lists", C.c_uint32),
                ("algorithmic_bytes", C.c_uint64), ("scan_launches", C.c_uint32), ("scan_kernel_ms", C.c_float),
                ("tc_used", C.c_uint32), ("tc_fallbacks", C.c_uint32), ("tc_candidates", C.c_uint64), ("tc_cluster", C.c_uint32), ("tc_kernel", C.c_uint32)]


# every symbol include/rxgpu.h declares (checked by tests/test_abi.py against the header text)
_SIGNATURES = {
    "rxgpu_last_error": (C.c_char_p, []),
    "rxgpu_abi_version": (C.c_int, []),
    "rxgpu_device_count": (C.c_int, []),
    "rxgpu_index_create": (C.c_int, [C.POINTER(C.c_void_p), C.c_int, C.c_uint32, C.c_uint64, C.c_int, C.c_uint32]),
    "rxgpu_index_clone": (C.c_int, [C.POINTER(C.c_void_p), C.c_void_p, C.c_uint64]),
    "rxgpu_index_destroy": (None, [C.c_void_p]),
    "rxgpu_index_resize": (C.c_int, [C.c_void_p, C.c_uint64]),
    "rxgpu_index_upsert": (C.c_int, [C.c_void_p, C.c_uint64, _f32p]),
    "rxgpu_index_upsert_batch": (C.c_int, [C.c_void_p, C.c_uint64, _u64p, _f32p]),
    "rxgpu_index_remove": (C.c_int, [C.c_void_p, C.c_uint64]),
    "rxgpu_index_get": (C.c_int, [C.c_void_p, C.c_uint64, C.POINTER(_f32p)]),
    "rxgpu_index_size": (C.c_uint64, [C.c_void_p]),
    "rxgpu_index_capacity": (C.c_uint64, [C.c_void_p]),
    "rxgpu_index_element_size": (C.c_uint64, [C.c_void_p]),
    "rxgpu_index_device_bytes": (C.c_uint64, [C.c_void_p]),
    "rxgpu_index_dim": (C.c_uint32, [C.c_void_p]),
    "rxgpu_index_metric": (C.c_int, [C.c_void_p]),
    "rxgpu_index_device": (C.c_int, [C.c_void_p]),
    "rxgpu_search_knn": (C.c_int, [C.c_void_p, C.c_uint32, _f32p, C.c_uint32, _f32p, _u64p, _u32p]),
    "rxgpu_search_range": (C.c_int, [C.c_void_p, _f32p, C.c_float, C.c_uint64, _f32p, _u64p, _u64p]),
    "rxgpu_search_range_batch": (C.c_int, [C.c_void_p, C.c_uint32, _f32p, _f32p, C.c_uint64, _f32p, _u64p, _u64p]),
    "rxgpu_last_range_results": (C.c_int, [C.c_uint64, C.c_uint64, _f32p, _u64p]),
    "rxgpu_comm_unique_id": (C.c_int, [C.c_void_p]),
    "rxgpu_comm_create": (C.c_int, [C.POINTER(C.c_void_p), C.c_int, C.c_int, C.c_void_p, C.c_int]),
    "rxgpu_comm_destroy": (None, [C.c_void_p]),
    "rxgpu_comm_rank": (C.c_int, [C.c_void_p]),
    "rxgpu_comm_size": (C.c_int, [C.c_void_p]),
    "rxgpu_sharded_search_knn": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_int, C.c_uint32, _f32p, _u64p, _u32p]),
    "rxgpu_sharded_search_range_batch": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_int, _f32p, C.c_uint64, _f32p, _u64p,
                                                   _u64p]),
    "rxgpu_shard_payload_bytes": (C.c_uint64, [C.c_uint32, C.c_uint32]),
    "rxgpu_merge_shards_device": (C.c_int, [C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                            C.c_void_p, C.c_void_p, C.c_void_p]),
    "rxgpu_search_knn_device": (C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.c_void_p]),
    "rxgpu_search_tie_rows_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_float, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p,
                                               C.c_void_p, C.c_void_p]),
    "rxgpu_merge_shards": (C.c_int, [C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, _f32p, _u32p, _u64p, _u32p, _u64p, _f32p, _u64p,
                                     _u64p, _u32p, _u8p]),
    "rxgpu_tie_replay": (C.c_int, [C.c_uint32, C.c_float, C.c_uint32, _f32p, _u64p, _u64p, C.c_uint32, _f32p, _u64p, _u64p, _f32p,
                                   _u64p, _u32p]),
    "rxgpu_select_knn": (C.c_int, [C.c_void_p, _f32p, C.POINTER(SelectParams), C.c_uint64, _i32p, _f32p, _u64p]),
    "rxgpu_select_postprocess": (C.c_int, [C.c_int, C.POINTER(SelectParams), C.c_uint64, _f32p, _u64p, _i32p, _f32p, _u64p]),
    "rxgpu_hnsw_import": (C.c_int, [C.c_void_p, C.POINTER(HnswGraph)]),
    "rxgpu_hnsw_search_knn": (C.c_int, [C.c_void_p, C.c_uint32, _f32p, C.c_uint32, C.c_uint32, _f32p, _u64p, _u32p, _u32p]),
    "rxgpu_hnsw_mark_deleted": (C.c_int, [C.c_void_p, C.c_uint64]),
    "rxgpu_hnsw_deleted_count": (C.c_uint64, [C.c_void_p]),
    "rxgpu_gather_labels_device": (C.c_int, [C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p]),
    "rxgpu_hnsw_search_range": (C.c_int, [C.c_void_p, _f32p, C.c_float, C.c_uint32, C.c_uint64, _f32p, _u64p, C.POINTER(C.c_uint64)]),
    "rxgpu_hnsw_search_range_batch": (C.c_int, [C.c_void_p, C.c_uint32, _f32p, _f32p, C.c_uint32, C.c_uint64, _f32p, _u64p, _u64p]),
    "rxgpu_hnsw_build": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint64, _i32p, C.c_uint64, C.POINTER(HnswBuildStats)]),
    "rxgpu_hnsw_build_plan": (C.c_int, [C.c_uint32, C.c_uint64, C.c_uint64, C.c_int32, _i32p, C.c_uint64, _i32p, _u64p, C.POINTER(C.c_uint64)]),
    "rxgpu_hnsw_export": (C.c_int, [C.c_void_p, C.c_uint64, _u32p, _u32p, _i32p, C.POINTER(C.c_int64), _u32p, C.POINTER(HnswGraph)]),
    "rxgpu_hnsw_search_knn_device": (C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p,
                                               C.c_void_p, C.c_void_p, C.c_void_p]),
    "rxgpu_ivf_create": (C.c_int, [C.c_void_p, C.c_uint32, _f32p]),
    "rxgpu_ivf_add": (C.c_int, [C.c_void_p, C.c_uint64, _u32p, _u64p, _f32p]),
    "rxgpu_ivf_remove": (C.c_int, [C.c_void_p, C.c_uint64]),
    "rxgpu_ivf_size": (C.c_uint64, [C.c_void_p]),
    "rxgpu_ivf_list_stats": (C.c_int, [C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    "rxgpu_hnsw_load_index_cache": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "rxgpu_hnsw_update": (C.c_int, [C.c_void_p, C.c_int32, C.c_uint32, C.c_uint32, C.c_void_p]),
    "rxgpu_hnsw_update_count": (C.c_uint64, [C.c_void_p]),
    "rxgpu_hnsw_stream_begin": (C.c_int, [C.c_void_p, _f32p, C.c_uint32, C.POINTER(C.c_void_p)]),
    "rxgpu_hnsw_stream_next": (C.c_int, [C.c_void_p, C.c_uint32, _f32p, _u64p, _u32p, C.POINTER(C.c_int)]),
    "rxgpu_hnsw_stream_end": (None, [C.c_void_p]),
    "rxgpu_sq8_attach": (C.c_int, [C.c_void_p, C.POINTER(Sq8Params), _u8p, _f32p]),
    "rxgpu_sq8_export": (C.c_int, [C.c_void_p, _u8p, _f32p]),
    "rxgpu_sq8_prepare_query": (C.c_int, [C.c_void_p, _f32p, C.c_float, _u8p, _f32p]),
    "rxgpu_sq8_search_knn": (C.c_int, [C.c_void_p, C.c_uint32, _f32p, _f32p, C.c_uint32, _f32p, _u64p, _u32p]),
    "rxgpu_hnsw_search_knn_sq8": (C.c_int, [C.c_void_p, C.c_uint32, _f32p, _f32p, C.c_uint32, C.c_uint32, _f32p, _u64p, _u32p, _u32p]),
    "rxgpu_ivf_import": (C.c_int, [C.c_void_p, C.c_uint32, _f32p, _u64p]),
    "rxgpu_ivf_train": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint64, _f32p, _f32p, C.POINTER(IvfTrainParams), _f32p, C.POINTER(IvfTrainStats)]),
    "rxgpu_ivf_assign": (C.c_int, [C.c_void_p, C.c_uint64, _f32p, _f32p, _u32p, _f32p]),
    "rxgpu_ivf_add_assign": (C.c_int, [C.c_void_p, C.c_uint64, _u64p, _f32p, _f32p, _u32p]),
    "rxgpu_kmeans_plan": (C.c_int, [C.c_uint64, C.c_uint32, C.c_int32, C.c_int32, _i32p, _i32p]),
    "rxgpu_ivf_search_knn": (C.c_int, [C.c_void_p, C.c_uint32, _f32p, C.c_uint32, C.c_uint32, _f32p, _u64p, _u32p]),
    "rxgpu_ivf_search_knn_large_k": (C.c_int, [C.c_void_p, C.c_uint32, _f32p, C.c_uint32, C.c_uint32, _f32p, _u64p, _u32p]),
    "rxgpu_ivf_search_range": (C.c_int, [C.c_void_p, _f32p, C.c_float, C.c_uint32, C.c_uint64, _f32p, _u64p, C.POINTER(C.c_uint64)]),
    "rxgpu_ivf_search_range_batch": (C.c_int, [C.c_void_p, C.c_uint32, _f32p, _f32p, C.c_uint32, C.c_uint64, _f32p, _u64p, _u64p]),
    "rxgpu_ft_create": (C.c_int, [C.POINTER(C.c_void_p), C.c_uint32, C.c_uint32, _u32p, _f32p, _u8p, C.c_int]),
    "rxgpu_ft_destroy": (None, [C.c_void_p]),
    "rxgpu_ft_add_postings": (C.c_int, [C.c_void_p, C.POINTER(FtPostings), _u32p]),
    "rxgpu_ft_add_postings_packed": (C.c_int, [C.c_void_p, _u8p, C.c_uint64, C.c_uint32, _u32p]),
    "rxgpu_ft_decode_packed": (C.c_int, [_u8p, C.c_uint64, C.c_uint32, _u32p, _u32p, _u32p, C.c_uint64, C.POINTER(C.c_uint64)]),
    "rxgpu_ft_merge": (C.c_int, [C.c_void_p, C.POINTER(FtConfig), C.c_uint32, C.POINTER(FtTerm), _u8p, C.c_int, C.c_uint64, C.c_void_p,
                                 C.POINTER(C.c_uint64)]),
    "rxgpu_ft_add_postings_packed_batch": (C.c_int, [C.c_void_p, C.c_uint32, C.POINTER(C.c_void_p), C.POINTER(C.c_uint64), _u32p, _u32p]),
    "rxgpu_ft_merge_query": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, _u8p, C.c_int, C.c_uint64, C.c_void_p, C.POINTER(C.c_uint64)]),
    "rxgpu_ft_merge_query_areas": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, _u8p, C.c_int, C.c_int32, C.c_uint64, C.c_void_p, _u32p,
                                              C.c_void_p, _u32p, C.POINTER(C.c_uint64)]),
    "rxgpu_ft_select_query": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, _u8p, _u8p, C.c_int, C.c_uint64, _i32p, _f32p,
                                         C.POINTER(C.c_uint64)]),
    "rxgpu_ft_set_rows": (C.c_int, [C.c_void_p, _u32p, _i32p]),
    "rxgpu_sharded_ft_select": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint32, C.POINTER(FtConfig), C.c_uint32, C.POINTER(FtTerm), _u8p, _u8p,
                                           C.c_int, C.c_uint64, _i32p, _f32p, C.POINTER(C.c_uint64)]),
    "rxgpu_comm_create_local": (C.c_int, [C.POINTER(C.c_void_p), C.c_int, C.POINTER(C.c_int)]),
    "rxgpu_sharded_ivf_train": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint64, _f32p, _f32p, C.POINTER(IvfTrainParams), _f32p,
                                          C.POINTER(IvfTrainStats)]),
    "rxgpu_sharded_ivf_search_knn": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_int, C.c_uint32, C.c_uint32, _f32p, _u64p,
                                               _u32p]),
    "rxgpu_sharded_ivf_search_range_batch": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_int, _f32p, C.c_uint32, C.c_uint64,
                                                       _f32p, _u64p, _u64p]),
    "rxgpu_ft_select": (C.c_int, [C.c_void_p, C.POINTER(FtConfig), C.c_uint32, C.POINTER(FtTerm), _u8p, _u8p, C.c_int, C.c_uint64, _i32p, _f32p,
                                  C.POINTER(C.c_uint64)]),
    "rxgpu_ft_last_stats": (None, [C.POINTER(FtStats)]),
    "rxgpu_index_append_synth": (C.c_int, [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64]),
    "rxgpu_synth_fill_device": (C.c_int, [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64, C.c_int, C.c_void_p]),
    "rxgpu_set_query_tile": (C.c_int, [C.c_void_p, C.c_uint32]),
    "rxgpu_last_search_stats": (None, [C.POINTER(SearchStats)]),
    "rxgpu_set_profile": (C.c_int, [C.c_int]),
    "rxgpu_tc_diag": (C.c_int, [C.c_int, C.c_void_p]),
    "rxgpu_tc_audit": (C.c_int, [C.c_void_p, C.c_uint32, _f32p, _f32p, C.c_uint32, _u32p, _u32p, _f32p, _f32p, C.c_void_p, C.c_void_p, _f32p,
                                 _f32p, _i32p, _f32p]),
    "rxgpu_set_tensor_core_filter": (C.c_int, [C.c_void_p, C.c_int]),
}

_lib = None


def lib():
    """Load librxgpu.so; fails loudly when it has not been built (``python -c 'import __graft_entry__ as g; g.build()'``)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RxGpuError(37, f"{LIB_PATH} is missing: build the CUDA extension first (no CPU fallback exists)")
        l = C.CDLL(LIB_PATH)
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(l, name)
            fn.restype = res
            fn.argtypes = args
        _lib = l
    return _lib


def _check(rc):
    if rc != 0:
        raise RxGpuError(rc, lib().rxgpu_last_error().decode(errors="replace"))


def _p(a, t):
    return a.ctypes.data_as(t)


def device_count() -> int:
    return lib().rxgpu_device_count()


def last_search_stats() -> dict:
    s = SearchStats()
    lib().rxgpu_last_search_stats(C.byref(s))
    return {f: getattr(s, f) for f, _ in SearchStats._fields_}


class GpuBruteforceSearch:
    """One shard of a float_vector brute-force index resident in the HBM of one GPU."""

    def __init__(self, metric: int, dim: int, capacity: int, device: int = 0, host_mirror: bool = False, _handle=None):
        self._lib = lib()
        self.metric, self.dim = metric, dim
        if _handle is not None:
            self._h = _handle
            return
        h = C.c_void_p()
        _check(self._lib.rxgpu_index_create(C.byref(h), metric, dim, capacity, device, FLAG_HOST_MIRROR if host_mirror else 0))
        self._h = h

    def close(self):
        if getattr(self, "_h", None):
            self._lib.rxgpu_index_destroy(self._h)
            self._h = None

    __del__ = close

    # -- BruteforceSearch surface ------------------------------------------------------------------------------------
    def clone(self, new_capacity: int) -> "GpuBruteforceSearch":
        h = C.c_void_p()
        _check(self._lib.rxgpu_index_clone(C.byref(h), self._h, new_capacity))
        return GpuBruteforceSearch(self.metric, self.dim, new_capacity, _handle=h)

    def max_elements(self) -> int:
        return self._lib.rxgpu_index_capacity(self._h)

    def current_element_count(self) -> int:
        return self._lib.rxgpu_index_size(self._h)

    size = current_element_count

    def element_size(self) -> int:
        return self._lib.rxgpu_index_element_size(self._h)

    def device_bytes(self) -> int:
        return self._lib.rxgpu_index_device_bytes(self._h)

    def add_point(self, vec, label: int):
        vec = np.ascontiguousarray(vec, dtype=np.float32)
        assert vec.size == self.dim
        _check(self._lib.rxgpu_index_upsert(self._h, label, _p(vec, _f32p)))

    def add_points(self, labels, vecs):
        vecs = np.ascontiguousarray(vecs, dtype=np.float32)
        labels = np.ascontiguousarray(labels, dtype=np.uint64)
        assert vecs.shape == (len(labels), self.dim)
        _check(self._lib.rxgpu_index_upsert_batch(self._h, len(labels), _p(labels, _u64p), _p(vecs, _f32p)))

    def remove_point(self, label: int):
        _check(self._lib.rxgpu_index_remove(self._h, label))

    def resize_index(self, new_capacity: int):
        _check(self._lib.rxgpu_index_resize(self._h, new_capacity))

    def float_ptr_by_external_label(self, label: int) -> np.ndarray:
        p = _f32p()
        _check(self._lib.rxgpu_index_get(self._h, label, C.byref(p)))
        return np.ctypeslib.as_array(p, (self.dim,)).copy()

    def search_knn(self, queries, k: int):
        """queries: [nq, dim] (or [dim]); returns (dists [nq,k], labels [nq,k], counts [nq]) best-first, map-space sign."""
        q = np.ascontiguousarray(queries, dtype=np.float32)
        single = q.ndim == 1
        q = q.reshape(-1, self.dim)
        nq = q.shape[0]
        d = np.zeros((nq, max(k, 1)), np.float32)
        l = np.zeros((nq, max(k, 1)), np.uint64)
        c = np.zeros(nq, np.uint32)
        _check(self._lib.rxgpu_search_knn(self._h, nq, _p(q, _f32p), k, _p(d, _f32p), _p(l, _u64p), _p(c, _u32p)))
        if single:
            return d[0, :c[0]], l[0, :c[0]]
        return d[:, :k], l[:, :k], c

    def search_range(self, query, radius: float, max_out: int | None = None):
        q = np.ascontiguousarray(query, dtype=np.float32)
        max_out = self.size() if max_out is None else max_out
        d = np.zeros(max(max_out, 1), np.float32)
        l = np.zeros(max(max_out, 1), np.uint64)
        n = C.c_uint64(0)
        _check(self._lib.rxgpu_search_range(self._h, _p(q, _f32p), radius, max_out, _p(d, _f32p), _p(l, _u64p), C.byref(n)))
        m = min(n.value, max_out)
        return d[:m], l[:m], n.value

    def search_range_batch(self, queries, radius, max_out: int | None = None):
        """queries: [nq, dim]; radius: a scalar or [nq] (map space, as search_range).  Returns (dists [nq, max_out],
        labels [nq, max_out], counts [nq]): row q holds the best min(counts[q], max_out) matches of query q, best-first, and
        counts[q] is its total number of matches.  max_out defaults to the row count, at most 131072 (the largest that still
        sizes the filter's candidate lists by it)."""
        q = np.ascontiguousarray(queries, dtype=np.float32).reshape(-1, self.dim)
        nq = q.shape[0]
        r = np.ascontiguousarray(np.broadcast_to(np.asarray(radius, dtype=np.float32), (nq,)))
        max_out = min(self.size(), 1 << 17) if max_out is None else max_out
        d = np.zeros((nq, max(max_out, 1)), np.float32)
        l = np.zeros((nq, max(max_out, 1)), np.uint64)
        c = np.zeros(nq, np.uint64)
        _check(self._lib.rxgpu_search_range_batch(self._h, nq, _p(q, _f32p), _p(r, _f32p), max_out, _p(d, _f32p), _p(l, _u64p),
                                                  _p(c, _u64p)))
        return d[:, :max_out], l[:, :max_out], c

    def select(self, query, k: int | None = None, radius: float | None = None, need_sort=True, is_array=False, raw=False,
               max_out: int | None = None):
        """FloatVectorIndex::Select equivalent: returns (row_ids int32, ranks float32)."""
        q = np.ascontiguousarray(query, dtype=np.float32)
        prm = SelectParams(k or 0, int(radius is not None), float(radius or 0.0), int(need_sort), int(is_array), int(raw))
        max_out = max_out if max_out is not None else max(self.size(), 1)
        ids = np.zeros(max_out, np.int32)
        ranks = np.zeros(max_out, np.float32)
        n = C.c_uint64(0)
        _check(self._lib.rxgpu_select_knn(self._h, _p(q, _f32p), C.byref(prm), max_out, _p(ids, _i32p), _p(ranks, _f32p), C.byref(n)))
        m = min(n.value, max_out)
        return ids[:m], ranks[:m]

    # -- device-resident entry points ----------------------------------------------------------------------------------
    def search_knn_device(self, nq, d_queries_ptr, k1, d_dist_ptr, d_idx_ptr, d_label_ptr, d_count_ptr, stream=0):
        _check(self._lib.rxgpu_search_knn_device(self._h, nq, d_queries_ptr, k1, d_dist_ptr, d_idx_ptr, d_label_ptr, d_count_ptr,
                                                 stream or None))

    def search_tie_rows_device(self, d_query_ptr, dstar, k, d_dist_ptr, d_idx_ptr, d_label_ptr, d_count_ptr, stream=0):
        _check(self._lib.rxgpu_search_tie_rows_device(self._h, d_query_ptr, dstar, k, d_dist_ptr, d_idx_ptr, d_label_ptr, d_count_ptr,
                                                      stream or None))

    # -- HNSW (graph built by the reference's CPU code, searched on the device) ---------------------------------------
    def hnsw_import(self, graph: dict):
        """graph: arrays as produced by the reference's graph (level0 [n,1+maxM0] u32, levels [n] i32, upper_offsets [n+1] i64,
        upper [slots,1+M] u32) plus n / M / maxM0 / maxlevel / enterpoint; internal id i must be row i of this index."""
        l0 = np.ascontiguousarray(graph["level0"], np.uint32)
        lv = np.ascontiguousarray(graph["levels"], np.int32)
        uo = np.ascontiguousarray(graph["upper_offsets"], np.int64)
        up = np.ascontiguousarray(graph["upper"], np.uint32)
        g = HnswGraph(graph["n"], graph["M"], graph["maxM0"], graph["maxlevel"], graph["enterpoint"], len(up), l0.ctypes.data,
                      lv.ctypes.data, uo.ctypes.data, up.ctypes.data if len(up) else None)
        _check(self._lib.rxgpu_hnsw_import(self._h, C.byref(g)))

    def hnsw_search_knn(self, queries, k: int, ef: int = 0, with_stats=False):
        q = np.ascontiguousarray(queries, dtype=np.float32).reshape(-1, self.dim)
        nq = q.shape[0]
        d = np.zeros((nq, max(k, 1)), np.float32)
        l = np.zeros((nq, max(k, 1)), np.uint64)
        c = np.zeros(nq, np.uint32)
        st = np.zeros((nq, 2), np.uint32)
        _check(self._lib.rxgpu_hnsw_search_knn(self._h, nq, _p(q, _f32p), k, ef, _p(d, _f32p), _p(l, _u64p), _p(c, _u32p),
                                               _p(st, _u32p)))
        return (d, l, c, st) if with_stats else (d, l, c)

    def hnsw_build(self, M: int, ef_construction: int, first: int = 0, levels=None, seed: int = 100) -> dict:
        """Insert rows [first, size) into the device graph (rxgpu_hnsw_build); `first` = the graph's node count (0: no graph yet).
        levels: one per inserted row, or None to draw them like the reference's getRandomLevel.  Returns the build's stats."""
        lv = None if levels is None else np.ascontiguousarray(levels, np.int32)
        st = HnswBuildStats()
        _check(self._lib.rxgpu_hnsw_build(self._h, M, ef_construction, first, None if lv is None else _p(lv, _i32p), seed, C.byref(st)))
        return {f: getattr(st, f) for f, _ in HnswBuildStats._fields_}

    def hnsw_export(self, nodes=None) -> dict:
        """The device graph (rxgpu_hnsw_export) as a dict in the layout of hnsw_import: every node, or the nodes listed (their
        upper-level lists then follow one another, upper_offsets indexing them)."""
        info = HnswGraph()
        _check(self._lib.rxgpu_hnsw_export(self._h, 0, None, None, None, None, None, C.byref(info)))
        nd = None if nodes is None else np.ascontiguousarray(nodes, np.uint32)
        cnt = info.n if nd is None else len(nd)
        ndp = None if nd is None else _p(nd, _u32p)
        offs = np.zeros(cnt + 1, np.int64)
        levels = np.zeros(max(cnt, 1), np.int32)
        level0 = np.zeros((max(cnt, 1), 1 + info.maxM0), np.uint32)
        _check(self._lib.rxgpu_hnsw_export(self._h, cnt, ndp, _p(level0, _u32p), _p(levels, _i32p), offs.ctypes.data_as(C.POINTER(C.c_int64)),
                                           None, None))
        upper = np.zeros((max(int(offs[cnt]), 1), 1 + info.M), np.uint32)
        _check(self._lib.rxgpu_hnsw_export(self._h, cnt, ndp, None, None, None, _p(upper, _u32p), None))
        return dict(n=info.n, maxlevel=info.maxlevel, enterpoint=info.enterpoint, M=info.M, maxM0=info.maxM0, level0=level0[:cnt],
                    levels=levels[:cnt], upper_offsets=offs, upper=upper[:int(offs[cnt])])

    def ivf_create(self, centroids):
        c = np.ascontiguousarray(centroids, np.float32).reshape(-1, self.dim)
        _check(self._lib.rxgpu_ivf_create(self._h, len(c), _p(c, _f32p)))

    def ivf_add(self, list_nos, labels, vecs):
        ln = np.ascontiguousarray(list_nos, np.uint32)
        lb = np.ascontiguousarray(labels, np.uint64)
        v = np.ascontiguousarray(vecs, np.float32).reshape(-1, self.dim)
        assert len(ln) == len(lb) == len(v)
        _check(self._lib.rxgpu_ivf_add(self._h, len(ln), _p(ln, _u32p), _p(lb, _u64p), _p(v, _f32p)))

    def ivf_train(self, nlist: int, vecs, norm_coefs=None, niter: int = 10, seed: int = 1234, max_points_per_centroid: int = 256):
        """k-means on the device (rxgpu_ivf_train); leaves empty lists over the trained centroids, as ivf_create does.
        Returns (centroids [nlist, dim], per-iteration stats: a list of dicts obj / nsplit / assign_ms / update_ms / host_ms)"""
        v = np.ascontiguousarray(vecs, np.float32).reshape(-1, self.dim)
        nc = None if norm_coefs is None else np.ascontiguousarray(norm_coefs, np.float32)
        prm = IvfTrainParams(niter, seed, max_points_per_centroid)
        cent = np.zeros((max(nlist, 1), self.dim), np.float32)
        st = (IvfTrainStats * max(niter, 1))()
        _check(self._lib.rxgpu_ivf_train(self._h, nlist, len(v), _p(v, _f32p), None if nc is None else _p(nc, _f32p), C.byref(prm),
                                         _p(cent, _f32p), st))
        stats = [{f: getattr(st[i], f) for f, _ in IvfTrainStats._fields_} for i in range(max(niter, 0))]
        return cent[:nlist], stats

    def ivf_assign(self, vecs, norm_coefs=None):
        """quantizer->assign on the device (rxgpu_ivf_assign): (list numbers, distances in map space)"""
        v = np.ascontiguousarray(vecs, np.float32).reshape(-1, self.dim)
        nc = None if norm_coefs is None else np.ascontiguousarray(norm_coefs, np.float32)
        ln = np.zeros(max(len(v), 1), np.uint32)
        d = np.zeros(max(len(v), 1), np.float32)
        _check(self._lib.rxgpu_ivf_assign(self._h, len(v), _p(v, _f32p), None if nc is None else _p(nc, _f32p), _p(ln, _u32p), _p(d, _f32p)))
        return ln[:len(v)], d[:len(v)]

    def ivf_add_assign(self, labels, vecs, norm_coefs=None):
        """ivf_assign then ivf_add with those lists (rxgpu_ivf_add_assign), all or nothing; returns the list numbers"""
        lb = np.ascontiguousarray(labels, np.uint64)
        v = np.ascontiguousarray(vecs, np.float32).reshape(-1, self.dim)
        assert len(lb) == len(v)
        nc = None if norm_coefs is None else np.ascontiguousarray(norm_coefs, np.float32)
        ln = np.zeros(max(len(v), 1), np.uint32)
        _check(self._lib.rxgpu_ivf_add_assign(self._h, len(v), _p(lb, _u64p), _p(v, _f32p), None if nc is None else _p(nc, _f32p),
                                              _p(ln, _u32p)))
        return ln[:len(v)]

    def ivf_remove(self, label: int):
        _check(self._lib.rxgpu_ivf_remove(self._h, int(label)))

    def ivf_size(self) -> int:
        return int(self._lib.rxgpu_ivf_size(self._h))

    def ivf_list_stats(self) -> dict:
        v = [C.c_uint64(0) for _ in range(4)]
        _check(self._lib.rxgpu_ivf_list_stats(self._h, *[C.byref(x) for x in v]))
        return dict(zip(("slab_rows", "dead_rows", "relocations", "compactions"), (x.value for x in v)))

    def hnsw_update(self, graph: dict, nodes, new_rows=None, deleted=()):
        """Patch the imported graph in place (rxgpu_hnsw_update): `nodes` = internal ids whose lists changed, taken from `graph`
        (same layout as hnsw_import); `new_rows` = {internal id: (label, vector)} for inserted / replaced rows."""
        new_rows = new_rows or {}
        order = sorted(new_rows) + [int(v) for v in nodes if int(v) not in new_rows]
        l0 = np.ascontiguousarray(graph["level0"], np.uint32)
        up = np.ascontiguousarray(graph["upper"], np.uint32).reshape(-1, 1 + graph["M"])
        uo = graph["upper_offsets"]
        upd = (HnswNodeUpdate * max(len(order), 1))()
        keep = []
        dele = set(int(v) for v in deleted)
        for i, v in enumerate(order):
            lvl = int(graph["levels"][v])
            upd[i].node, upd[i].level = v, lvl
            upd[i].level0 = l0[v].ctypes.data
            upd[i].upper = up[int(uo[v])].ctypes.data if lvl > 0 else None
            if v in new_rows:
                vec = np.ascontiguousarray(new_rows[v][1], np.float32)
                keep.append(vec)
                upd[i].vec, upd[i].label = vec.ctypes.data, int(new_rows[v][0])
            upd[i].deleted = 1 if v in dele else 0
        _check(self._lib.rxgpu_hnsw_update(self._h, graph["maxlevel"], graph["enterpoint"], len(order), upd))

    def hnsw_update_count(self) -> int:
        return int(self._lib.rxgpu_hnsw_update_count(self._h))

    def hnsw_mark_deleted(self, label: int):
        _check(self._lib.rxgpu_hnsw_mark_deleted(self._h, int(label)))

    def hnsw_deleted_count(self) -> int:
        return int(self._lib.rxgpu_hnsw_deleted_count(self._h))

    def hnsw_search_knn_device(self, nq, d_queries_ptr, k, ef, d_dist_ptr, d_idx_ptr, d_count_ptr, d_stats_ptr=0, stream=0):
        _check(self._lib.rxgpu_hnsw_search_knn_device(self._h, nq, d_queries_ptr, k, ef, d_dist_ptr, d_idx_ptr, d_count_ptr,
                                                      d_stats_ptr or None, stream or None))

    def gather_labels_device(self, n, d_idx_ptr, d_label_ptr, stream=0):
        _check(self._lib.rxgpu_gather_labels_device(self._h, n, d_idx_ptr, d_label_ptr, stream or None))

    def hnsw_search_range(self, query, radius: float, ef: int, max_out: int | None = None):
        q = np.ascontiguousarray(query, dtype=np.float32)
        max_out = self.size() if max_out is None else max_out
        d = np.zeros(max(max_out, 1), np.float32)
        l = np.zeros(max(max_out, 1), np.uint64)
        n = C.c_uint64(0)
        _check(self._lib.rxgpu_hnsw_search_range(self._h, _p(q, _f32p), radius, ef, max_out, _p(d, _f32p), _p(l, _u64p), C.byref(n)))
        m = min(n.value, max_out)
        return d[:m], l[:m], n.value

    def hnsw_search_range_batch(self, queries, radii, ef: int, max_out: int):
        """rxgpu_hnsw_search_range_batch.  queries: [nq, dim]; radii: a scalar or [nq] (map space, as hnsw_search_range).  Returns
        (dists [nq, max_out], labels [nq, max_out], counts [nq]): row q holds the best min(counts[q], max_out) matches of query q,
        best-first, and counts[q] is its total number of matches."""
        q = np.ascontiguousarray(queries, dtype=np.float32).reshape(-1, self.dim)
        nq = q.shape[0]
        r = np.ascontiguousarray(np.broadcast_to(np.asarray(radii, dtype=np.float32), (nq,)))
        d = np.zeros((nq, max(max_out, 1)), np.float32)
        l = np.zeros((nq, max(max_out, 1)), np.uint64)
        c = np.zeros(nq, np.uint64)
        _check(self._lib.rxgpu_hnsw_search_range_batch(self._h, nq, _p(q, _f32p), _p(r, _f32p), ef, max_out, _p(d, _f32p), _p(l, _u64p),
                                                       _p(c, _u64p)))
        return d[:, :max_out], l[:, :max_out], c

    def hnsw_stream(self, query, batch_size: int, ef: int = 0, max_batches: int = 10**9):
        """Begin/ContinueStreamingSearch: yields (dist, label) batches, best first inside a batch, until exhausted"""
        q = np.ascontiguousarray(query, np.float32)
        s = C.c_void_p()
        _check(self._lib.rxgpu_hnsw_stream_begin(self._h, _p(q, _f32p), ef, C.byref(s)))
        try:
            for _ in range(max_batches):
                d = np.zeros(max(batch_size, 1), np.float32)
                l = np.zeros(max(batch_size, 1), np.uint64)
                n, ex = C.c_uint32(0), C.c_int(0)
                _check(self._lib.rxgpu_hnsw_stream_next(s, batch_size, _p(d, _f32p), _p(l, _u64p), C.byref(n), C.byref(ex)))
                yield d[:n.value].copy(), l[:n.value].copy()
                if ex.value:
                    break
        finally:
            self._lib.rxgpu_hnsw_stream_end(s)

    # -- SQ8 (the reference's scalar quantisation of an HNSW map) ---------------------------------------------------------
    def sq8_attach(self, params: dict, codes=None, offsets=None):
        """params: min_q, max_q, alpha, alpha_2, delta (hnswlib::QuantizingParams).  codes/offsets from the reference, or None to
        quantise the rows on the device with the reference's arithmetic."""
        p = Sq8Params(params["min_q"], params["max_q"], params["alpha"], params["alpha_2"], params["delta"])
        if codes is None:
            _check(self._lib.rxgpu_sq8_attach(self._h, C.byref(p), None, None))
        else:
            c = np.ascontiguousarray(codes, np.uint8)
            o = np.ascontiguousarray(offsets, np.float32)
            assert c.shape == (self.size(), self.dim) and o.shape == (self.size(),)
            _check(self._lib.rxgpu_sq8_attach(self._h, C.byref(p), _p(c, _u8p), _p(o, _f32p)))

    def sq8_export(self):
        codes = np.zeros((self.size(), self.dim), np.uint8)
        offs = np.zeros(self.size(), np.float32)
        _check(self._lib.rxgpu_sq8_export(self._h, _p(codes, _u8p), _p(offs, _f32p)))
        return codes, offs

    def sq8_prepare_query(self, query, query_norm=1.0):
        q = np.ascontiguousarray(query, np.float32)
        codes = np.zeros(self.dim, np.uint8)
        off = C.c_float(0)
        _check(self._lib.rxgpu_sq8_prepare_query(self._h, _p(q, _f32p), query_norm, _p(codes, _u8p), C.byref(off)))
        return codes, off.value

    def _sq8_search(self, fn, queries, k, query_norms, extra):
        q = np.ascontiguousarray(queries, dtype=np.float32).reshape(-1, self.dim)
        nq = q.shape[0]
        qn = None if query_norms is None else np.ascontiguousarray(query_norms, np.float32)
        d = np.zeros((nq, max(k, 1)), np.float32)
        l = np.zeros((nq, max(k, 1)), np.uint64)
        c = np.zeros(nq, np.uint32)
        _check(fn(self._h, nq, _p(q, _f32p), None if qn is None else _p(qn, _f32p), k, *extra, _p(d, _f32p), _p(l, _u64p), _p(c, _u32p)))
        return d, l, c

    def sq8_search_knn(self, queries, k: int, query_norms=None):
        return self._sq8_search(self._lib.rxgpu_sq8_search_knn, queries, k, query_norms, ())

    def hnsw_search_knn_sq8(self, queries, k: int, ef: int = 0, query_norms=None, with_stats=False):
        q = np.ascontiguousarray(queries, dtype=np.float32).reshape(-1, self.dim)
        nq = q.shape[0]
        qn = None if query_norms is None else np.ascontiguousarray(query_norms, np.float32)
        d = np.zeros((nq, max(k, 1)), np.float32)
        l = np.zeros((nq, max(k, 1)), np.uint64)
        c = np.zeros(nq, np.uint32)
        st = np.zeros((nq, 2), np.uint32)
        _check(self._lib.rxgpu_hnsw_search_knn_sq8(self._h, nq, _p(q, _f32p), None if qn is None else _p(qn, _f32p), k, ef, _p(d, _f32p),
                                                   _p(l, _u64p), _p(c, _u32p), _p(st, _u32p)))
        return (d, l, c, st) if with_stats else (d, l, c)

    # -- IVF (lists trained and assigned by the reference's FAISS; rows of this index grouped by list) -------------------
    def ivf_import(self, centroids, list_sizes):
        c = np.ascontiguousarray(centroids, np.float32)
        ls = np.ascontiguousarray(list_sizes, np.uint64)
        _check(self._lib.rxgpu_ivf_import(self._h, len(ls), _p(c, _f32p), _p(ls, _u64p)))

    def ivf_search_knn(self, queries, k: int, nprobe: int):
        q = np.ascontiguousarray(queries, dtype=np.float32).reshape(-1, self.dim)
        nq = q.shape[0]
        d = np.zeros((nq, max(k, 1)), np.float32)
        l = np.zeros((nq, max(k, 1)), np.uint64)
        c = np.zeros(nq, np.uint32)
        _check(self._lib.rxgpu_ivf_search_knn(self._h, nq, _p(q, _f32p), k, nprobe, _p(d, _f32p), _p(l, _u64p), _p(c, _u32p)))
        return d, l, c

    def ivf_search_knn_large_k(self, queries, k: int, nprobe: int):
        """ivf_search_knn at any k in [1, 65535] and any nprobe (rxgpu_ivf_search_knn_large_k)"""
        q = np.ascontiguousarray(queries, dtype=np.float32).reshape(-1, self.dim)
        nq = q.shape[0]
        d = np.zeros((nq, max(k, 1)), np.float32)
        l = np.zeros((nq, max(k, 1)), np.uint64)
        c = np.zeros(nq, np.uint32)
        _check(self._lib.rxgpu_ivf_search_knn_large_k(self._h, nq, _p(q, _f32p), k, nprobe, _p(d, _f32p), _p(l, _u64p), _p(c, _u32p)))
        return d, l, c

    def ivf_search_range(self, query, radius: float, nprobe: int, max_out: int | None = None):
        q = np.ascontiguousarray(query, dtype=np.float32)
        max_out = max(self.size(), self.ivf_size()) if max_out is None else max_out
        d = np.zeros(max(max_out, 1), np.float32)
        l = np.zeros(max(max_out, 1), np.uint64)
        n = C.c_uint64(0)
        _check(self._lib.rxgpu_ivf_search_range(self._h, _p(q, _f32p), radius, nprobe, max_out, _p(d, _f32p), _p(l, _u64p), C.byref(n)))
        m = min(n.value, max_out)
        return d[:m], l[:m], n.value

    def ivf_search_range_batch(self, queries, radii, nprobe: int, max_out: int):
        """rxgpu_ivf_search_range_batch.  queries: [nq, dim]; radii: a scalar or [nq] (map space, as ivf_search_range).  Returns
        (dists [nq, max_out], labels [nq, max_out], counts [nq]): row q holds the best min(counts[q], max_out) matches of query q,
        best-first, and counts[q] is its total number of matches."""
        q = np.ascontiguousarray(queries, dtype=np.float32).reshape(-1, self.dim)
        nq = q.shape[0]
        r = np.ascontiguousarray(np.broadcast_to(np.asarray(radii, dtype=np.float32), (nq,)))
        d = np.zeros((nq, max(max_out, 1)), np.float32)
        l = np.zeros((nq, max(max_out, 1)), np.uint64)
        c = np.zeros(nq, np.uint64)
        _check(self._lib.rxgpu_ivf_search_range_batch(self._h, nq, _p(q, _f32p), _p(r, _f32p), nprobe, max_out, _p(d, _f32p), _p(l, _u64p),
                                                      _p(c, _u64p)))
        return d[:, :max_out], l[:, :max_out], c

    # -- bench / test support ------------------------------------------------------------------------------------------
    def append_synth(self, seed: int, first_row: int, n: int):
        _check(self._lib.rxgpu_index_append_synth(self._h, seed, first_row, n))

    def set_query_tile(self, qt: int):
        _check(self._lib.rxgpu_set_query_tile(self._h, qt))

    def set_tensor_core_filter(self, mode: int):
        """0 = auto, 1 = whenever possible, 2 = never (exact fp32 scan only); 3 / 4 / 5 = as 1 in single CTAs / clusters of up to
        two / clusters of up to four CTAs that share every row tile (0 and 1: clusters of up to two on >= 2^23 rows)"""
        _check(self._lib.rxgpu_set_tensor_core_filter(self._h, mode))

    def tc_audit(self, queries, tau, query_block: int = 128, row_bound: bool = True) -> dict:
        """rxgpu_tc_audit: the int8 filter's certificate for these queries at thresholds tau (map space, a scalar or [nq]), as
        host arrays: slot_row [S], rowc [S, 4], blockc [B, 8], row_codes [S, dim], query_codes [nq, dim], qc [nq, 4],
        kab [query blocks, 2], block_thr [nq, B] and, with row_bound, row_bound [nq, S, 2] = (d~, err)."""
        q = np.ascontiguousarray(queries, dtype=np.float32).reshape(-1, self.dim)
        nq = q.shape[0]
        t = np.ascontiguousarray(np.broadcast_to(np.asarray(tau, dtype=np.float32), (nq,)))
        shape = np.zeros(2, np.uint32)
        _check(self._lib.rxgpu_tc_audit(self._h, 0, None, None, query_block, _p(shape, _u32p), *([None] * 9)))
        S, B = int(shape[0]), int(shape[1])
        o = {"slot_row": np.zeros(max(S, 1), np.uint32), "rowc": np.zeros((max(S, 1), 4), np.float32),
             "blockc": np.zeros((max(B, 1), 8), np.float32), "row_codes": np.zeros((max(S, 1), self.dim), np.int8),
             "query_codes": np.zeros((max(nq, 1), self.dim), np.int8), "qc": np.zeros((max(nq, 1), 4), np.float32),
             "kab": np.zeros((max((nq + query_block - 1) // query_block, 1), 2), np.float32),
             "block_thr": np.zeros((max(nq, 1), max(B, 1)), np.int32),
             "row_bound": np.zeros((max(nq, 1), max(S, 1), 2), np.float32) if row_bound and S else None}
        _check(self._lib.rxgpu_tc_audit(self._h, nq, _p(q, _f32p), _p(t, _f32p), query_block, _p(shape, _u32p), _p(o["slot_row"], _u32p),
                                        _p(o["rowc"], _f32p), _p(o["blockc"], _f32p), o["row_codes"].ctypes.data,
                                        o["query_codes"].ctypes.data, _p(o["qc"], _f32p), _p(o["kab"], _f32p), _p(o["block_thr"], _i32p),
                                        None if o["row_bound"] is None else _p(o["row_bound"], _f32p)))
        nqb = (nq + query_block - 1) // query_block
        out = {"slot_row": o["slot_row"][:S], "rowc": o["rowc"][:S], "blockc": o["blockc"][:B], "row_codes": o["row_codes"][:S],
               "query_codes": o["query_codes"][:nq], "qc": o["qc"][:nq], "kab": o["kab"][:nqb], "block_thr": o["block_thr"][:nq, :B],
               "row_bound": None if o["row_bound"] is None else o["row_bound"][:nq, :S]}
        return out


COMM_ID_BYTES = 128


def comm_unique_id() -> bytes:
    buf = C.create_string_buffer(COMM_ID_BYTES)
    _check(lib().rxgpu_comm_unique_id(buf))
    return buf.raw


class ShardComm:
    """rxgpu_comm: this rank's end of the communicator the sharded searches exchange their per-shard lists over (NCCL between
    processes, or a host rendezvous between the threads of one process: local_group)."""

    def __init__(self, nranks: int, rank: int, comm_id: bytes | None, device: int, _handle=None):
        self._lib = lib()
        if _handle is not None:  # one of the communicators rxgpu_comm_create_local made
            self._h = _handle
            return
        self._h = C.c_void_p()
        idbuf = C.create_string_buffer(comm_id, COMM_ID_BYTES) if comm_id is not None else None
        _check(self._lib.rxgpu_comm_create(C.byref(self._h), nranks, rank, idbuf, device))

    @staticmethod
    def local_group(nranks: int, devices=None):
        """rxgpu_comm_create_local: the ranks of ONE process (one host thread per rank); devices may repeat"""
        hs = (C.c_void_p * nranks)()
        dv = None if devices is None else (C.c_int * nranks)(*devices)
        _check(lib().rxgpu_comm_create_local(hs, nranks, dv))
        return [ShardComm(nranks, r, None, 0, _handle=C.c_void_p(hs[r])) for r in range(nranks)]

    def close(self):
        if self._h:
            self._lib.rxgpu_comm_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def search_knn(self, shard: "GpuBruteforceSearch", queries, k: int, nq: int | None = None):
        """queries: host ndarray [nq, dim] or a device pointer (int) with nq given.  Collective: every rank calls it."""
        if isinstance(queries, np.ndarray):
            q = np.ascontiguousarray(queries, np.float32)
            nq, qp, on_dev = q.shape[0], q.ctypes.data_as(C.c_void_p), 0
        else:
            qp, on_dev = C.c_void_p(int(queries)), 1
        kk = max(k, 1)
        od = np.zeros((nq, kk), np.float32)
        ol = np.zeros((nq, kk), np.uint64)
        oc = np.zeros(nq, np.uint32)
        _check(self._lib.rxgpu_sharded_search_knn(self._h, shard._h, nq, qp, on_dev, k, _p(od, _f32p), _p(ol, _u64p), _p(oc, _u32p)))
        return od, ol, oc

    def search_range_batch(self, shard: "GpuBruteforceSearch", queries, radius, max_out: int, nq: int | None = None):
        """rxgpu_sharded_search_range_batch.  queries: host ndarray [nq, dim] or a device pointer (int) with nq given; radius: a
        scalar or [nq] (map space).  Returns (dists [nq, max_out], labels [nq, max_out], counts [nq]) as
        GpuBruteforceSearch.search_range_batch returns them for one index holding every shard's rows.  Collective: every rank calls it."""
        if isinstance(queries, np.ndarray):
            q = np.ascontiguousarray(queries, np.float32)
            nq, qp, on_dev = q.shape[0], q.ctypes.data_as(C.c_void_p), 0
        else:
            qp, on_dev = C.c_void_p(int(queries)), 1
        r = np.ascontiguousarray(np.broadcast_to(np.asarray(radius, dtype=np.float32), (nq,)))
        od = np.zeros((nq, max(max_out, 1)), np.float32)
        ol = np.zeros((nq, max(max_out, 1)), np.uint64)
        oc = np.zeros(nq, np.uint64)
        _check(self._lib.rxgpu_sharded_search_range_batch(self._h, shard._h, nq, qp, on_dev, _p(r, _f32p), max_out, _p(od, _f32p),
                                                          _p(ol, _u64p), _p(oc, _u64p)))
        return od[:, :max_out], ol[:, :max_out], oc

    def ivf_train(self, shard: "GpuBruteforceSearch", nlist: int, vecs, norm_coefs=None, niter: int = 10, seed: int = 1234,
                  max_points_per_centroid: int = 256):
        """rxgpu_sharded_ivf_train: this rank's rows [n_local, dim] (a rank may have none); every rank gets what
        GpuBruteforceSearch.ivf_train returns for the concatenation of all ranks' rows.  Collective: every rank calls it."""
        v = np.ascontiguousarray(vecs, np.float32).reshape(-1, shard.dim)
        nc = None if norm_coefs is None else np.ascontiguousarray(norm_coefs, np.float32)
        prm = IvfTrainParams(niter, seed, max_points_per_centroid)
        cent = np.zeros((max(nlist, 1), shard.dim), np.float32)
        st = (IvfTrainStats * max(niter, 1))()
        _check(self._lib.rxgpu_sharded_ivf_train(self._h, shard._h, nlist, len(v), _p(v, _f32p), None if nc is None else _p(nc, _f32p),
                                                 C.byref(prm), _p(cent, _f32p), st))
        stats = [{f: getattr(st[i], f) for f, _ in IvfTrainStats._fields_} for i in range(max(niter, 0))]
        return cent[:nlist], stats

    def ivf_search_knn(self, shard: "GpuBruteforceSearch", queries, k: int, nprobe: int, nq: int | None = None):
        """rxgpu_sharded_ivf_search_knn.  queries: host ndarray [nq, dim] or a device pointer (int) with nq given.  Returns
        (dists [nq, k], labels [nq, k], counts [nq]).  Collective: every rank calls it."""
        if isinstance(queries, np.ndarray):
            q = np.ascontiguousarray(queries, np.float32).reshape(-1, shard.dim)
            nq, qp, on_dev = q.shape[0], q.ctypes.data_as(C.c_void_p), 0
        else:
            qp, on_dev = C.c_void_p(int(queries)), 1
        od = np.zeros((nq, max(k, 1)), np.float32)
        ol = np.zeros((nq, max(k, 1)), np.uint64)
        oc = np.zeros(nq, np.uint32)
        _check(self._lib.rxgpu_sharded_ivf_search_knn(self._h, shard._h, nq, qp, on_dev, k, nprobe, _p(od, _f32p), _p(ol, _u64p), _p(oc, _u32p)))
        return od, ol, oc

    def ivf_search_range_batch(self, shard: "GpuBruteforceSearch", queries, radius, nprobe: int, max_out: int, nq: int | None = None):
        """rxgpu_sharded_ivf_search_range_batch.  queries: host ndarray [nq, dim] or a device pointer (int) with nq given; radius: a
        scalar or [nq] (map space).  Returns (dists [nq, max_out], labels [nq, max_out], counts [nq]) as
        GpuBruteforceSearch.ivf_search_range_batch returns them for one index holding every shard's rows.  Collective."""
        if isinstance(queries, np.ndarray):
            q = np.ascontiguousarray(queries, np.float32).reshape(-1, shard.dim)
            nq, qp, on_dev = q.shape[0], q.ctypes.data_as(C.c_void_p), 0
        else:
            qp, on_dev = C.c_void_p(int(queries)), 1
        r = np.ascontiguousarray(np.broadcast_to(np.asarray(radius, dtype=np.float32), (nq,)))
        od = np.zeros((nq, max(max_out, 1)), np.float32)
        ol = np.zeros((nq, max(max_out, 1)), np.uint64)
        oc = np.zeros(nq, np.uint64)
        _check(self._lib.rxgpu_sharded_ivf_search_range_batch(self._h, shard._h, nq, qp, on_dev, _p(r, _f32p), nprobe, max_out, _p(od, _f32p),
                                                              _p(ol, _u64p), _p(oc, _u64p)))
        return od[:, :max_out], ol[:, :max_out], oc


def select_postprocess(metric, dist, label, k=None, has_radius=False, need_sort=True, is_array=False, raw=False):
    """HnswIndexBase::select / selectRaw post-processing of a map's best-first answer (host only): (row_ids, ranks)"""
    d = np.ascontiguousarray(dist, np.float32)
    l = np.ascontiguousarray(label, np.uint64)
    prm = SelectParams(k or 0, int(has_radius), 0.0, int(need_sort), int(is_array), int(raw))
    ids = np.zeros(max(len(d), 1), np.int32)
    ranks = np.zeros(max(len(d), 1), np.float32)
    n = C.c_uint64(0)
    _check(lib().rxgpu_select_postprocess(metric, C.byref(prm), len(d), _p(d, _f32p), _p(l, _u64p), _p(ids, _i32p), _p(ranks, _f32p), C.byref(n)))
    return ids[:n.value], ranks[:n.value]


def merge_shards(k, dist, idx, label, count, shard_base):
    """dist/idx/label: [nshards, nq, k1]; count: [nshards, nq]; returns (dist, gidx, label, count, need_tie)."""
    dist = np.ascontiguousarray(dist, np.float32)
    idx = np.ascontiguousarray(idx, np.uint32)
    label = np.ascontiguousarray(label, np.uint64)
    count = np.ascontiguousarray(count, np.uint32)
    base = np.ascontiguousarray(shard_base, np.uint64)
    ns, nq, k1 = dist.shape
    od = np.zeros((nq, max(k, 1)), np.float32)
    og = np.zeros((nq, max(k, 1)), np.uint64)
    ol = np.zeros((nq, max(k, 1)), np.uint64)
    oc = np.zeros(nq, np.uint32)
    nt = np.zeros(nq, np.uint8)
    _check(lib().rxgpu_merge_shards(ns, nq, k, k1, _p(dist, _f32p), _p(idx, _u32p), _p(label, _u64p), _p(count, _u32p), _p(base, _u64p),
                                    _p(od, _f32p), _p(og, _u64p), _p(ol, _u64p), _p(oc, _u32p), _p(nt, _u8p)))
    return od, og, ol, oc, nt


def tie_replay(k, dstar, lower, first):
    """lower / first: tuples (dist, gidx, label) of equal-length arrays; returns (dist, label)."""
    ld, lg, ll = (np.ascontiguousarray(a, t) for a, t in zip(lower, (np.float32, np.uint64, np.uint64)))
    fd, fg, fl = (np.ascontiguousarray(a, t) for a, t in zip(first, (np.float32, np.uint64, np.uint64)))
    od = np.zeros(max(k, 1), np.float32)
    ol = np.zeros(max(k, 1), np.uint64)
    oc = C.c_uint32(0)
    _check(lib().rxgpu_tie_replay(k, dstar, len(ld), _p(ld, _f32p), _p(lg, _u64p), _p(ll, _u64p), len(fd), _p(fd, _f32p), _p(fg, _u64p),
                                  _p(fl, _u64p), _p(od, _f32p), _p(ol, _u64p), C.byref(oc)))
    return od[:oc.value], ol[:oc.value]


class GpuFtIndex:
    """Device-resident ft_fast merge state: document statistics + posting lists; merge() = ft::Merger::Merge."""

    def __init__(self, total_docs, words_in_field, avg_words, removed=None, device=0):
        self._lib = lib()
        w = np.ascontiguousarray(words_in_field, np.uint32).reshape(total_docs, -1)
        self.total_docs, self.nfields = total_docs, w.shape[1]
        a = np.ascontiguousarray(avg_words, np.float32)
        r = None if removed is None else np.ascontiguousarray(removed, np.uint8)
        h = C.c_void_p()
        _check(self._lib.rxgpu_ft_create(C.byref(h), total_docs, self.nfields, _p(w, _u32p), _p(a, _f32p), None if r is None else _p(r, _u8p),
                                         device))
        self._h = h

    def close(self):
        if getattr(self, "_h", None):
            self._lib.rxgpu_ft_destroy(self._h)
            self._h = None

    __del__ = close

    def add_postings(self, doc_ids, pos_begin, positions) -> int:
        d = np.ascontiguousarray(doc_ids, np.uint32)
        b = np.ascontiguousarray(pos_begin, np.uint32)
        p = np.ascontiguousarray(positions, np.uint32)
        pl = FtPostings(len(d), _p(d, _u32p), _p(b, _u32p), _p(p, _u32p))
        out = C.c_uint32(0)
        _check(self._lib.rxgpu_ft_add_postings(self._h, C.byref(pl), C.byref(out)))
        return out.value

    def add_postings_packed(self, data, count: int) -> int:
        """data: the bytes of a PackedIdRelVec (the reference's varint-delta posting stream), count: its number of records"""
        b = np.ascontiguousarray(data, np.uint8)
        out = C.c_uint32(0)
        _check(self._lib.rxgpu_ft_add_postings_packed(self._h, _p(b, _u8p), len(b), count, C.byref(out)))
        return out.value

    def add_postings_packed_batch(self, datas, counts):
        """datas: list of byte arrays (PackedIdRelVec streams), decoded on the device; returns the list ids"""
        bufs = [np.ascontiguousarray(d, np.uint8) for d in datas]
        n = len(bufs)
        ptrs = (C.c_void_p * max(n, 1))(*[b.ctypes.data if len(b) else None for b in bufs])
        lens = (C.c_uint64 * max(n, 1))(*[len(b) for b in bufs])
        cnt = np.ascontiguousarray(counts, np.uint32)
        out = np.zeros(max(n, 1), np.uint32)
        _check(self._lib.rxgpu_ft_add_postings_packed_batch(self._h, n, ptrs, lens, _p(cnt, _u32p), _p(out, _u32p)))
        return out[:n].tolist()

    def merge(self, cfg: dict, field_cfg: list, terms: list, excluded=None, rank_sort_type=1, max_out=None, synonyms=None):
        """cfg / field_cfg: dicts with the FtConfig / FtFieldConfig member names; terms: dicts(op, boost, term_len_boost, field_boosts,
        postings, procs[, suppressed, synonym_ids]); synonyms: lists of such dicts (multi-word synonyms).  Returns a structured array
        (id, proc, field, normalized_proc)."""
        c, arr, keep = self._config_and_terms(cfg, field_cfg, terms)
        ex = None if excluded is None else np.ascontiguousarray(excluded, np.uint8)
        max_out = self.total_docs if max_out is None else max_out
        out = np.zeros(max(max_out, 1), FT_MERGE_INFO_DTYPE)
        n = C.c_uint64(0)
        if synonyms:
            q = self._query(arr, len(terms), synonyms, keep)
            _check(self._lib.rxgpu_ft_merge_query(self._h, C.byref(c), C.byref(q), None if ex is None else _p(ex, _u8p), rank_sort_type,
                                                  max_out, out.ctypes.data, C.byref(n)))
        else:
            _check(self._lib.rxgpu_ft_merge(self._h, C.byref(c), len(terms), arr, None if ex is None else _p(ex, _u8p), rank_sort_type,
                                            max_out, out.ctypes.data, C.byref(n)))
        return out[:min(n.value, max_out)].copy()

    def merge_areas(self, cfg: dict, field_cfg: list, terms: list, max_areas_in_doc=5, excluded=None, rank_sort_type=1, max_out=None,
                    synonyms=None):
        """merge() with highlight areas (rxgpu_ft_merge_query_areas, MergeDataAreas<Area>): returns (infos, begin, areas, raw).  For
        entry i and field f the committed areas are areas[begin[i * nfields + f]:begin[i * nfields + f + 1]] as (start, end) rows;
        raw[i] = the document's area count before the commit."""
        c, arr, keep = self._config_and_terms(cfg, field_cfg, terms)
        q = self._query(arr, len(terms), synonyms or [], keep)
        ex = None if excluded is None else np.ascontiguousarray(excluded, np.uint8)
        max_out = self.total_docs if max_out is None else max_out
        out = np.zeros(max(max_out, 1), FT_MERGE_INFO_DTYPE)
        a = min(max(int(max_areas_in_doc), 1), 64)
        begin = np.zeros(max(max_out, 1) * self.nfields + 1, np.uint32)
        areas = np.zeros((max(max_out * self.nfields * a, 1), 2), np.uint32)
        raw = np.zeros(max(max_out, 1), np.uint32)
        n = C.c_uint64(0)
        _check(self._lib.rxgpu_ft_merge_query_areas(self._h, C.byref(c), C.byref(q), None if ex is None else _p(ex, _u8p), rank_sort_type,
                                                    int(max_areas_in_doc), max_out, out.ctypes.data, _p(begin, _u32p), areas.ctypes.data,
                                                    _p(raw, _u32p), C.byref(n)))
        m = min(n.value, max_out)
        begin = begin[:m * self.nfields + 1].copy()
        return out[:m].copy(), begin, areas[:int(begin[-1])].copy(), raw[:m].copy()

    def _query(self, arr, nterms, synonyms, keep):
        syn = (FtSynonym * len(synonyms))()
        for i, terms in enumerate(synonyms):
            ta = self._terms(terms, keep)
            keep.append(ta)
            syn[i] = FtSynonym(len(terms), ta)
        keep.append(syn)
        return FtQuery(nterms, arr, len(synonyms), syn)

    def set_rows(self, row_begin, row_ids):
        """vdoc -> row ids (CSR), the IndexText::vdocs_[vdoc].RowIds() of the reference"""
        rb = np.ascontiguousarray(row_begin, np.uint32)
        ri = np.ascontiguousarray(row_ids, np.int32)
        _check(self._lib.rxgpu_ft_set_rows(self._h, _p(rb, _u32p), _p(ri, _i32p)))

    def select(self, cfg, field_cfg, terms, limit, excluded=None, row_status=None, rank_sort_type=1, synonyms=None):
        """merge + postProcessResults + afterSelect + sortAfterSelect on the device: (row_ids, ranks, total rows)"""
        c, arr, keep = self._config_and_terms(cfg, field_cfg, terms)
        ex = None if excluded is None else np.ascontiguousarray(excluded, np.uint8)
        rs = None if row_status is None else np.ascontiguousarray(row_status, np.uint8)
        ids = np.zeros(max(limit, 1), np.int32)
        ranks = np.zeros(max(limit, 1), np.float32)
        n = C.c_uint64(0)
        if synonyms:
            q = self._query(arr, len(terms), synonyms, keep)
            _check(self._lib.rxgpu_ft_select_query(self._h, C.byref(c), C.byref(q), None if ex is None else _p(ex, _u8p),
                                                   None if rs is None else _p(rs, _u8p), rank_sort_type, limit, _p(ids, _i32p), _p(ranks, _f32p),
                                                   C.byref(n)))
        else:
            _check(self._lib.rxgpu_ft_select(self._h, C.byref(c), len(terms), arr, None if ex is None else _p(ex, _u8p),
                                             None if rs is None else _p(rs, _u8p), rank_sort_type, limit, _p(ids, _i32p), _p(ranks, _f32p),
                                             C.byref(n)))
        m = min(n.value, limit)
        return ids[:m], ranks[:m], n.value

    def sharded_select(self, comm: "ShardComm", doc_base: int, cfg, field_cfg, terms, limit, excluded=None, row_status=None, rank_sort_type=1):
        """rxgpu_sharded_ft_select: collective over the docid-range shards of one namespace; every rank gets the namespace's rows"""
        c, arr, keep = self._config_and_terms(cfg, field_cfg, terms)
        ex = None if excluded is None else np.ascontiguousarray(excluded, np.uint8)
        rs = None if row_status is None else np.ascontiguousarray(row_status, np.uint8)
        ids = np.zeros(max(limit, 1), np.int32)
        ranks = np.zeros(max(limit, 1), np.float32)
        n = C.c_uint64(0)
        _check(self._lib.rxgpu_sharded_ft_select(comm._h, self._h, doc_base, C.byref(c), len(terms), arr, None if ex is None else _p(ex, _u8p),
                                                 None if rs is None else _p(rs, _u8p), rank_sort_type, limit, _p(ids, _i32p), _p(ranks, _f32p),
                                                 C.byref(n)))
        m = min(n.value, limit)
        return ids[:m], ranks[:m], n.value

    def _config_and_terms(self, cfg, field_cfg, terms):
        fc = (FtFieldConfig * self.nfields)(*[FtFieldConfig(**f) for f in field_cfg])
        c = FtConfig(cfg["merge_limit"], cfg["min_rank"], cfg["bm25_k1"], cfg["bm25_b"], cfg["bm25_type"], cfg["distance_boost"],
                     cfg["distance_weight"], cfg["full_match_boost"], self.nfields, fc, cfg.get("summation_ranks_by_fields_ratio", 0.0))
        keep = [fc]
        arr = self._terms(terms, keep)
        return c, arr, keep

    @staticmethod
    def _terms(terms, keep):
        arr = (FtTerm * max(len(terms), 1))()
        for i, t in enumerate(terms):
            fb = np.ascontiguousarray(t["field_boosts"], np.float32)
            po = np.ascontiguousarray(t["postings"], np.uint32)
            pr = np.ascontiguousarray(t["procs"], np.float32)
            ns = None if t.get("need_sum_rank") is None else np.ascontiguousarray(t["need_sum_rank"], np.uint8)
            su = None if t.get("suppressed") is None else np.ascontiguousarray(t["suppressed"], np.uint8)
            sy = np.ascontiguousarray(t.get("synonym_ids", ()), np.uint32)
            keep += [fb, po, pr, ns, su, sy]
            arr[i] = FtTerm(t["op"], t["boost"], t["term_len_boost"], _p(fb, _f32p), len(po), _p(po, _u32p), _p(pr, _f32p),
                            None if ns is None else _p(ns, _u8p), None if su is None else _p(su, _u8p), len(sy),
                            _p(sy, _u32p) if len(sy) else None, int(t.get("phrase_num", 0)), int(t.get("distance", 0)))
        return arr

    def last_stats(self) -> dict:
        s = FtStats()
        self._lib.rxgpu_ft_last_stats(C.byref(s))
        return {f: getattr(s, f) for f, _ in FtStats._fields_}


def kmeans_plan(n: int, nlist: int, seed: int = 1234, max_points_per_centroid: int = 256):
    """host only: (sample, init) of rxgpu_ivf_train -- the input rows it trains on and the input row each initial centroid copies"""
    ns = min(n, nlist * max_points_per_centroid)
    sample = np.zeros(max(ns, 1), np.int32)
    init = np.zeros(max(nlist, 1), np.int32)
    _check(lib().rxgpu_kmeans_plan(n, nlist, seed, max_points_per_centroid, _p(sample, _i32p), _p(init, _i32p)))
    return sample[:ns], init[:nlist]


def hnsw_build_plan(M: int, n: int, first: int = 0, maxlevel: int = -1, levels=None, seed: int = 100):
    """host only: (levels, batch ends) of rxgpu_hnsw_build for rows [first, n) onto a graph whose top level is maxlevel"""
    lv = None if levels is None else np.ascontiguousarray(levels, np.int32)
    out = np.zeros(max(n - first, 1), np.int32)
    ends = np.zeros(max(n - first, 1), np.uint64)
    nb = C.c_uint64(0)
    _check(lib().rxgpu_hnsw_build_plan(M, first, n, maxlevel, None if lv is None else _p(lv, _i32p), seed, _p(out, _i32p), _p(ends, _u64p),
                                       C.byref(nb)))
    return out[:n - first], ends[:nb.value]


def ft_decode_packed(data, count: int):
    """host-only decoder of the reference's packed posting stream -> (doc_ids, pos_begin, positions)"""
    b = np.ascontiguousarray(data, np.uint8)
    npos = C.c_uint64(0)
    lib_ = lib()
    _check(lib_.rxgpu_ft_decode_packed(_p(b, _u8p), len(b), count, None, None, None, 0, C.byref(npos)))
    d = np.zeros(count, np.uint32)
    pb = np.zeros(count + 1, np.uint32)
    ps = np.zeros(max(npos.value, 1), np.uint32)
    _check(lib_.rxgpu_ft_decode_packed(_p(b, _u8p), len(b), count, _p(d, _u32p), _p(pb, _u32p), _p(ps, _u32p), npos.value, C.byref(npos)))
    return d, pb, ps[:npos.value]
