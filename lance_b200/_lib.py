"""ctypes binding of liblance_b200.so (the C ABI in include/lance_b200.h).

There is no fallback of any kind: if the shared library is missing, or no CUDA device is usable,
every entry point raises.  This module never imports oracle/ and never computes on the CPU.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.path.join(_HERE, "liblance_b200.so")

OK, INVALID_ARG, UNSUPPORTED, CUDA_ERROR, NCCL_ERROR, OOM, NO_DEVICE = range(7)
_STATUS_NAMES = ["OK", "INVALID_ARG", "UNSUPPORTED", "CUDA_ERROR", "NCCL_ERROR", "OOM", "NO_DEVICE"]

F32, F16, BF16, U8 = 0, 1, 2, 3
L2, COSINE, DOT = 0, 1, 2
METRICS = {"l2": L2, "euclidean": L2, "cosine": COSINE, "dot": DOT}


class LanceB200Error(RuntimeError):
    def __init__(self, status, message):
        super().__init__(f"lance_b200: {_STATUS_NAMES[status] if status < 7 else status}: {message}")
        self.status = status


class KMeansParams(C.Structure):
    _fields_ = [("max_iters", C.c_uint32), ("tolerance", C.c_double), ("redos", C.c_uint32),
                ("balance_factor", C.c_float), ("hierarchical_k", C.c_uint32),
                ("sample_rate", C.c_uint64), ("seed", C.c_uint64), ("init_centroids", C.c_void_p),
                ("metric", C.c_int), ("partition_index", C.c_uint32), ("partition_index_batch", C.c_uint32)]


class PQParams(C.Structure):
    _fields_ = [("num_sub_vectors", C.c_uint32), ("num_bits", C.c_uint32), ("max_iters", C.c_uint32),
                ("kmeans_redos", C.c_uint32), ("sample_rate", C.c_uint64), ("codebook", C.c_void_p),
                ("seed", C.c_uint64)]


class BuildParams(C.Structure):
    _fields_ = [("num_partitions", C.c_uint32), ("ivf", KMeansParams), ("pq", PQParams),
                ("seed", C.c_uint64)]


class FlatBuildParams(C.Structure):
    _fields_ = [("num_partitions", C.c_uint32), ("ivf", KMeansParams), ("seed", C.c_uint64)]


class SqBuildParams(C.Structure):
    """lb2_ivfsq_build_params (include/lance_b200.h)."""
    _fields_ = [("num_partitions", C.c_uint32), ("ivf", KMeansParams), ("num_bits", C.c_uint32),
                ("sample_rate", C.c_uint64), ("seed", C.c_uint64)]


class HnswSqBuildParams(C.Structure):
    """lb2_ivfhnswsq_build_params (include/lance_b200.h)."""
    _fields_ = [("sq", SqBuildParams), ("max_level", C.c_uint32), ("m", C.c_uint32), ("ef_construction", C.c_uint32),
                ("insert_batch", C.c_uint32)]


class HnswPqBuildParams(C.Structure):
    """lb2_ivfhnswpq_build_params (include/lance_b200.h)."""
    _fields_ = [("pq", BuildParams), ("max_level", C.c_uint32), ("m", C.c_uint32), ("ef_construction", C.c_uint32),
                ("insert_batch", C.c_uint32)]


class HnswFlatBuildParams(C.Structure):
    """lb2_ivfhnswflat_build_params (include/lance_b200.h)."""
    _fields_ = [("flat", FlatBuildParams), ("max_level", C.c_uint32), ("m", C.c_uint32), ("ef_construction", C.c_uint32),
                ("insert_batch", C.c_uint32)]


class RqBuildParams(C.Structure):
    """lb2_ivfrq_build_params (include/lance_b200.h)."""
    _fields_ = [("num_partitions", C.c_uint32), ("ivf", KMeansParams), ("num_bits", C.c_uint32),
                ("seed", C.c_uint64)]


class OptimizeParams(C.Structure):
    """lb2_optimize_params (include/lance_b200.h)."""
    _fields_ = [("new_centroids", C.c_void_p), ("new_k", C.c_uint32), ("part_map", C.c_void_p),
                ("add_part_ids", C.c_void_p), ("add_payload", C.c_void_p), ("add_rq_add", C.c_void_p),
                ("add_rq_scale", C.c_void_p), ("add_row_ids", C.c_void_p), ("n_add", C.c_uint64),
                ("remove_row_ids", C.c_void_p), ("n_remove", C.c_uint64), ("remap_old_ids", C.c_void_p),
                ("remap_new_ids", C.c_void_p), ("n_remap", C.c_uint64), ("seed", C.c_uint64),
                ("insert_batch", C.c_uint32)]


class SplitParams(C.Structure):
    """lb2_split_params (include/lance_b200.h)."""
    _fields_ = [("part", C.c_uint32), ("vectors", C.c_void_p), ("row_ids", C.c_void_p), ("n", C.c_uint64),
                ("cand_vectors", C.c_void_p), ("cand_row_ids", C.c_void_p), ("cand_part_ids", C.c_void_p),
                ("n_cand", C.c_uint64), ("opt", OptimizeParams), ("new_centroids_out", C.c_void_p),
                ("dest_out", C.c_void_p)]


class JoinParams(C.Structure):
    """lb2_join_params (include/lance_b200.h)."""
    _fields_ = [("part", C.c_uint32), ("vectors", C.c_void_p), ("row_ids", C.c_void_p), ("n", C.c_uint64),
                ("remove_row_ids", C.c_void_p), ("n_remove", C.c_uint64), ("remap_old_ids", C.c_void_p),
                ("remap_new_ids", C.c_void_p), ("n_remap", C.c_uint64), ("seed", C.c_uint64),
                ("insert_batch", C.c_uint32), ("dest_out", C.c_void_p)]


class IndexStorage(C.Structure):
    """lb2_index_storage (include/lance_b200.h)."""
    _fields_ = [("num_partitions", C.c_uint32), ("num_rows", C.c_uint64), ("num_bytes", C.c_uint64),
                ("part_lengths", C.c_void_p), ("row_ids", C.c_void_p), ("payload", C.c_void_p),
                ("add_factors", C.c_void_p), ("scale_factors", C.c_void_p), ("max_level", C.c_uint32),
                ("m", C.c_uint32), ("ef_construction", C.c_uint32), ("num_graph_rows", C.c_uint64),
                ("num_edges", C.c_uint64), ("entry_point", C.c_void_p), ("level_offsets", C.c_void_p),
                ("vector_id", C.c_void_p), ("list_offsets", C.c_void_p), ("neighbors", C.c_void_p),
                ("distances", C.c_void_p)]


class BuildStats(C.Structure):
    _fields_ = [("ms_ivf_train", C.c_float), ("ms_pq_train", C.c_float), ("ms_transform", C.c_float),
                ("ms_group", C.c_float), ("ms_total", C.c_float), ("ivf_iters", C.c_uint32),
                ("pq_iters_max", C.c_uint32), ("ivf_loss", C.c_double)]


# every symbol declared in include/lance_b200.h (checked by tests/test_abi.py)
EXPORTS = [
    "lb2_version", "lb2_last_error", "lb2_device_count", "lb2_set_device", "lb2_synchronize",
    "lb2_malloc", "lb2_free", "lb2_malloc_host", "lb2_free_host", "lb2_memcpy", "lb2_launch_count",
    "lb2_profile_enable", "lb2_profile_get", "lb2_profile_reset", "lb2_profile_dump", "lb2_timer_start", "lb2_timer_stop",
    "lb2_distance_batch", "lb2_normalize", "lb2_kmeans_params_default", "lb2_kmeans_train",
    "lb2_compute_partitions", "lb2_find_partitions", "lb2_compute_residual", "lb2_pq_params_default",
    "lb2_pq_train", "lb2_pq_encode", "lb2_pq_build_lut", "lb2_pq_scan", "lb2_flat_topk", "lb2_flat_topk_range",
    "lb2_ivfpq_transform", "lb2_index_create", "lb2_index_load", "lb2_index_search", "lb2_index_search_refine",
    "lb2_index_search_ex", "lb2_index_row_mask", "lb2_pq_scan_4bit",
    "lb2_index_info", "lb2_index_export", "lb2_index_export_partition", "lb2_index_destroy", "lb2_ivfpq_build_params_default",
    "lb2_ivfpq_build", "lb2_ivfflat_build_params_default", "lb2_ivfflat_build", "lb2_index_create_flat",
    "lb2_index_load_flat", "lb2_index_export_flat", "lb2_comm_unique_id", "lb2_comm_init", "lb2_comm_destroy",
    "lb2_comm_info", "lb2_index_search_sharded", "lb2_set_stream", "lb2_trim_memory", "lb2_index_search_async", "lb2_index_repartition", "lb2_index_update",
    "lb2_index_transform", "lb2_index_optimize",
    "lb2_index_partition_to_split", "lb2_index_partition_to_join", "lb2_index_reassign_candidates", "lb2_index_split",
    "lb2_index_join",
    "lb2_sq_train", "lb2_sq_encode", "lb2_ivfsq_build_params_default", "lb2_ivfsq_build", "lb2_index_create_sq",
    "lb2_index_load_sq", "lb2_index_export_sq", "lb2_ivfhnswsq_build_params_default", "lb2_ivfhnswsq_build",
    "lb2_index_load_hnsw_sq", "lb2_index_hnsw_sq_info", "lb2_index_export_hnsw_sq", "lb2_index_search_hnsw", "lb2_rq_rotation", "lb2_ivfrq_transform",
    "lb2_ivfrq_build_params_default", "lb2_ivfrq_build", "lb2_index_create_rq", "lb2_index_load_rq",
    "lb2_index_export_rq", "lb2_index_search_probed", "lb2_flat_search", "lb2_index_search_combined",
    "lb2_ivfhnswpq_build_params_default", "lb2_ivfhnswpq_build", "lb2_index_load_hnsw_pq", "lb2_index_hnsw_pq_info",
    "lb2_index_export_hnsw_pq", "lb2_ivfhnswflat_build_params_default", "lb2_ivfhnswflat_build",
    "lb2_index_load_hnsw_flat", "lb2_index_hnsw_flat_info", "lb2_index_export_hnsw_flat",
    "lb2_index_export_storage", "lb2_index_load_storage",
    "lb2_partition_index_uses_graph", "lb2_partition_index_build", "lb2_partition_index_assign",
    "lb2_partition_index_info", "lb2_partition_index_export", "lb2_partition_index_destroy",
    "lb2_index_set_partition_index", "lb2_index_search_batch", "lb2_index_search_candidates",
    "lb2_index_refine_taken", "lb2_flat_search_batch", "lb2_index_search_combined_batch",
]

_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(SO_PATH):
            raise LanceB200Error(NO_DEVICE, f"{SO_PATH} is missing: build it with "
                                 "`python -c 'import __graft_entry__ as g; g.build()'` "
                                 "(there is no CPU fallback)")
        L = C.CDLL(SO_PATH)
        L.lb2_version.restype = C.c_char_p
        L.lb2_last_error.restype = C.c_size_t
        L.lb2_last_error.argtypes = [C.c_char_p, C.c_size_t]
        L.lb2_device_count.restype = C.c_int
        L.lb2_profile_dump.restype = C.c_size_t
        L.lb2_profile_dump.argtypes = [C.c_char_p, C.c_size_t]
        for name in EXPORTS:
            if name not in ("lb2_version", "lb2_last_error", "lb2_device_count", "lb2_profile_dump",
                            "lb2_kmeans_params_default", "lb2_pq_params_default",
                            "lb2_ivfpq_build_params_default", "lb2_ivfflat_build_params_default",
                            "lb2_ivfsq_build_params_default", "lb2_ivfrq_build_params_default",
                            "lb2_ivfhnswsq_build_params_default", "lb2_ivfhnswpq_build_params_default",
                            "lb2_ivfhnswflat_build_params_default"):
                getattr(L, name).restype = C.c_int
        L.lb2_sq_encode.argtypes = [C.c_void_p, C.c_uint64, C.c_uint32, C.c_int, C.c_double, C.c_double, C.c_void_p]
        L.lb2_index_create_sq.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_int, C.c_int, C.c_double,
                                          C.c_double, C.POINTER(C.c_void_p)]
        L.lb2_rq_rotation.argtypes = [C.c_uint32, C.c_uint64, C.c_void_p]
        L.lb2_index_search_candidates.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p,
                                                  C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p,
                                                  C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.lb2_index_refine_taken.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint32, C.c_void_p,
                                             C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint32,
                                             C.c_void_p, C.c_void_p, C.c_void_p]
        L.lb2_flat_search_batch.argtypes = [C.c_void_p, C.c_uint64, C.c_uint32, C.c_int, C.c_int, C.c_void_p,
                                            C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32,
                                            C.c_void_p, C.c_void_p, C.c_void_p]
        L.lb2_index_search_combined_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p,
                                                      C.c_uint32, C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p,
                                                      C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        _lib = L
    return _lib


def check(status):
    if status != OK:
        buf = C.create_string_buffer(2048)
        lib().lb2_last_error(buf, 2048)
        raise LanceB200Error(status, buf.value.decode(errors="replace"))


def device_count():
    return int(lib().lb2_device_count())


class SearchParams(C.Structure):
    """lb2_search_params (include/lance_b200.h)."""
    _fields_ = [("k", C.c_uint32), ("nprobes", C.c_uint32), ("refine_factor", C.c_uint32),
                ("refine_vectors", C.c_void_p), ("num_vectors", C.c_uint64), ("allow_bitmap", C.c_void_p),
                ("has_lower_bound", C.c_uint32), ("has_upper_bound", C.c_uint32),
                ("lower_bound", C.c_float), ("upper_bound", C.c_float)]


class ProbeParams(C.Structure):
    """lb2_probe_params (include/lance_b200.h)."""
    _fields_ = [("minimum_nprobes", C.c_uint32), ("maximum_nprobes", C.c_uint32), ("late_width", C.c_uint32),
                ("has_max_len", C.c_uint32), ("max_len", C.c_uint64), ("mask_ids", C.c_void_p),
                ("num_mask_ids", C.c_uint64)]


class QueryFilter(C.Structure):
    """lb2_query_filter (include/lance_b200.h)."""
    _fields_ = [("allow_bitmap", C.c_void_p), ("has_max_len", C.c_uint32), ("max_len", C.c_uint64),
                ("mask_ids", C.c_void_p), ("num_mask_ids", C.c_uint64)]


class QueryParams(C.Structure):
    """lb2_query_params (include/lance_b200.h)."""
    _fields_ = [("k", C.c_uint32), ("nprobes", C.c_uint32), ("minimum_nprobes", C.c_uint32),
                ("maximum_nprobes", C.c_uint32), ("refine_factor", C.c_uint32), ("filter", C.c_uint32),
                ("ef", C.c_uint32), ("has_lower_bound", C.c_uint32), ("has_upper_bound", C.c_uint32),
                ("lower_bound", C.c_float), ("upper_bound", C.c_float)]


class FlatSearchParams(C.Structure):
    """lb2_flat_search_params (include/lance_b200.h)."""
    _fields_ = [("k", C.c_uint32), ("allow_bitmap", C.c_void_p), ("has_lower_bound", C.c_uint32),
                ("has_upper_bound", C.c_uint32), ("lower_bound", C.c_float), ("upper_bound", C.c_float)]


class UnindexedRows(C.Structure):
    """lb2_unindexed_rows (include/lance_b200.h)."""
    _fields_ = [("vectors", C.c_void_p), ("n", C.c_uint64), ("row_ids", C.c_void_p), ("allow_bitmap", C.c_void_p)]


class FlatQueryParams(C.Structure):
    """lb2_flat_query_params (include/lance_b200.h)."""
    _fields_ = [("k", C.c_uint32), ("filter", C.c_uint32), ("has_lower_bound", C.c_uint32),
                ("has_upper_bound", C.c_uint32), ("lower_bound", C.c_float), ("upper_bound", C.c_float)]


class UnindexedBatch(C.Structure):
    """lb2_unindexed_batch (include/lance_b200.h)."""
    _fields_ = [("rows", UnindexedRows), ("filter_bitmaps", C.c_void_p)]


class DeviceArray:
    """A typed, shaped view of device memory owned by this object (lb2_malloc / lb2_free)."""

    def __init__(self, shape, dtype):
        self.shape = tuple(int(s) for s in (shape if isinstance(shape, (tuple, list)) else (shape,)))
        self.dtype = np.dtype(dtype)
        self.nbytes = int(np.prod(self.shape, dtype=np.int64)) * self.dtype.itemsize
        p = C.c_void_p()
        check(lib().lb2_malloc(C.byref(p), C.c_size_t(self.nbytes)))
        self.ptr = p.value

    @classmethod
    def from_numpy(cls, a):
        a = np.ascontiguousarray(a)
        out = cls(a.shape, a.dtype)
        if a.nbytes:
            check(lib().lb2_memcpy(C.c_void_p(out.ptr), C.c_void_p(a.ctypes.data), C.c_size_t(a.nbytes)))
        return out

    def numpy(self):
        out = np.empty(self.shape, self.dtype)
        if self.nbytes:
            check(lib().lb2_memcpy(C.c_void_p(out.ctypes.data), C.c_void_p(self.ptr), C.c_size_t(self.nbytes)))
        return out

    def free(self):
        if getattr(self, "ptr", None):
            lib().lb2_free(C.c_void_p(self.ptr))
            self.ptr = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class PinnedArray:
    """numpy view over pinned host memory (lb2_malloc_host)."""

    def __init__(self, shape, dtype):
        self.shape = tuple(int(s) for s in (shape if isinstance(shape, (tuple, list)) else (shape,)))
        self.dtype = np.dtype(dtype)
        self.nbytes = int(np.prod(self.shape, dtype=np.int64)) * self.dtype.itemsize
        p = C.c_void_p()
        check(lib().lb2_malloc_host(C.byref(p), C.c_size_t(max(self.nbytes, 1))))
        self.ptr = p.value
        buf = (C.c_uint8 * max(self.nbytes, 1)).from_address(self.ptr)
        self.array = np.frombuffer(buf, dtype=self.dtype, count=int(np.prod(self.shape, dtype=np.int64))).reshape(self.shape)

    def free(self):
        if getattr(self, "ptr", None):
            self.array = None
            lib().lb2_free_host(C.c_void_p(self.ptr))
            self.ptr = None


def as_ptr(a):
    """(pointer, keepalive) for a numpy array, DeviceArray, PinnedArray or None."""
    if a is None:
        return None, None
    if isinstance(a, (DeviceArray, PinnedArray)):
        return C.c_void_p(a.ptr), a
    a = np.ascontiguousarray(a)
    return C.c_void_p(a.ctypes.data), a
