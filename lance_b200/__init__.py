"""lance_b200 -- H100-native IVF-PQ hot path behind lancedb/lance's own operator API.

Host-side mirror (Python, test/bench tooling) of the reference's
`lance-index::vector::{kmeans,ivf,pq,flat}` + `lance-linalg::distance` functions: same names,
argument meaning and error behaviour; every call goes straight through the C ABI
(include/lance_b200.h) into hand-written sm_90a kernels.  No CPU fallback exists.

Inputs may be numpy arrays (host memory) or `DeviceArray`s (resident in HBM).
"""
import ctypes as C

import numpy as np

from ._lib import (BF16, COSINE, DOT, F16, F32, L2, METRICS, U8, BuildParams, BuildStats, FlatBuildParams,
                   DeviceArray, KMeansParams as _CKMeansParams, LanceB200Error, PinnedArray,
                   PQParams as _CPQParams, RqBuildParams as _CRqBuildParams, SqBuildParams as _CSqBuildParams,
                   HnswSqBuildParams as _CHnswSqBuildParams, HnswPqBuildParams as _CHnswPqBuildParams,
                   HnswFlatBuildParams as _CHnswFlatBuildParams, IndexStorage as _CIndexStorage, as_ptr,
                   check, device_count, lib)

__all__ = ["device_count", "DeviceArray", "PinnedArray", "LanceB200Error", "train_kmeans",
           "compute_partitions", "kmeans_find_partitions", "compute_residual", "normalize_fsl",
           "l2_distance_batch", "dot_distance_batch", "cosine_distance_batch", "PQBuildParams", "ProductQuantizer",
           "build_distance_table_l2", "compute_pq_distance", "flat_topk", "flat_search", "flat_search_batch", "IvfPqIndex",
           "IvfBuildParams", "IvfFlatIndex", "SQBuildParams", "ScalarQuantizer", "IvfSqIndex", "HnswBuildParams",
           "IvfHnswSqIndex", "IvfHnswPqIndex", "IvfHnswFlatIndex", "RQBuildParams",
           "RabitQuantizer", "IvfRqIndex", "PartitionIndex", "launch_count", "profile"]


def _metric(m):
    if isinstance(m, str):
        return METRICS[m.lower()]
    return int(m)


def _shape2(a):
    return a.shape


def _f32(a):
    if isinstance(a, (DeviceArray, PinnedArray)):
        assert a.dtype == np.float32
        return a
    return np.ascontiguousarray(a, dtype=np.float32)


_DTYPES = {np.dtype(np.float32): F32, np.dtype(np.float16): F16, np.dtype(np.uint8): U8}


def _typed(a, bf16=False):
    """(array, lb2_dtype): f32 / f16 / u8 buffers are passed as they are (bf16 = uint16 + bf16=True)."""
    if bf16:
        if isinstance(a, (DeviceArray, PinnedArray)):
            assert np.dtype(a.dtype) == np.uint16
            return a, BF16
        return np.ascontiguousarray(a, dtype=np.uint16), BF16
    if isinstance(a, (DeviceArray, PinnedArray)):
        return a, _DTYPES[np.dtype(a.dtype)]
    a = np.asarray(a)
    if a.dtype not in _DTYPES:
        a = a.astype(np.float32)
    return np.ascontiguousarray(a), _DTYPES[a.dtype]


def _model_np(dt):
    return {F32: np.float32, F16: np.float16, BF16: np.uint16, U8: np.float32}[dt]


def _model_arr(a, dt):
    """a model array in the model type of `dt`; f32 arrays of a bf16 model (as exports return them) keep their bits"""
    a = np.asarray(a)
    if dt == BF16 and a.dtype == np.float32:
        return np.ascontiguousarray((np.ascontiguousarray(a).view(np.uint32) >> 16).astype(np.uint16))
    return np.ascontiguousarray(a, dtype=_model_np(dt))


def set_device(i):
    check(lib().lb2_set_device(C.c_int(i)))


def synchronize():
    check(lib().lb2_synchronize())


def trim_memory():
    """lb2_trim_memory: release this thread's cached bulk-copy staging buffer and the pool's free blocks."""
    check(lib().lb2_trim_memory())


def set_stream(cuda_stream=None):
    """lb2_set_stream: order every later call of this thread on a caller-owned cudaStream_t (int handle); None =
    back to the thread's private stream."""
    check(lib().lb2_set_stream(C.c_void_p(cuda_stream)))


def launch_count(reset=False):
    n = C.c_uint64(0)
    check(lib().lb2_launch_count(C.byref(n), C.c_int(int(reset))))
    return n.value


class profile:
    """Per-kernel-family CUDA-event timing (lb2_profile_*)."""

    @staticmethod
    def enable(on=True):
        check(lib().lb2_profile_enable(C.c_int(int(on))))

    @staticmethod
    def reset():
        check(lib().lb2_profile_reset())

    @staticmethod
    def dump():
        """{name: (launches, total_ms)} for every kernel family seen since the last reset"""
        n = lib().lb2_profile_dump(None, 0)
        buf = C.create_string_buffer(n + 1)
        lib().lb2_profile_dump(buf, n + 1)
        out = {}
        for line in buf.value.decode().splitlines():
            name, cnt, ms = line.split("\t")
            out[name] = (int(cnt), float(ms))
        return out

    @staticmethod
    def get(name):
        n, ms = C.c_uint64(0), C.c_double(0)
        check(lib().lb2_profile_get(name.encode(), C.byref(n), C.byref(ms)))
        return n.value, ms.value


def timer_start():
    check(lib().lb2_timer_start())


def timer_stop():
    ms = C.c_float(0)
    check(lib().lb2_timer_stop(C.byref(ms)))
    return ms.value


# ---- lance-linalg ---------------------------------------------------------------------------
def l2_distance_batch(frm, to, dimension, bf16=False):
    """lance_linalg::distance::l2_distance_batch (l2.rs:194-203)."""
    return _distance_batch(frm, to, dimension, L2, bf16)


def dot_distance_batch(frm, to, dimension, bf16=False):
    """lance_linalg::distance::dot_distance_batch (dot.rs:164-172): 1 - dot."""
    return _distance_batch(frm, to, dimension, DOT, bf16)


def cosine_distance_batch(frm, to, dimension, bf16=False):
    """lance_linalg::distance::cosine_distance_batch (cosine.rs:266-290)."""
    return _distance_batch(frm, to, dimension, COSINE, bf16)


def _distance_batch(frm, to, d, metric, bf16=False):
    """f32 / f16 / u8 inputs keep their element type, and so do bf16 ones given as uint16 bit patterns with
    bf16=True: the arithmetic is the reference's rule for that type (u8: exact integer sums, 16-bit dot: 32 lanes)."""
    to, dt = _typed(to, bf16)
    frm = np.ascontiguousarray(frm, dtype=to.dtype) if not isinstance(frm, (DeviceArray, PinnedArray)) else frm
    n = int(np.prod(to.shape)) // d
    out = np.empty(n, np.float32)
    fp, _k1 = as_ptr(frm)
    tp, _k2 = as_ptr(to)
    check(lib().lb2_distance_batch(fp, tp, C.c_uint64(n), C.c_uint32(d), C.c_int(dt),
                                   C.c_int(metric), C.c_void_p(out.ctypes.data)))
    return out


def normalize_fsl(vectors, bf16=False):
    """lance_linalg::kernels::normalize_fsl (kernels.rs:201-211).  The result has the model type: the input's own
    type for f32 / f16 / bf16 (bf16=True: uint16 bit patterns), f32 for u8."""
    vectors, dt = _typed(vectors, bf16)
    n, d = vectors.shape
    out = np.empty((n, d), _model_np(dt))
    vp, _k = as_ptr(vectors)
    check(lib().lb2_normalize(vp, C.c_uint64(n), C.c_uint32(d), C.c_int(dt),
                              C.c_void_p(out.ctypes.data)))
    return out


# ---- lance-index::vector::kmeans -------------------------------------------------------------
class KMeans:
    """Result of train_kmeans (kmeans.rs:527-545: centroids, dimension, distance_type, loss)."""

    def __init__(self, centroids, dimension, distance_type, loss, iters):
        self.centroids, self.dimension, self.distance_type = centroids, dimension, distance_type
        self.loss, self.iters = loss, iters


def train_kmeans(array, dimension, k, max_iters=50, redos=1, distance_type="l2", sample_rate=256,
                 balance_factor=0.0, tolerance=1e-4, seed=0, centroids=None, hierarchical_k=16):
    """lance_index::vector::kmeans::train_kmeans (kmeans.rs:1309-1347).
    hierarchical_k: branching of the hierarchical scheme used for k > 256 without `centroids`; 0 or 1 = flat Lloyd."""
    array, dt = _typed(array)
    n = int(np.prod(array.shape)) // dimension
    p = _CKMeansParams()
    lib().lb2_kmeans_params_default(C.byref(p))
    p.max_iters, p.redos, p.sample_rate, p.seed = max_iters, redos, sample_rate, seed
    p.hierarchical_k = hierarchical_k
    p.balance_factor, p.tolerance, p.metric = balance_factor, tolerance, _metric(distance_type)
    init = None if centroids is None else np.ascontiguousarray(centroids, dtype=_model_np(dt))
    ip, _k0 = as_ptr(init)
    p.init_centroids = ip.value if ip is not None else None
    out = np.empty((k, dimension), _model_np(dt))
    loss, iters = C.c_double(0), C.c_uint32(0)
    ap, _k1 = as_ptr(array)
    check(lib().lb2_kmeans_train(ap, C.c_uint64(n), C.c_uint32(dimension), C.c_int(dt),
                                 C.c_uint32(k), C.byref(p), C.c_void_p(out.ctypes.data),
                                 C.byref(loss), C.byref(iters)))
    return KMeans(out, dimension, distance_type, loss.value, iters.value)


def compute_partitions(centroids, vectors, distance_type="l2", bf16=False):
    """compute_partitions_arrow_array (kmeans.rs:1187-1246) ->
    (part_ids u32[n], dists f32[n], valid bool[n]); valid False == the reference's None.
    The model has the rows' element type (bf16=True: both are uint16 bit patterns)."""
    vectors, dt = _typed(vectors, bf16)
    centroids = np.ascontiguousarray(centroids, dtype=_model_np(dt))
    k, d = centroids.shape
    n = vectors.shape[0]
    part = np.empty(n, np.uint32)
    dist = np.empty(n, np.float32)
    valid = np.empty(n, np.uint8)
    cp, _k1 = as_ptr(centroids)
    vp, _k2 = as_ptr(vectors)
    check(lib().lb2_compute_partitions(cp, C.c_uint32(k), C.c_uint32(d), C.c_int(dt),
                                       C.c_int(_metric(distance_type)), vp, C.c_uint64(n),
                                       C.c_void_p(part.ctypes.data), C.c_void_p(dist.ctypes.data),
                                       C.c_void_p(valid.ctypes.data)))
    return part, dist, valid.astype(bool)


def kmeans_find_partitions(centroids, queries, nprobes, distance_type="l2", bf16=False):
    """kmeans_find_partitions_arrow_array (kmeans.rs:1076-1158), batched over queries.  The queries keep their element
    type (bf16=True: uint16 bit patterns); the centroids are given in the model type."""
    queries, dt = _typed(queries, bf16)
    centroids = np.ascontiguousarray(centroids, dtype=_model_np(dt))
    single = len(queries.shape) == 1
    k, d = centroids.shape
    nq = 1 if single else queries.shape[0]
    ids = np.empty((nq, nprobes), np.uint32)
    dists = np.empty((nq, nprobes), np.float32)
    cp, _k1 = as_ptr(centroids)
    qp, _k2 = as_ptr(queries)
    check(lib().lb2_find_partitions(cp, C.c_uint32(k), C.c_uint32(d), C.c_int(dt),
                                    C.c_int(_metric(distance_type)), qp, C.c_uint64(nq),
                                    C.c_uint32(nprobes), C.c_void_p(ids.ctypes.data),
                                    C.c_void_p(dists.ctypes.data)))
    return (ids[0], dists[0]) if single else (ids, dists)


def compute_residual(centroids, vectors, partitions, bf16=False):
    """lance_index::vector::residual::compute_residual (residual.rs:111-154).  The vectors keep their element type
    (bf16=True: uint16 bit patterns); centroids and residuals have the model type."""
    vectors, dt = _typed(vectors, bf16)
    centroids = np.ascontiguousarray(centroids, dtype=_model_np(dt))
    k, d = centroids.shape
    n = vectors.shape[0]
    parts = np.ascontiguousarray(partitions, dtype=np.uint32)
    out = np.empty((n, d), _model_np(dt))
    cp, _k1 = as_ptr(centroids)
    vp, _k2 = as_ptr(vectors)
    check(lib().lb2_compute_residual(cp, C.c_uint32(k), C.c_uint32(d), C.c_int(dt), vp,
                                     C.c_uint64(n), C.c_void_p(parts.ctypes.data),
                                     C.c_void_p(out.ctypes.data)))
    return out


# ---- lance-index::vector::utils: SimpleIndex, the HNSW graph over the centroids ----------------------------
PARTITION_INDEX_MODES = {"exact": 0, "auto": 1, "hnsw": 2}


def _pi_mode(mode):
    if mode not in PARTITION_INDEX_MODES:
        raise ValueError(f"partition index mode {mode!r}: one of {sorted(PARTITION_INDEX_MODES)}")
    return PARTITION_INDEX_MODES[mode]


class PartitionIndex:
    """SimpleIndex (lance-index/src/vector/utils.rs:26-108): an HNSW graph over the IVF centroids that assigns each row
    by one graph search (k = 1, ef = 15) instead of the exact scan.  mode is LANCE_USE_HNSW_SPEEDUP_INDEXING's value:
    "exact" (disabled, the default), "auto" (unset: the graph when k * d >= 1 000 000) or "hnsw" (enabled).  Only f32
    models have a graph (u8 columns have f32 models); f16 / bf16 models, like "exact", assign by the exact scan
    (compute_partitions).  Cosine columns are normalised by the caller and assigned under "l2"."""

    def __init__(self, handle, centroids, dtype, distance_type):
        self._h, self._centroids, self._dt, self.distance_type = handle, centroids, dtype, distance_type

    @staticmethod
    def uses_graph(k, d, mode="auto", dtype=np.float32, bf16=False):
        """may_train_index's decision (utils.rs:67-91) for a k x d model over columns of `dtype`; host only"""
        dt = BF16 if bf16 else _DTYPES[np.dtype(dtype)]
        out = C.c_int()
        check(lib().lb2_partition_index_uses_graph(C.c_uint64(k), C.c_uint32(d), C.c_int(dt), C.c_int(_pi_mode(mode)),
                                                   C.byref(out)))
        return bool(out.value)

    @classmethod
    def build(cls, centroids, distance_type="l2", mode="hnsw", seed=0, insert_batch=1, dtype=np.float32, bf16=False):
        """lb2_partition_index_build over the model `centroids` [k][d] of a column of element type `dtype` (bf16=True:
        a bf16 column, uint16 bit patterns).  The graph (when the mode resolves to it) levels nodes with seed and is
        built serially (insert_batch 1) or in rounds of insert_batch concurrent inserts."""
        dt = BF16 if bf16 else _DTYPES[np.dtype(dtype)]
        centroids = np.ascontiguousarray(centroids, dtype=_model_np(dt))
        k, d = centroids.shape
        h = C.c_void_p()
        check(lib().lb2_partition_index_build(C.c_void_p(centroids.ctypes.data), C.c_uint32(k), C.c_uint32(d),
                                              C.c_int(dt), C.c_int(_metric(distance_type)), C.c_int(_pi_mode(mode)),
                                              C.c_uint64(seed), C.c_uint32(insert_batch), C.byref(h)))
        return cls(h if h.value else None, centroids, dt, distance_type)

    @property
    def has_graph(self):
        return self._h is not None

    def assign(self, vectors):
        """lb2_partition_index_assign -> (part_ids u32[n], dists f32[n], valid bool[n]); without a graph this is
        compute_partitions.  vectors: the column's rows (numpy, DeviceArray or PinnedArray), in its element type."""
        vectors, dt = _typed(vectors, self._dt == BF16)
        k, d = self._centroids.shape
        n = vectors.shape[0]
        part = np.empty(n, np.uint32)
        dist = np.empty(n, np.float32)
        valid = np.empty(n, np.uint8)
        vp, _keep = as_ptr(vectors)
        check(lib().lb2_partition_index_assign(self._h, C.c_void_p(self._centroids.ctypes.data), C.c_uint32(k),
                                               C.c_uint32(d), C.c_int(dt), C.c_int(_metric(self.distance_type)), vp,
                                               C.c_uint64(n), C.c_void_p(part.ctypes.data),
                                               C.c_void_p(dist.ctypes.data), C.c_void_p(valid.ctypes.data)))
        return part, dist, valid.astype(bool)

    def export(self):
        """the graph in IvfHnswFlatIndex.export()["graph"]'s layout (one partition of k rows), or None without one"""
        if self._h is None:
            return None
        k, d, ml, m, efc, nu = (C.c_uint32(), C.c_uint32(), C.c_uint32(), C.c_uint32(), C.c_uint32(), C.c_uint64())
        check(lib().lb2_partition_index_info(self._h, C.byref(k), C.byref(d), C.byref(ml), C.byref(m), C.byref(efc),
                                             C.byref(nu)))
        n, m, nu = k.value, m.value, nu.value
        g = dict(max_level=ml.value, m=m, ef_construction=efc.value, levels=np.empty(n, np.uint8),
                 counts0=np.empty(n, np.uint32), neighbors0=np.empty((n, 2 * m), np.uint32),
                 dists0=np.empty((n, 2 * m), np.float32), counts_up=np.empty(nu, np.uint32),
                 neighbors_up=np.empty((nu, m), np.uint32), dists_up=np.empty((nu, m), np.float32))
        ptr = {key: C.c_void_p(v.ctypes.data) if isinstance(v, np.ndarray) and v.size else None for key, v in g.items()}
        check(lib().lb2_partition_index_export(self._h, ptr["levels"], ptr["counts0"], ptr["neighbors0"],
                                               ptr["dists0"], ptr["counts_up"], ptr["neighbors_up"], ptr["dists_up"]))
        return g

    def close(self):
        if self._h is not None:
            lib().lb2_partition_index_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


# ---- lance-index::vector::pq -----------------------------------------------------------------
class PQBuildParams:
    """lance_index::vector::pq::builder::PQBuildParams (pq/builder.rs:27-59)."""

    def __init__(self, num_sub_vectors=16, num_bits=8, max_iters=50, kmeans_redos=1, codebook=None,
                 sample_rate=256, seed=0):
        self.num_sub_vectors, self.num_bits, self.max_iters = num_sub_vectors, num_bits, max_iters
        self.kmeans_redos, self.codebook, self.sample_rate, self.seed = kmeans_redos, codebook, sample_rate, seed

    def _c(self):
        p = _CPQParams()
        lib().lb2_pq_params_default(C.byref(p))
        p.num_sub_vectors, p.num_bits, p.max_iters = self.num_sub_vectors, self.num_bits, self.max_iters
        p.kmeans_redos, p.sample_rate, p.seed = self.kmeans_redos, self.sample_rate, self.seed
        self._cb = None if self.codebook is None else _f32(self.codebook)
        cp, _ = as_ptr(self._cb)
        p.codebook = cp.value if cp is not None else None
        return p

    def build(self, data, distance_type="l2"):
        """PQBuildParams::build (pq/builder.rs:162-194) -> ProductQuantizer."""
        data = _f32(data)
        n, d = data.shape
        p = self._c()
        out = np.empty((self.num_sub_vectors, 1 << self.num_bits, d // self.num_sub_vectors), np.float32)
        iters = np.zeros(self.num_sub_vectors, np.uint32)
        dp, _k = as_ptr(data)
        check(lib().lb2_pq_train(dp, C.c_uint64(n), C.c_uint32(d), C.c_int(F32),
                                 C.c_int(_metric(distance_type)), C.byref(p),
                                 C.c_void_p(out.ctypes.data), C.c_void_p(iters.ctypes.data)))
        pq = ProductQuantizer(self.num_sub_vectors, self.num_bits, d, out, distance_type)
        pq.train_iters = iters
        return pq


class ProductQuantizer:
    """lance_index::vector::pq::ProductQuantizer (pq.rs:42-48); codebook [M][2^nbits][d/M]."""

    def __init__(self, num_sub_vectors, num_bits, dimension, codebook, distance_type="l2"):
        self.num_sub_vectors, self.num_bits, self.dimension = num_sub_vectors, num_bits, dimension
        self.codebook = _f32(codebook).reshape(num_sub_vectors, 1 << num_bits, dimension // num_sub_vectors)
        self.distance_type = distance_type

    def quantize(self, vectors, centroids=None, part_ids=None):
        """Quantization::quantize (pq.rs:430) = transform_impl (pq.rs:116-191); with
        centroids+part_ids the residual transform (residual.rs:161-205) is fused in."""
        vectors = _f32(vectors)
        n, d = vectors.shape
        out = np.empty((n, self.num_sub_vectors // 2 if self.num_bits == 4 else self.num_sub_vectors), np.uint8)
        cent = None if centroids is None else _f32(centroids)
        parts = None if part_ids is None else np.ascontiguousarray(part_ids, dtype=np.uint32)
        vp, _k1 = as_ptr(vectors)
        cp, _k2 = as_ptr(cent)
        pp, _k3 = as_ptr(parts)
        check(lib().lb2_pq_encode(C.c_void_p(self.codebook.ctypes.data), C.c_uint32(self.num_sub_vectors),
                                  C.c_uint32(self.num_bits), C.c_uint32(d), C.c_int(F32),
                                  C.c_int(_metric(self.distance_type)), cp,
                                  C.c_uint32(0 if cent is None else cent.shape[0]), pp, vp, C.c_uint64(n),
                                  C.c_void_p(out.ctypes.data)))
        return out


def build_distance_table_l2(codebook, num_bits, num_sub_vectors, query, distance_type="l2"):
    """lance_index::vector::pq::distance::build_distance_table_l2 / _dot (pq/distance.rs:24-92)."""
    codebook, query = _f32(codebook), _f32(query)
    d = query.size
    out = np.empty(num_sub_vectors << num_bits, np.float32)
    check(lib().lb2_pq_build_lut(C.c_void_p(codebook.ctypes.data), C.c_uint32(num_sub_vectors),
                                 C.c_uint32(num_bits), C.c_uint32(d), C.c_int(_metric(distance_type)),
                                 C.c_void_p(query.ctypes.data), C.c_void_p(out.ctypes.data)))
    return out


def compute_pq_distance(distance_table, num_bits, num_sub_vectors, code_transposed, distance_type="l2"):
    """pq/distance.rs:109-144 on transposed codes [M][n]."""
    lut = _f32(distance_table)
    code = np.ascontiguousarray(code_transposed, dtype=np.uint8)
    n = code.size // num_sub_vectors
    out = np.empty(n, np.float32)
    check(lib().lb2_pq_scan(C.c_void_p(lut.ctypes.data), C.c_uint32(num_sub_vectors),
                            C.c_uint32(num_bits), C.c_int(_metric(distance_type)),
                            C.c_void_p(code.ctypes.data), C.c_uint64(n), C.c_void_p(out.ctypes.data)))
    return out


def compute_pq_distance_4bit(distance_table, num_sub_vectors, code_transposed, k_hint, distance_type="l2"):
    """pq/distance.rs:147-242 on transposed packed codes [M/2][n]; distance_table [M][16]."""
    lut = _f32(distance_table)
    code = np.ascontiguousarray(code_transposed, dtype=np.uint8)
    n = code.size // (num_sub_vectors // 2)
    out = np.empty(n, np.float32)
    check(lib().lb2_pq_scan_4bit(C.c_void_p(lut.ctypes.data), C.c_uint32(num_sub_vectors),
                                 C.c_int(_metric(distance_type)), C.c_void_p(code.ctypes.data), C.c_uint64(n),
                                 C.c_uint64(k_hint), C.c_void_p(out.ctypes.data)))
    return out


def flat_topk(dists, row_ids, k, lower_bound=None, upper_bound=None):
    """FlatIndex::search fast path (flat/index.rs:97-127) over a distance array, optionally with the
    range branch (:100-115)."""
    dists = _f32(dists)
    n = dists.size
    rid = None if row_ids is None else np.ascontiguousarray(row_ids, dtype=np.uint64)
    oi, od, cnt = np.empty(k, np.uint64), np.empty(k, np.float32), np.zeros(1, np.uint32)
    rp, _k = as_ptr(rid)
    check(lib().lb2_flat_topk_range(C.c_void_p(dists.ctypes.data), rp, C.c_uint64(n), C.c_uint32(k),
                                    C.c_int(lower_bound is not None), C.c_float(lower_bound or 0.0),
                                    C.c_int(upper_bound is not None), C.c_float(upper_bound or 0.0),
                                    C.c_void_p(oi.ctypes.data), C.c_void_p(od.ctypes.data),
                                    C.c_void_p(cnt.ctypes.data)))
    return oi[:cnt[0]], od[:cnt[0]]


def _bitmap(a):
    """an allow bitmap (uint64 words) as numpy / Pinned / Device array, or None"""
    if a is None or isinstance(a, (DeviceArray, PinnedArray)):
        return a
    return np.ascontiguousarray(a, dtype=np.uint64)


def _row_ids(a):
    if a is None or isinstance(a, (DeviceArray, PinnedArray)):
        return a
    return np.ascontiguousarray(a, dtype=np.uint64)


def flat_search(vectors, queries, k, distance_type="l2", row_ids=None, allow_bitmap=None, lower_bound=None,
                upper_bound=None, bf16=False):
    """flat_knn over one vector column (scanner.rs:3336-3411), batched: the k smallest (distance, row id) pairs of
    every query, with compute_distance's arithmetic for the column's element type (flat.rs:94-150).  `vectors` [n][d]
    and `queries` [nq][d] share the element type (bf16=True: uint16 bit patterns); row_ids (distinct) default to the
    row numbers; allow_bitmap: (n + 63) // 64 uint64 words, bit i = row i may be returned (validity AND filter);
    the range keeps lower <= distance < upper.  Returns (ids [nq][k], dists [nq][k], counts [nq]); unused slots hold
    (2**64 - 1, +inf)."""
    from ._lib import FlatSearchParams
    vectors, dt = _typed(vectors, bf16)
    if not isinstance(queries, (DeviceArray, PinnedArray)):
        queries = np.ascontiguousarray(queries, dtype=vectors.dtype)
    n, d = vectors.shape
    nq = queries.shape[0]
    ids, dists, counts = np.empty((nq, k), np.uint64), np.empty((nq, k), np.float32), np.empty(nq, np.uint32)
    vp, _k0 = as_ptr(vectors)
    qp, _k1 = as_ptr(queries)
    rp, _k2 = as_ptr(_row_ids(row_ids))
    bp, _k3 = as_ptr(_bitmap(allow_bitmap))
    p = FlatSearchParams(k, bp.value if bp is not None else None, int(lower_bound is not None),
                         int(upper_bound is not None), float(lower_bound or 0.0), float(upper_bound or 0.0))
    check(lib().lb2_flat_search(vp, C.c_uint64(n), C.c_uint32(d), C.c_int(dt), C.c_int(_metric(distance_type)), rp,
                                qp, C.c_uint64(nq), C.byref(p), as_ptr(ids)[0], as_ptr(dists)[0], as_ptr(counts)[0]))
    return ids, dists, counts


def _per_query(name, what, v, nq, dtype, default):
    """a per-query argument: a scalar broadcast to [nq], or an [nq] array"""
    a = np.asarray(default if v is None else v, dtype=dtype)
    if a.ndim == 0:
        return np.full(nq, a, dtype)
    if a.shape != (nq,):
        raise ValueError(f"{name}: {what} must be a scalar or an array of {nq} values, got shape {a.shape}")
    return a


def _out_rows(name, out, nq, kmax):
    """(ids, dists, k_stride): `out`'s arrays, or new [nq][kmax] ones"""
    if out is None:
        ids, dists = np.empty((nq, kmax), np.uint64), np.empty((nq, kmax), np.float32)
    else:
        ids, dists = out
    k_stride = int(ids.shape[1]) if len(ids.shape) == 2 else kmax
    if tuple(ids.shape) != (nq, k_stride) or tuple(dists.shape) != (nq, k_stride) or k_stride < kmax:
        raise ValueError(f"{name}: out arrays must be [{nq}][>= {kmax}], got {ids.shape} and {dists.shape}")
    return ids, dists, k_stride


def _bitmap_table(bitmaps, keep):
    """a C array of bitmap pointers (NULL for a None entry), with what it points at appended to keep"""
    table = (C.c_void_p * max(1, len(bitmaps)))()
    for i, b in enumerate(bitmaps):
        bp, kb = as_ptr(_bitmap(b))
        if bp is not None and bp.value is None:  # an empty numpy array has no buffer address to pass
            kb = np.zeros(1, np.uint64)
            bp = C.c_void_p(kb.ctypes.data)
        keep += [b, kb]
        table[i] = bp.value if bp is not None else None
    return table


def flat_search_batch(vectors, queries, k, distance_type="l2", row_ids=None, filters=None, filter_of=None,
                      lower_bound=None, upper_bound=None, out=None, bf16=False):
    """lb2_flat_search_batch: flat_search where every query has its own k, range and filter, in one call.  Row q
    equals flat_search of query q alone with k[q], filters[filter_of[q]] as its allow bitmap (-1 = none) and its
    bounds (NaN or None = no bound).  Every per-query argument is a scalar or an [nq] array; `filters` is a list of
    allow bitmaps over the n rows ((n + 63) // 64 uint64 words; None admits every row).  Returns (ids, dists,
    counts): ids / dists [nq][max k] (or `out`'s arrays and their row length); unused slots hold (2**64 - 1, +inf)."""
    from ._lib import FlatQueryParams
    vectors, dt = _typed(vectors, bf16)
    if not isinstance(queries, (DeviceArray, PinnedArray)):
        queries = np.ascontiguousarray(queries, dtype=vectors.dtype)
    n, d = vectors.shape
    nq = int(queries.shape[0])
    name = "flat_search_batch"
    ks = _per_query(name, "k", k, nq, np.int64, 0)
    if nq and (ks < 1).any():
        raise ValueError(f"{name}: every k must be at least 1")
    filters = list(filters or [])
    fof = _per_query(name, "filter_of", filter_of, nq, np.int64, -1)
    if ((fof < -1) | (fof >= len(filters))).any():
        raise ValueError(f"{name}: filter_of must be -1 or below the {len(filters)} filters")
    lows = _per_query(name, "lower_bound", lower_bound, nq, np.float32, np.nan)
    ups = _per_query(name, "upper_bound", upper_bound, nq, np.float32, np.nan)
    ids, dists, k_stride = _out_rows(name, out, nq, int(ks.max()) if nq else 1)
    cp = np.zeros(max(1, nq), np.dtype({"names": [f for f, _ in FlatQueryParams._fields_],
                                        "formats": [np.float32 if t is C.c_float else np.uint32
                                                    for _, t in FlatQueryParams._fields_]}))
    assert cp.dtype.itemsize == C.sizeof(FlatQueryParams)
    cp["k"][:nq] = ks
    cp["filter"][:nq] = np.where(fof < 0, 0xFFFFFFFF, fof)
    cp["has_lower_bound"][:nq], cp["has_upper_bound"][:nq] = ~np.isnan(lows), ~np.isnan(ups)
    cp["lower_bound"][:nq], cp["upper_bound"][:nq] = np.nan_to_num(lows, nan=0.0), np.nan_to_num(ups, nan=0.0)
    keep = []
    table = _bitmap_table(filters, keep)
    counts = np.empty(nq, np.uint32)
    vp, _k0 = as_ptr(vectors)
    qp, _k1 = as_ptr(queries)
    rp, _k2 = as_ptr(_row_ids(row_ids))
    check(lib().lb2_flat_search_batch(vp, C.c_uint64(n), C.c_uint32(d), C.c_int(dt), C.c_int(_metric(distance_type)),
                                      rp, qp, C.c_uint64(nq), C.c_void_p(cp.ctypes.data), table,
                                      C.c_uint32(len(filters)), C.c_uint32(k_stride), as_ptr(ids)[0],
                                      as_ptr(dists)[0], as_ptr(counts)[0]))
    return ids, dists, counts


def ivfpq_transform(centroids, codebook, vectors, distance_type="l2", num_bits=8, bf16=False):
    """IvfTransformer::transform for IVF_PQ (lance-index/src/vector/ivf.rs:188-236,357).
    The rows keep their element type; the model has the rows' model type (bf16=True: uint16 bit patterns)."""
    vectors, dt = _typed(vectors, bf16)
    centroids = np.ascontiguousarray(centroids, dtype=_model_np(dt))
    codebook = np.ascontiguousarray(codebook, dtype=_model_np(dt))
    k, d = centroids.shape
    M = codebook.shape[0]
    n = vectors.shape[0]
    part, codes, valid = np.empty(n, np.uint32), np.empty((n, M // 2 if num_bits == 4 else M), np.uint8), np.empty(n, np.uint8)
    cp, _k1 = as_ptr(centroids)
    bp, _k2 = as_ptr(codebook)
    vp, _k3 = as_ptr(vectors)
    check(lib().lb2_ivfpq_transform(cp, C.c_uint32(k), bp, C.c_uint32(M), C.c_uint32(num_bits),
                                    C.c_uint32(d), C.c_int(dt), C.c_int(_metric(distance_type)), vp,
                                    C.c_uint64(n), C.c_void_p(part.ctypes.data),
                                    C.c_void_p(codes.ctypes.data), C.c_void_p(valid.ctypes.data)))
    return part, codes, valid.astype(bool)


# ---- the index (rust/lance/src/index/vector/{builder.rs, ivf/v2.rs}) ---------------------------
class IvfBuildParams:
    """lance_index::vector::ivf::builder::IvfBuildParams (ivf/builder.rs:20-78) + PQBuildParams."""

    def __init__(self, num_partitions=256, num_sub_vectors=16, num_bits=8, max_iters=50,
                 sample_rate=256, pq_max_iters=50, pq_sample_rate=256, seed=0, centroids=None,
                 codebook=None, partition_index="exact", partition_index_batch=1):
        self.num_partitions, self.num_sub_vectors, self.num_bits = num_partitions, num_sub_vectors, num_bits
        self.max_iters, self.sample_rate, self.pq_max_iters = max_iters, sample_rate, pq_max_iters
        self.pq_sample_rate, self.seed, self.centroids, self.codebook = pq_sample_rate, seed, centroids, codebook
        # how the full pass assigns rows (PartitionIndex's modes: "exact", "auto", "hnsw") and the graph's insert_batch
        self.partition_index, self.partition_index_batch = partition_index, partition_index_batch


def _ivf_fields(bp, num_partitions, max_iters, sample_rate, seed, centroids, partition_index, partition_index_batch):
    """the IVF fields of a build's parameters (num_partitions, ivf, seed); returns the centroid array bp points into
    (keep it alive across the build)"""
    bp.num_partitions = num_partitions
    bp.ivf.max_iters, bp.ivf.sample_rate, bp.ivf.seed, bp.seed = max_iters, sample_rate, seed, seed
    bp.ivf.partition_index = _pi_mode(partition_index)
    bp.ivf.partition_index_batch = partition_index_batch
    if centroids is None:
        return None
    keep = _f32(centroids)
    bp.ivf.init_centroids = as_ptr(keep)[0].value
    return keep


def _hnsw_fields(bp, hnsw_params):
    """the graph fields of an IVF_HNSW_* build's parameters"""
    hnsw_params = hnsw_params or HnswBuildParams()
    bp.max_level, bp.m, bp.ef_construction = hnsw_params.max_level, hnsw_params.m, hnsw_params.ef_construction
    bp.insert_batch = hnsw_params.insert_batch


def _build(cls, build_fn, bp, data, distance_type, row_ids, bf16=False):
    """cls(handle, stats) of the C build `build_fn` of `data` with the parameters bp"""
    data, dt = _typed(data, bf16)
    n, d = data.shape
    rid = None if row_ids is None else (row_ids if isinstance(row_ids, (DeviceArray, PinnedArray))
                                        else np.ascontiguousarray(row_ids, dtype=np.uint64))
    h, st = C.c_void_p(), BuildStats()
    dp, _k1 = as_ptr(data)
    rp, _k2 = as_ptr(rid)
    check(build_fn(dp, C.c_uint64(n), C.c_uint32(d), C.c_int(dt), C.c_int(_metric(distance_type)), C.byref(bp), rp,
                   C.byref(h), C.byref(st)))
    ix = cls(h, st)
    ix._dt = dt
    return ix


def _fill_build_params(bp, params):
    """lb2_ivfpq_build_params from IvfBuildParams; returns the arrays bp points into (keep them alive)"""
    keep = [_ivf_fields(bp, params.num_partitions, params.max_iters, params.sample_rate, params.seed, params.centroids,
                        getattr(params, "partition_index", "exact"), getattr(params, "partition_index_batch", 1))]
    bp.pq.num_sub_vectors, bp.pq.num_bits = params.num_sub_vectors, params.num_bits
    bp.pq.max_iters, bp.pq.sample_rate, bp.pq.seed = params.pq_max_iters, params.pq_sample_rate, params.seed + 1000
    if params.codebook is not None:
        c = _f32(params.codebook)
        keep.append(c)
        bp.pq.codebook = as_ptr(c)[0].value
    return keep


class IvfPqIndex:
    """Device-resident IVFIndex<FlatIndex, ProductQuantizer> (ivf/v2.rs:104)."""

    def __init__(self, handle, stats=None):
        self._h = handle
        self.stats = stats

    @classmethod
    def build(cls, data, distance_type="l2", params=None, row_ids=None, bf16=False):
        """IvfIndexBuilder::build (builder.rs:236): create_index("IVF_PQ").
        bf16=True: `data` is a uint16 array holding bfloat16 bit patterns (numpy has no bf16 dtype)."""
        bp = BuildParams()
        lib().lb2_ivfpq_build_params_default(C.byref(bp))
        keep = _fill_build_params(bp, params or IvfBuildParams())  # noqa: F841 (alive across the build)
        return _build(cls, lib().lb2_ivfpq_build, bp, data, distance_type, row_ids, bf16)

    @classmethod
    def from_parts(cls, centroids, codebook, part_ids, codes, row_ids=None, distance_type="l2", num_bits=8):
        """Open an index from a trained model + the shuffle output (user-supplied
        ivf_centroids / pq_codebook / precomputed buffers, ivf/builder.rs:20-60)."""
        centroids, codebook = _f32(centroids), _f32(codebook)
        k, d = centroids.shape
        M = codebook.shape[0]
        h = C.c_void_p()
        check(lib().lb2_index_create(C.c_void_p(centroids.ctypes.data), C.c_uint32(k), C.c_uint32(d),
                                     C.c_int(F32), C.c_int(_metric(distance_type)),
                                     C.c_void_p(codebook.ctypes.data), C.c_uint32(M),
                                     C.c_uint32(num_bits), C.byref(h)))
        ix = cls(h)
        part_ids = np.ascontiguousarray(part_ids, dtype=np.uint32)
        codes = np.ascontiguousarray(codes, dtype=np.uint8)
        rid = None if row_ids is None else np.ascontiguousarray(row_ids, dtype=np.uint64)
        rp, _k = as_ptr(rid)
        check(lib().lb2_index_load(h, C.c_void_p(part_ids.ctypes.data), C.c_void_p(codes.ctypes.data),
                                   rp, C.c_uint64(part_ids.size)))
        return ix

    def info(self):
        k, d, M, nb, n = C.c_uint32(), C.c_uint32(), C.c_uint32(), C.c_uint32(), C.c_uint64()
        check(lib().lb2_index_info(self._h, C.byref(k), C.byref(d), C.byref(M), C.byref(nb), C.byref(n)))
        return dict(num_partitions=k.value, dimension=d.value, num_sub_vectors=M.value,
                    num_bits=nb.value, num_rows=n.value)

    def export(self, out=None):
        """lb2_index_export; `out` = dict of preallocated arrays (same keys) to write into."""
        i = self.info()
        K, d, M, n = i["num_partitions"], i["dimension"], i["num_sub_vectors"], i["num_rows"]
        if out is not None:
            cent, cb, off, codes, rid = (out[k] for k in ("centroids", "codebook", "part_offsets", "codes", "row_ids"))
        else:
            cent = np.empty((K, d), np.float32)
            nbits = i["num_bits"]
            cb = np.empty((M, 1 << nbits, d // M), np.float32)
            off = np.empty(K + 1, np.uint64)
            codes = np.empty((n, M // 2 if nbits == 4 else M), np.uint8)   # 4-bit: two codes per byte
            rid = np.empty(n, np.uint64)
        check(lib().lb2_index_export(self._h, C.c_void_p(cent.ctypes.data), C.c_void_p(cb.ctypes.data),
                                     C.c_void_p(off.ctypes.data), C.c_void_p(codes.ctypes.data),
                                     C.c_void_p(rid.ctypes.data)))
        return dict(centroids=cent, codebook=cb, part_offsets=off, codes=codes, row_ids=rid)

    def export_partition_transposed(self, partition):
        """lb2_index_export_partition: (codes [code bytes][n_p] column-major, row_ids [n_p]) -- the reference's
        storage / index-file layout of one partition (pq/storage.rs:430-450)."""
        i = self.info()
        cw = i["num_sub_vectors"] // 2 if i["num_bits"] == 4 else i["num_sub_vectors"]
        n = C.c_uint64(0)
        check(lib().lb2_index_export_partition(self._h, C.c_uint32(partition), None, None, C.byref(n)))
        codes, rid = np.empty((cw, n.value), np.uint8), np.empty(n.value, np.uint64)
        check(lib().lb2_index_export_partition(self._h, C.c_uint32(partition), C.c_void_p(codes.ctypes.data),
                                               C.c_void_p(rid.ctypes.data), C.byref(n)))
        return codes, rid

    def search(self, queries, k=10, nprobes=1, out=None):
        """to_table(nearest={q,k,nprobes}) for a batch of queries: IVFIndex::find_partitions +
        search_in_partition + global merge (v2.rs:455-500, scanner.rs:3450-3466).
        `out` = optional (row_ids, dists) arrays (numpy/Pinned/Device) to write into."""
        dt = getattr(self, "_dt", F32)
        if isinstance(queries, (DeviceArray, PinnedArray)):
            assert np.dtype(queries.dtype).itemsize == {F32: 4, F16: 2, BF16: 2, U8: 1}[dt]
        else:
            queries = np.ascontiguousarray(queries, dtype={F32: np.float32, F16: np.float16, U8: np.uint8, BF16: np.uint16}[dt])
        nq = queries.shape[0]
        if out is None:
            ids, dists = np.empty((nq, k), np.uint64), np.empty((nq, k), np.float32)
        else:
            ids, dists = out
        qp, _k1 = as_ptr(queries)
        ip, _k2 = as_ptr(ids)
        dp, _k3 = as_ptr(dists)
        check(lib().lb2_index_search(self._h, qp, C.c_uint64(nq), C.c_uint32(k), C.c_uint32(nprobes),
                                     ip, dp, None))
        return ids, dists

    def search_refine(self, vectors, queries, k=10, nprobes=1, refine_factor=1, out=None):
        """to_table(nearest={..., refine_factor}): PQ candidates re-ranked with exact distances from
        the raw column (scanner.rs:2884-2905).  `vectors` = the indexed column (row id = row number)."""
        dt = getattr(self, "_dt", F32)
        npdt = {F32: np.float32, F16: np.float16, U8: np.uint8, BF16: np.uint16}[dt]
        if not isinstance(queries, (DeviceArray, PinnedArray)):
            queries = np.ascontiguousarray(queries, dtype=npdt)
        if not isinstance(vectors, (DeviceArray, PinnedArray)):
            vectors = np.ascontiguousarray(vectors, dtype=npdt)
        nq = queries.shape[0]
        if out is None:
            ids, dists = np.empty((nq, k), np.uint64), np.empty((nq, k), np.float32)
        else:
            ids, dists = out
        qp, _k1 = as_ptr(queries)
        vp, _k0 = as_ptr(vectors)
        ip, _k2 = as_ptr(ids)
        dp, _k3 = as_ptr(dists)
        check(lib().lb2_index_search_refine(self._h, vp, C.c_uint64(vectors.shape[0]), qp, C.c_uint64(nq),
                                            C.c_uint32(k), C.c_uint32(nprobes), C.c_uint32(refine_factor),
                                            ip, dp, None))
        return ids, dists

    def row_mask(self, allow_row_ids=None, block_row_ids=None):
        """RowIdMask (lance-core/src/utils/mask.rs:84-93) -> bitmap over storage positions
        (uint64 words), built on the device by lb2_index_row_mask."""
        from ._lib import lib as _l
        n = self.info()["num_rows"]
        bm = np.zeros((n + 63) // 64, np.uint64)
        a = None if allow_row_ids is None else np.ascontiguousarray(np.sort(np.asarray(allow_row_ids, dtype=np.uint64)))
        b = None if block_row_ids is None else np.ascontiguousarray(np.sort(np.asarray(block_row_ids, dtype=np.uint64)))
        check(_l().lb2_index_row_mask(self._h,
                                      C.c_void_p(a.ctypes.data) if a is not None and a.size else None,
                                      C.c_uint64(0 if a is None else a.size), C.c_int(a is not None),
                                      C.c_void_p(b.ctypes.data) if b is not None and b.size else None,
                                      C.c_uint64(0 if b is None else b.size), C.c_int(b is not None),
                                      C.c_void_p(bm.ctypes.data)))
        return bm

    def search_ex(self, queries, k=10, nprobes=1, allow_bitmap=None, refine_factor=0, vectors=None, out=None,
                  lower_bound=None, upper_bound=None):
        """lb2_index_search_ex: prefilter (bitmap from row_mask), range bounds and/or refine in one call."""
        from ._lib import SearchParams
        dt = getattr(self, "_dt", F32)
        npdt = {F32: np.float32, F16: np.float16, U8: np.uint8, BF16: np.uint16}[dt]
        if not isinstance(queries, (DeviceArray, PinnedArray)):
            queries = np.ascontiguousarray(queries, dtype=npdt)
        if vectors is not None and not isinstance(vectors, (DeviceArray, PinnedArray)):
            vectors = np.ascontiguousarray(vectors, dtype=npdt)
        nq = queries.shape[0]
        if out is None:
            ids, dists = np.empty((nq, k), np.uint64), np.empty((nq, k), np.float32)
        else:
            ids, dists = out
        qp, _k1 = as_ptr(queries)
        vp, _k0 = as_ptr(vectors)
        bp, _k4 = as_ptr(None if allow_bitmap is None else (allow_bitmap if isinstance(allow_bitmap, (DeviceArray, PinnedArray)) else np.ascontiguousarray(allow_bitmap, dtype=np.uint64)))
        ip, _k2 = as_ptr(ids)
        dp, _k3 = as_ptr(dists)
        sp = SearchParams(k, nprobes, refine_factor, vp.value if vp is not None else None,
                          0 if vectors is None else vectors.shape[0], bp.value if bp is not None else None,
                          int(lower_bound is not None), int(upper_bound is not None),
                          float(lower_bound or 0.0), float(upper_bound or 0.0))
        check(lib().lb2_index_search_ex(self._h, qp, C.c_uint64(nq), C.byref(sp), ip, dp, None))
        return ids, dists

    def search_probed(self, queries, k, minimum_nprobes=1, maximum_nprobes=None, late_width=1, allow_bitmap=None,
                      mask_ids=None, mask_max_len=None, refine_factor=0, vectors=None, lower_bound=None,
                      upper_bound=None):
        """lb2_index_search_probed: a query with minimum / maximum nprobes as ANNIvfSubIndexExec runs it (early
        pruning, late search, the no-rows shortcut; knn.rs:714-1130).  maximum_nprobes=None probes up to every
        partition; late_width = the late search's concurrency (get_num_compute_intensive_cpus()).  allow_bitmap as in
        search_ex; mask_max_len = RowIdMask::max_len(), mask_ids = RowIdMask::iter_ids() (None: not iterable).
        Returns (ids, dists, counts, nprobes): nprobes[q] = partitions the query searched."""
        from ._lib import ProbeParams, SearchParams
        dt = getattr(self, "_dt", F32)
        npdt = {F32: np.float32, F16: np.float16, U8: np.uint8, BF16: np.uint16}[dt]
        if not isinstance(queries, (DeviceArray, PinnedArray)):
            queries = np.ascontiguousarray(queries, dtype=npdt)
        if vectors is not None and not isinstance(vectors, (DeviceArray, PinnedArray)):
            vectors = np.ascontiguousarray(vectors, dtype=npdt)
        nq = queries.shape[0]
        ids, dists = np.empty((nq, k), np.uint64), np.empty((nq, k), np.float32)
        counts, nprobes = np.empty(nq, np.uint32), np.empty(nq, np.uint32)
        if mask_ids is not None and not isinstance(mask_ids, (DeviceArray, PinnedArray)):
            mask_ids = np.ascontiguousarray(np.sort(np.asarray(mask_ids, dtype=np.uint64)))
        qp, _k1 = as_ptr(queries)
        vp, _k0 = as_ptr(vectors)
        bp, _k4 = as_ptr(None if allow_bitmap is None else (allow_bitmap if isinstance(allow_bitmap, (DeviceArray, PinnedArray)) else np.ascontiguousarray(allow_bitmap, dtype=np.uint64)))
        mp, _k5 = as_ptr(mask_ids)
        if mask_ids is not None and mp.value is None:  # an empty numpy array has no buffer address to pass
            _k5 = np.zeros(1, np.uint64)
            mp = C.c_void_p(_k5.ctypes.data)
        sp = SearchParams(k, 0, refine_factor, vp.value if vp is not None else None,
                          0 if vectors is None else vectors.shape[0], bp.value if bp is not None else None,
                          int(lower_bound is not None), int(upper_bound is not None),
                          float(lower_bound or 0.0), float(upper_bound or 0.0))
        pp = ProbeParams(minimum_nprobes, maximum_nprobes or 0, late_width, int(mask_max_len is not None),
                         int(mask_max_len or 0), mp.value if mp is not None else None,
                         0 if mask_ids is None else int(mask_ids.shape[0]))
        check(lib().lb2_index_search_probed(self._h, qp, C.c_uint64(nq), C.byref(sp), C.byref(pp), as_ptr(ids)[0],
                                            as_ptr(dists)[0], as_ptr(counts)[0], as_ptr(nprobes)[0]))
        return ids, dists, counts, nprobes

    def search_batch(self, queries, k, nprobes=None, minimum_nprobes=None, maximum_nprobes=None, refine_factor=0,
                     vectors=None, filters=None, filter_of=None, lower_bound=None, upper_bound=None, ef=None,
                     late_width=1, out=None):
        """lb2_index_search_batch: every query with its own parameters, in one device pass.  Row q equals search_ex
        (or, with ef, the HNSW kinds' search_ex with ef) of query q alone with its own parameters and filter.
        Every per-query argument is a scalar or an [nq] array: k, nprobes, refine_factor, filter_of (index into
        `filters`, -1 = none), lower_bound / upper_bound (NaN or None = no bound), ef (0 or None = k' + k' / 2).
        `filters` is a list of allow bitmaps (as row_mask builds them) or (bitmap, max_len, mask_ids) tuples.
        A query with nprobes 0 (or every query when nprobes is None) runs the probe rule with its own minimum_nprobes
        (default 1) and maximum_nprobes (None or 0 = every partition), equal to search_probed; a filter tuple's
        max_len and mask_ids and late_width serve those queries.
        Returns (ids, dists, counts, nprobes): ids / dists [nq][max k] (or `out`'s arrays and their row length)."""
        if vectors is not None and not isinstance(vectors, (DeviceArray, PinnedArray)):
            vectors = np.ascontiguousarray(vectors, dtype=self._npdt())
        queries, nq, ks, rfs, cp, cf, nf, _keep = self._batch_params(
            "search_batch", queries, k, nprobes, minimum_nprobes, maximum_nprobes, refine_factor, filters, filter_of,
            lower_bound, upper_bound, ef)
        if (rfs > 0).any() and vectors is None:
            raise ValueError("search_batch: refine_factor > 0 needs vectors")
        kmax = int(ks.max()) if nq else 1
        if out is None:
            ids, dists = np.empty((nq, kmax), np.uint64), np.empty((nq, kmax), np.float32)
        else:
            ids, dists = out
        k_stride = int(ids.shape[1]) if len(ids.shape) == 2 else kmax
        if tuple(ids.shape) != (nq, k_stride) or tuple(dists.shape) != (nq, k_stride) or k_stride < kmax:
            raise ValueError(f"search_batch: out arrays must be [{nq}][>= {kmax}], got {ids.shape} and {dists.shape}")
        counts, probes = np.empty(nq, np.uint32), np.empty(nq, np.uint32)
        qp, _k1 = as_ptr(queries)
        vp, _k0 = as_ptr(vectors)
        check(lib().lb2_index_search_batch(self._h, qp, C.c_uint64(nq), C.c_void_p(cp.ctypes.data), cf, C.c_uint32(nf), vp,
                                           C.c_uint64(0 if vectors is None else vectors.shape[0]),
                                           C.c_uint32(late_width), C.c_uint32(k_stride), as_ptr(ids)[0],
                                           as_ptr(dists)[0], as_ptr(counts)[0], as_ptr(probes)[0]))
        return ids, dists, counts, probes

    def _npdt(self):
        return {F32: np.float32, F16: np.float16, U8: np.uint8, BF16: np.uint16}[getattr(self, "_dt", F32)]

    def _batch_params(self, name, queries, k, nprobes=None, minimum_nprobes=None, maximum_nprobes=None,
                      refine_factor=0, filters=None, filter_of=None, lower_bound=None, upper_bound=None, ef=None):
        """the checked per-query arguments of a batch call: (queries, nq, ks, rfs, the lb2_query_params array, the
        lb2_query_filter array, the number of filters, keepalive)"""
        from ._lib import QueryFilter, QueryParams
        if not isinstance(queries, (DeviceArray, PinnedArray)):
            queries = np.ascontiguousarray(queries, dtype=self._npdt())
        nq = int(queries.shape[0])

        def per_query(what, v, dtype, default):
            a = np.asarray(default if v is None else v, dtype=dtype)
            if a.ndim == 0:
                return np.full(nq, a, dtype)
            if a.shape != (nq,):
                raise ValueError(f"{name}: {what} must be a scalar or an array of {nq} values, got shape {a.shape}")
            return a

        ks = per_query("k", k, np.int64, 0)
        if nq and (ks < 1).any():
            raise ValueError(f"{name}: every k must be at least 1")
        nps = per_query("nprobes", nprobes, np.int64, 0)
        mins = per_query("minimum_nprobes", minimum_nprobes, np.int64, 1)
        maxs = per_query("maximum_nprobes", maximum_nprobes, np.int64, 0)
        if (nps < 0).any():
            raise ValueError(f"{name}: nprobes must not be negative (0: minimum / maximum nprobes)")
        ruled = nps == 0
        if (mins[ruled] < 1).any() or (maxs[ruled] < 0).any():
            raise ValueError(f"{name}: minimum_nprobes must be at least 1 and maximum_nprobes not negative")
        mins, maxs = np.where(ruled, mins, 0), np.where(ruled, maxs, 0)
        rfs = per_query("refine_factor", refine_factor, np.int64, 0)
        if (rfs < 0).any():
            raise ValueError(f"{name}: refine_factor must not be negative")
        filters = list(filters or [])
        fof = per_query("filter_of", filter_of, np.int64, -1)
        if ((fof < -1) | (fof >= len(filters))).any():
            raise ValueError(f"{name}: filter_of must be -1 or below the {len(filters)} filters")
        lows = per_query("lower_bound", lower_bound, np.float32, np.nan)
        ups = per_query("upper_bound", upper_bound, np.float32, np.nan)
        efs = per_query("ef", ef, np.int64, 0)
        if (efs < 0).any():
            raise ValueError(f"{name}: ef must not be negative")
        keep = []
        cf = (QueryFilter * max(1, len(filters)))()
        for i, f in enumerate(filters):
            bm, max_len, mask_ids = (f if isinstance(f, tuple) else (f, None, None))
            if bm is not None and not isinstance(bm, (DeviceArray, PinnedArray)):
                bm = np.ascontiguousarray(bm, dtype=np.uint64)
            if mask_ids is not None and not isinstance(mask_ids, (DeviceArray, PinnedArray)):
                mask_ids = np.ascontiguousarray(np.sort(np.asarray(mask_ids, dtype=np.uint64)))
            bp, kb = as_ptr(bm)
            mp, km = as_ptr(mask_ids)
            if mask_ids is not None and mp.value is None:  # an empty numpy array has no buffer address to pass
                km = np.zeros(1, np.uint64)
                mp = C.c_void_p(km.ctypes.data)
            keep += [bm, mask_ids, kb, km]
            cf[i] = QueryFilter(bp.value if bp is not None else None, int(max_len is not None), int(max_len or 0),
                                mp.value if mp is not None else None, 0 if mask_ids is None else int(mask_ids.shape[0]))
        # the lb2_query_params array, filled column by column (same layout as QueryParams)
        cp = np.zeros(max(1, nq), np.dtype({"names": [f for f, _ in QueryParams._fields_],
                                            "formats": [np.float32 if t is C.c_float else np.uint32
                                                        for _, t in QueryParams._fields_]}))
        for field, col in (("k", ks), ("nprobes", nps), ("minimum_nprobes", mins), ("maximum_nprobes", maxs),
                           ("refine_factor", rfs), ("ef", efs)):
            cp[field][:nq] = col
        cp["filter"][:nq] = np.where(fof < 0, 0xFFFFFFFF, fof)
        cp["has_lower_bound"][:nq], cp["has_upper_bound"][:nq] = ~np.isnan(lows), ~np.isnan(ups)
        cp["lower_bound"][:nq], cp["upper_bound"][:nq] = np.nan_to_num(lows, nan=0.0), np.nan_to_num(ups, nan=0.0)
        assert cp.dtype.itemsize == C.sizeof(QueryParams)
        return queries, nq, ks, rfs, cp, cf, len(filters), keep

    def search_candidates(self, queries, k, nprobes=None, minimum_nprobes=None, maximum_nprobes=None,
                          refine_factor=0, filters=None, filter_of=None, lower_bound=None, upper_bound=None, ef=None,
                          late_width=1, distinct=False, kc_stride=None):
        """lb2_index_search_candidates: the index half of a refined batch.  Takes search_batch's per-query arguments
        (no vectors).  Row q of ids / dists [nq][kc_stride] (default: the largest k * max(1, refine_factor)) is the
        list search_batch re-ranks for query q, counts[q] entries long; unused slots hold UINT64_MAX / +inf.
        Returns (ids, dists, counts, nprobes), and with distinct=True also (distinct_ids, positions): the batch's
        ascending distinct row ids and, per slot, the index of its id in them (UINT64_MAX for an unused slot).
        Take the rows of distinct_ids and pass them to refine_taken."""
        queries, nq, ks, rfs, cp, cf, nf, _keep = self._batch_params(
            "search_candidates", queries, k, nprobes, minimum_nprobes, maximum_nprobes, refine_factor, filters,
            filter_of, lower_bound, upper_bound, ef)
        kcmax = int((ks * np.maximum(rfs, 1)).max()) if nq else 1
        kc_stride = kcmax if kc_stride is None else int(kc_stride)
        ids, dists = np.empty((nq, kc_stride), np.uint64), np.empty((nq, kc_stride), np.float32)
        counts, probes = np.empty(nq, np.uint32), np.empty(nq, np.uint32)
        uniq = np.empty(max(1, nq * kc_stride), np.uint64) if distinct else None
        pos = np.empty((nq, kc_stride), np.uint64) if distinct else None
        m = np.zeros(1, np.uint64)
        check(lib().lb2_index_search_candidates(self._h, as_ptr(queries)[0], C.c_uint64(nq), C.c_void_p(cp.ctypes.data),
                                                cf, C.c_uint32(nf), C.c_uint32(late_width), C.c_uint32(kc_stride),
                                                as_ptr(ids)[0], as_ptr(dists)[0], as_ptr(counts)[0], as_ptr(probes)[0],
                                                as_ptr(uniq)[0], as_ptr(m if distinct else None)[0], as_ptr(pos)[0]))
        if not distinct:
            return ids, dists, counts, probes
        return ids, dists, counts, probes, uniq[:int(m[0])].copy(), pos

    def refine_taken(self, queries, candidates, taken, positions, k, refine_factor=0, lower_bound=None,
                     upper_bound=None, out=None):
        """lb2_index_refine_taken: the exact re-rank of the rows the caller took.  `candidates` = (ids, dists,
        counts) of search_candidates; `taken` [m][d] (numpy, PinnedArray or DeviceArray, the index's element type)
        holds the rows of its distinct_ids, and `positions` is its positions array.  k, refine_factor and the
        bounds are search_candidates' per-query values.  Equal to search_batch with the column as `vectors`.
        Returns (ids, dists, counts): ids / dists [nq][max k] (or `out`'s arrays and their row length)."""
        cid, cd, cc = candidates
        queries, nq, ks, _rfs, cp, _cf, _nf, _keep = self._batch_params(
            "refine_taken", queries, k, 1, None, None, refine_factor, None, None, lower_bound, upper_bound, None)
        cid = cid if isinstance(cid, DeviceArray) else np.ascontiguousarray(cid, np.uint64)
        cd = cd if isinstance(cd, DeviceArray) else np.ascontiguousarray(cd, np.float32)
        cc = cc if isinstance(cc, DeviceArray) else np.ascontiguousarray(cc, np.uint32)
        if tuple(cid.shape[:1]) != (nq,) or len(cid.shape) != 2 or tuple(cd.shape) != tuple(cid.shape):
            raise ValueError(f"refine_taken: candidate arrays must be [{nq}][kc_stride], got {cid.shape} and {cd.shape}")
        kc_stride = int(cid.shape[1])
        if positions is not None and not isinstance(positions, DeviceArray):
            positions = np.ascontiguousarray(positions, np.uint64)
        if positions is not None and tuple(positions.shape) != tuple(cid.shape):
            raise ValueError(f"refine_taken: positions must be [{nq}][{kc_stride}], got {positions.shape}")
        if not isinstance(taken, (DeviceArray, PinnedArray)):
            taken = np.ascontiguousarray(taken, dtype=self._npdt())
        kmax = int(ks.max()) if nq else 1
        if out is None:
            ids, dists = np.empty((nq, kmax), np.uint64), np.empty((nq, kmax), np.float32)
        else:
            ids, dists = out
        k_stride = int(ids.shape[1]) if len(ids.shape) == 2 else kmax
        if tuple(ids.shape) != (nq, k_stride) or tuple(dists.shape) != (nq, k_stride) or k_stride < kmax:
            raise ValueError(f"refine_taken: out arrays must be [{nq}][>= {kmax}], got {ids.shape} and {dists.shape}")
        counts = np.empty(nq, np.uint32)
        check(lib().lb2_index_refine_taken(self._h, as_ptr(queries)[0], C.c_uint64(nq), C.c_void_p(cp.ctypes.data),
                                           C.c_uint32(kc_stride), as_ptr(cid)[0], as_ptr(cd)[0], as_ptr(cc)[0],
                                           as_ptr(taken)[0], C.c_uint64(int(taken.shape[0])), as_ptr(positions)[0],
                                           C.c_uint32(k_stride), as_ptr(ids)[0], as_ptr(dists)[0], as_ptr(counts)[0]))
        return ids, dists, counts

    def search_combined(self, queries, k, vectors, unindexed_vectors, unindexed_row_ids, nprobes=None,
                        minimum_nprobes=None, maximum_nprobes=None, late_width=1, refine_factor=0, allow_bitmap=None,
                        unindexed_allow_bitmap=None, mask_ids=None, mask_max_len=None, lower_bound=None,
                        upper_bound=None):
        """lb2_index_search_combined: a nearest() query on an index that does not cover every row (knn_combined,
        scanner.rs:2946-3027).  The index search (fixed `nprobes`, or minimum / maximum nprobes as in search_probed)
        runs with refine factor max(1, refine_factor) against `vectors` (the indexed column, row id = row number);
        the unindexed rows (`unindexed_vectors` with their `unindexed_row_ids`, filtered by `unindexed_allow_bitmap`)
        are searched flat with the index metric; the two lists are merged by (distance, row id).
        Returns (ids, dists, counts, nprobes); nprobes is None with a fixed nprobes."""
        from ._lib import ProbeParams, SearchParams, UnindexedRows
        dt = getattr(self, "_dt", F32)
        npdt = {F32: np.float32, F16: np.float16, U8: np.uint8, BF16: np.uint16}[dt]
        probed = nprobes is None
        if not isinstance(queries, (DeviceArray, PinnedArray)):
            queries = np.ascontiguousarray(queries, dtype=npdt)
        if not isinstance(vectors, (DeviceArray, PinnedArray)):
            vectors = np.ascontiguousarray(vectors, dtype=npdt)
        if not isinstance(unindexed_vectors, (DeviceArray, PinnedArray)):
            unindexed_vectors = np.ascontiguousarray(unindexed_vectors, dtype=npdt)
        nq = queries.shape[0]
        ids, dists, counts = np.empty((nq, k), np.uint64), np.empty((nq, k), np.float32), np.empty(nq, np.uint32)
        nprobes_out = np.empty(nq, np.uint32) if probed else None
        if mask_ids is not None and not isinstance(mask_ids, (DeviceArray, PinnedArray)):
            mask_ids = np.ascontiguousarray(np.sort(np.asarray(mask_ids, dtype=np.uint64)))
        qp, _k1 = as_ptr(queries)
        vp, _k0 = as_ptr(vectors)
        bp, _k2 = as_ptr(_bitmap(allow_bitmap))
        uvp, _k3 = as_ptr(unindexed_vectors)
        urp, _k4 = as_ptr(_row_ids(unindexed_row_ids))
        ubp, _k5 = as_ptr(_bitmap(unindexed_allow_bitmap))
        mp, _k6 = as_ptr(mask_ids)
        if mask_ids is not None and mp.value is None:  # an empty numpy array has no buffer address to pass
            _k6 = np.zeros(1, np.uint64)
            mp = C.c_void_p(_k6.ctypes.data)
        if urp is not None and urp.value is None:      # no unindexed rows: any valid address stands for the empty list
            _k4 = np.zeros(1, np.uint64)
            urp = C.c_void_p(_k4.ctypes.data)
        sp = SearchParams(k, 0 if probed else nprobes, refine_factor, vp.value, vectors.shape[0],
                          bp.value if bp is not None else None, int(lower_bound is not None),
                          int(upper_bound is not None), float(lower_bound or 0.0), float(upper_bound or 0.0))
        pp = None
        if probed:
            pp = ProbeParams(minimum_nprobes or 1, maximum_nprobes or 0, late_width, int(mask_max_len is not None),
                             int(mask_max_len or 0), mp.value if mp is not None else None,
                             0 if mask_ids is None else int(mask_ids.shape[0]))
        u = UnindexedRows(uvp.value, unindexed_vectors.shape[0], urp.value if urp is not None else None,
                          ubp.value if ubp is not None else None)
        check(lib().lb2_index_search_combined(self._h, qp, C.c_uint64(nq), C.byref(sp),
                                              C.byref(pp) if pp is not None else None, C.byref(u), as_ptr(ids)[0],
                                              as_ptr(dists)[0], as_ptr(counts)[0], as_ptr(nprobes_out)[0]))
        return ids, dists, counts, nprobes_out

    def search_combined_batch(self, queries, k, vectors, unindexed_vectors, unindexed_row_ids, nprobes=None,
                              minimum_nprobes=None, maximum_nprobes=None, refine_factor=0, filters=None,
                              filter_of=None, unindexed_allow_bitmap=None, unindexed_filters=None, lower_bound=None,
                              upper_bound=None, ef=None, late_width=1, out=None):
        """lb2_index_search_combined_batch: knn_combined (search_combined) for a batch whose queries differ in their
        parameters, in one call.  Takes search_batch's per-query arguments; `vectors` is the indexed column (row id =
        row number) and the index half runs with refine factor max(1, refine_factor).  The unindexed rows
        (`unindexed_vectors` with their `unindexed_row_ids`) are searched flat: a query without a filter admits the
        rows of `unindexed_allow_bitmap` (None: all), a query with filter f those of unindexed_filters[f] (one bitmap
        per filter, validity AND the filter over the unindexed rows; None admits every row).  Row q equals
        search_combined of query q alone.  Returns (ids, dists, counts, nprobes): ids / dists [nq][max k] (or
        `out`'s arrays and their row length)."""
        from ._lib import UnindexedBatch, UnindexedRows
        name = "search_combined_batch"
        if vectors is None:
            raise ValueError(f"{name}: the index's rows are re-scored exactly: vectors is required")
        if not isinstance(vectors, (DeviceArray, PinnedArray)):
            vectors = np.ascontiguousarray(vectors, dtype=self._npdt())
        if not isinstance(unindexed_vectors, (DeviceArray, PinnedArray)):
            unindexed_vectors = np.ascontiguousarray(unindexed_vectors, dtype=self._npdt())
        queries, nq, ks, _rfs, cp, cf, nf, keep = self._batch_params(
            name, queries, k, nprobes, minimum_nprobes, maximum_nprobes, refine_factor, filters, filter_of,
            lower_bound, upper_bound, ef)
        ufilters = list(unindexed_filters) if unindexed_filters is not None else ([] if nf == 0 else None)
        if ufilters is None or len(ufilters) != nf:
            raise ValueError(f"{name}: unindexed_filters must hold one bitmap (or None) for each of the {nf} filters")
        if unindexed_row_ids is None:
            raise ValueError(f"{name}: unindexed_row_ids is required")
        ids, dists, k_stride = _out_rows(name, out, nq, int(ks.max()) if nq else 1)
        counts, probes = np.empty(nq, np.uint32), np.empty(nq, np.uint32)
        table = _bitmap_table(ufilters, keep)
        urp, _k4 = as_ptr(_row_ids(unindexed_row_ids))
        if urp.value is None:  # no unindexed rows: any valid address stands for the empty list
            _k4 = np.zeros(1, np.uint64)
            urp = C.c_void_p(_k4.ctypes.data)
        uvp, _k3 = as_ptr(unindexed_vectors)
        ubp, _k5 = as_ptr(_bitmap(unindexed_allow_bitmap))
        u = UnindexedBatch(UnindexedRows(uvp.value, unindexed_vectors.shape[0], urp.value,
                                         ubp.value if ubp is not None else None), C.cast(table, C.c_void_p))
        qp, _k1 = as_ptr(queries)
        vp, _k0 = as_ptr(vectors)
        check(lib().lb2_index_search_combined_batch(self._h, qp, C.c_uint64(nq), C.c_void_p(cp.ctypes.data), cf,
                                                    C.c_uint32(nf), vp, C.c_uint64(vectors.shape[0]),
                                                    C.c_uint32(late_width), C.byref(u), C.c_uint32(k_stride),
                                                    as_ptr(ids)[0], as_ptr(dists)[0], as_ptr(counts)[0],
                                                    as_ptr(probes)[0]))
        return ids, dists, counts, probes

    def search_async(self, queries, out, k=10, nprobes=1, cuda_stream=None, done_event=None, allow_bitmap=None,
                     lower_bound=None, upper_bound=None):
        """lb2_index_search_async: enqueue a search on `cuda_stream` (cudaStream_t handle as int) and return at once.
        queries / out = (ids, dists) are DeviceArray or PinnedArray and must stay alive until the stream is done."""
        from ._lib import SearchParams
        assert all(isinstance(a, (DeviceArray, PinnedArray)) for a in (queries, out[0], out[1]))
        qp, _k1 = as_ptr(queries)
        ip, _k2 = as_ptr(out[0])
        dp, _k3 = as_ptr(out[1])
        bp, _k4 = as_ptr(allow_bitmap)
        sp = SearchParams(k, nprobes, 0, None, 0, bp.value if bp is not None else None,
                          int(lower_bound is not None), int(upper_bound is not None),
                          float(lower_bound or 0.0), float(upper_bound or 0.0))
        check(lib().lb2_index_search_async(self._h, qp, C.c_uint64(queries.shape[0]), C.byref(sp), ip, dp, None,
                                           C.c_void_p(cuda_stream), C.c_void_p(done_event)))

    def update(self, new_centroids=None, part_map=None, add_part_ids=None, add_codes=None, add_row_ids=None,
               remove_row_ids=None):
        """lb2_index_update: merge AssignOp-style changes (append / remove / re-map partitions) into a NEW index."""
        info = self.info()
        dt = getattr(self, "_dt", F32)
        cent = None if new_centroids is None else _typed(new_centroids, dt == BF16)[0]
        new_k = info["num_partitions"] if cent is None else cent.shape[0]
        pm = None if part_map is None else np.ascontiguousarray(part_map, dtype=np.uint32)
        ap = None if add_part_ids is None else np.ascontiguousarray(add_part_ids, dtype=np.uint32)
        ac = None if add_codes is None else np.ascontiguousarray(add_codes, dtype=np.uint8)
        ar = None if add_row_ids is None else np.ascontiguousarray(add_row_ids, dtype=np.uint64)
        rm = None if remove_row_ids is None else np.sort(np.ascontiguousarray(remove_row_ids, dtype=np.uint64))
        ptrs = [as_ptr(x)[0] for x in (cent, pm, ap, ac, ar, rm)]
        h = C.c_void_p()
        check(lib().lb2_index_update(self._h, ptrs[0], C.c_uint32(new_k), ptrs[1], ptrs[2], ptrs[3], ptrs[4],
                                     C.c_uint64(0 if ap is None else ap.size), ptrs[5],
                                     C.c_uint64(0 if rm is None else rm.size), C.byref(h)))
        out = type(self)(h)
        if hasattr(self, "_dt"):
            out._dt = self._dt
        return out

    def _payload_empty(self, n):
        """an array for n rows of this kind's stored payload, as export() returns it"""
        i = self.info()
        return np.empty((n, i["num_sub_vectors"] // 2 if i["num_bits"] == 4 else i["num_sub_vectors"]), np.uint8)

    def transform(self, vectors):
        """lb2_index_transform: IvfTransformer::transform with this index's model -> dict of part_ids, payload (what
        the kind stores for each row, as export() holds it), add_factors / scale_factors (IVF_RQ, else None) and valid
        (False: the kind's build drops the row)."""
        npdt = {F32: np.float32, F16: np.float16, U8: np.uint8, BF16: np.uint16}[getattr(self, "_dt", F32)]
        if not isinstance(vectors, (DeviceArray, PinnedArray)):
            vectors = np.ascontiguousarray(vectors, dtype=npdt)
        n = vectors.shape[0]
        rq = isinstance(self, IvfRqIndex)
        part, valid, payload = np.empty(n, np.uint32), np.empty(n, np.uint8), self._payload_empty(n)
        add, scale = (np.empty(n, np.float32), np.empty(n, np.float32)) if rq else (None, None)
        vp, _k = as_ptr(vectors)
        ptr = [as_ptr(a)[0] if a is not None and a.size else None for a in (part, payload, add, scale, valid)]
        check(lib().lb2_index_transform(self._h, vp, C.c_uint64(n), *ptr))
        return dict(part_ids=part, payload=payload, add_factors=add, scale_factors=scale, valid=valid.astype(bool))

    # the name of the kind's payload column in the reference's storage
    _STORAGE_COLUMN = "__pq_code"

    def export_storage(self):
        """lb2_index_export_storage: the whole index in the reference's storage layout, every partition's batch back
        to back (include/lance_b200.h, lb2_index_storage).  A dict of numpy arrays keyed by the reference's column
        names -- "_rowid", the payload column ("__pq_code" transposed per partition, "__sq_code", "flat" or the packed
        "__rabit_code", each [num_rows][bytes or elements per row] as the FixedSizeList values), IVF_RQ's
        "__add_factors" / "__scale_factors" -- plus "part_lengths".  A graph kind adds its HNSW metadata
        ("max_level", "m", "ef_construction", "entry_point" [K], "level_offsets" [K][max_level + 1]) and the level
        batches: "__vector_id", "list_offsets" (the Arrow list offsets over all partitions), "__neighbors",
        "_distance"."""
        st = _CIndexStorage()
        check(lib().lb2_index_export_storage(self._h, C.byref(st)))
        K, n, L, rows, e = st.num_partitions, st.num_rows, st.max_level, st.num_graph_rows, st.num_edges
        out = {"part_lengths": np.empty(K, np.uint64), "_rowid": np.empty(n, np.uint64),
               self._STORAGE_COLUMN: self._payload_empty(n)}
        if isinstance(self, IvfRqIndex):
            out["__add_factors"], out["__scale_factors"] = np.empty(n, np.float32), np.empty(n, np.float32)
        if L:
            out.update({"max_level": L, "m": st.m, "ef_construction": st.ef_construction,
                        "entry_point": np.empty(K, np.uint32), "level_offsets": np.empty((K, L + 1), np.uint64),
                        "__vector_id": np.empty(rows, np.uint32), "list_offsets": np.empty(rows + 1, np.uint64),
                        "__neighbors": np.empty(e, np.uint32), "_distance": np.empty(e, np.float32)})
        ptr = lambda k: C.c_void_p(out[k].ctypes.data) if k in out and out[k].size else None  # noqa: E731
        st.part_lengths, st.row_ids, st.payload = ptr("part_lengths"), ptr("_rowid"), ptr(self._STORAGE_COLUMN)
        st.add_factors, st.scale_factors = ptr("__add_factors"), ptr("__scale_factors")
        st.entry_point, st.level_offsets, st.vector_id = ptr("entry_point"), ptr("level_offsets"), ptr("__vector_id")
        st.list_offsets, st.neighbors, st.distances = ptr("list_offsets"), ptr("__neighbors"), ptr("_distance")
        check(lib().lb2_index_export_storage(self._h, C.byref(st)))
        return out

    @classmethod
    def _check_storage_class(cls, storage):
        """the graph columns are present exactly for the graph classes (IvfHnsw*Index)"""
        graph, hnsw = "level_offsets" in storage, issubclass(cls, _HnswGraphs)
        if graph != hnsw:
            raise ValueError(f"{cls.__name__}.from_storage: " + (
                "the storage has no HNSW graph columns (level_offsets, __vector_id, ...)" if hnsw else
                "the storage has HNSW graph columns: open it with the IvfHnsw*Index class of this kind"))

    def _load_storage(self, storage):
        """lb2_index_load_storage of a dict as export_storage returns it (a graph when it has "level_offsets")"""
        s = storage
        a = {"part_lengths": np.ascontiguousarray(s["part_lengths"], dtype=np.uint64),
             "_rowid": np.ascontiguousarray(s["_rowid"], dtype=np.uint64),
             "payload": np.ascontiguousarray(s[self._STORAGE_COLUMN])}
        for k in ("__add_factors", "__scale_factors", "_distance"):
            if k in s:
                a[k] = np.ascontiguousarray(s[k], dtype=np.float32)
        for k in ("entry_point", "__vector_id", "__neighbors"):
            if k in s:
                a[k] = np.ascontiguousarray(s[k], dtype=np.uint32)
        for k in ("level_offsets", "list_offsets"):
            if k in s:
                a[k] = np.ascontiguousarray(s[k], dtype=np.uint64)
        ptr = lambda k: C.c_void_p(a[k].ctypes.data) if k in a and a[k].size else None  # noqa: E731
        graph = "level_offsets" in a
        st = _CIndexStorage(a["part_lengths"].size, a["_rowid"].size, a["payload"].nbytes, ptr("part_lengths"),
                            ptr("_rowid"), ptr("payload"), ptr("__add_factors"), ptr("__scale_factors"),
                            int(s["max_level"]) if graph else 0, int(s["m"]) if graph else 0,
                            int(s.get("ef_construction", 0)) if graph else 0,
                            a["__vector_id"].size if graph else 0, a["__neighbors"].size if graph else 0,
                            ptr("entry_point"), ptr("level_offsets"), ptr("__vector_id"), ptr("list_offsets"),
                            ptr("__neighbors"), ptr("_distance"))
        check(lib().lb2_index_load_storage(self._h, C.byref(st)))

    @classmethod
    def from_storage(cls, centroids, codebook, storage, distance_type="l2", num_bits=8, dtype=np.float32, bf16=False):
        """Open an index from its model and its storage columns (a dict as export_storage returns; with the HNSW
        metadata and level batches for IvfHnswPqIndex).  dtype / bf16: the column's element type."""
        cls._check_storage_class(storage)
        dt = BF16 if bf16 else _DTYPES[np.dtype(dtype)]
        centroids, codebook = _model_arr(centroids, dt), _model_arr(codebook, dt)
        k, d = centroids.shape
        h = C.c_void_p()
        check(lib().lb2_index_create(C.c_void_p(centroids.ctypes.data), C.c_uint32(k), C.c_uint32(d), C.c_int(dt),
                                     C.c_int(_metric(distance_type)), C.c_void_p(codebook.ctypes.data),
                                     C.c_uint32(codebook.shape[0]), C.c_uint32(num_bits), C.byref(h)))
        ix = cls(h)
        ix._dt = dt
        ix._load_storage(storage)
        return ix

    def optimize(self, add_vectors=None, add_row_ids=None, add_part_ids=None, add_payload=None, add_factors=None,
                 new_centroids=None, part_map=None, remove_row_ids=None, remap=None, seed=0):
        """lb2_index_optimize: append, remove, re-map partitions and remap row ids into a NEW index of this class.
        add_vectors: raw rows run through transform() first, rows it marks invalid dropped (KeepFiniteVectors);
        otherwise add_part_ids / add_payload (/ add_factors = (add, scale) for IVF_RQ) as transform() returns them.
        remap: {old id: new id or None} or (old ids, new ids) with UINT64_MAX for None.  seed: the level draws of the
        graphs that are rebuilt (IVF_HNSW_*)."""
        return self._optimize(add_vectors, add_row_ids, add_part_ids, add_payload, add_factors, new_centroids, part_map,
                              remove_row_ids, remap, seed, 0)

    def _optimize(self, add_vectors, add_row_ids, add_part_ids, add_payload, add_factors, new_centroids, part_map,
                  remove_row_ids, remap, seed, insert_batch):
        p, _keep = self._optimize_params(add_vectors, add_row_ids, add_part_ids, add_payload, add_factors,
                                         new_centroids, part_map, remove_row_ids, remap, seed, insert_batch)
        h = C.c_void_p()
        check(lib().lb2_index_optimize(self._h, C.byref(p), C.byref(h)))
        return self._like(h)

    def _like(self, h):
        """a new index of this class over handle h, with this index's element type"""
        out = type(self)(h)
        if hasattr(self, "_dt"):
            out._dt = self._dt
        return out

    @staticmethod
    def _remap_arrays(remap):
        """{old id: new id or None} or (old ids, new ids) -> ascending (old ids, new ids), UINT64_MAX for None"""
        if remap is None:
            return None, None
        if isinstance(remap, dict):
            ro = np.fromiter(remap.keys(), np.uint64, len(remap))
            rn = np.fromiter((0xFFFFFFFFFFFFFFFF if v is None else v for v in remap.values()), np.uint64, len(remap))
            o = np.argsort(ro, kind="stable")
            return ro[o], rn[o]
        return tuple(np.ascontiguousarray(a, dtype=np.uint64) for a in remap)

    def _optimize_params(self, add_vectors, add_row_ids, add_part_ids, add_payload, add_factors, new_centroids,
                         part_map, remove_row_ids, remap, seed, insert_batch):
        """lb2_optimize_params of optimize()'s arguments, and the arrays it points into (keep them alive)"""
        from ._lib import OptimizeParams
        if add_vectors is not None:
            if add_part_ids is not None or add_payload is not None or add_factors is not None:
                raise ValueError("optimize: pass add_vectors or add_part_ids / add_payload / add_factors, not both")
            t = self.transform(add_vectors)
            ok = t["valid"]
            add_part_ids, add_payload = t["part_ids"][ok], t["payload"][ok]
            if t["add_factors"] is not None:
                add_factors = (t["add_factors"][ok], t["scale_factors"][ok])
            if add_row_ids is not None:
                add_row_ids = np.asarray(add_row_ids, dtype=np.uint64)[ok]
        info = self.info()
        dt = getattr(self, "_dt", F32)
        cent = None if new_centroids is None else _model_arr(new_centroids, dt)
        new_k = info["num_partitions"] if cent is None else cent.shape[0]
        pm = None if part_map is None else np.ascontiguousarray(part_map, dtype=np.uint32)
        ap = None if add_part_ids is None else np.ascontiguousarray(add_part_ids, dtype=np.uint32)
        ac = None if add_payload is None else np.ascontiguousarray(add_payload)
        ar = None if add_row_ids is None else np.ascontiguousarray(add_row_ids, dtype=np.uint64)
        fa = fs = None
        if add_factors is not None:
            fa, fs = (np.ascontiguousarray(f, dtype=np.float32) for f in add_factors)
        rm = None if remove_row_ids is None else np.sort(np.ascontiguousarray(remove_row_ids, dtype=np.uint64))
        ro, rn = self._remap_arrays(remap)
        keep = [cent, pm, ap, ac, fa, fs, ar, rm, ro, rn]
        ptr = [as_ptr(x)[0] if x is not None and x.size else None for x in keep]
        nz = lambda p: p.value if p is not None else None  # noqa: E731
        n_add = 0 if ap is None else ap.size
        p = OptimizeParams(nz(ptr[0]), new_k, nz(ptr[1]), nz(ptr[2]), nz(ptr[3]), nz(ptr[4]), nz(ptr[5]), nz(ptr[6]),
                           n_add, nz(ptr[7]), 0 if rm is None else rm.size, nz(ptr[8]), nz(ptr[9]),
                           0 if ro is None else ro.size, seed, insert_batch)
        return p, keep

    # ---- partition split and join (rust/lance/src/index/vector/builder.rs:1152-1814) ------------------------------
    def partition_to_split(self, new_part_ids=None):
        """lb2_index_partition_to_split (should_split): the partition to split, counting the add list's partition ids
        new_part_ids with the stored rows, or None"""
        a = None if new_part_ids is None else np.ascontiguousarray(new_part_ids, dtype=np.uint32)
        part = C.c_uint32()
        check(lib().lb2_index_partition_to_split(self._h, as_ptr(a)[0] if a is not None and a.size else None,
                                                 C.c_uint64(0 if a is None else a.size), C.byref(part)))
        return None if part.value == 0xFFFFFFFF else part.value

    def partition_to_join(self, remap=None):
        """lb2_index_partition_to_join (should_join): the partition to join, counting the rows the remap does not map
        to None, or None"""
        ro, rn = self._remap_arrays(remap)
        n = 0 if ro is None else ro.size
        part = C.c_uint32()
        check(lib().lb2_index_partition_to_join(self._h, as_ptr(ro)[0] if n else None, as_ptr(rn)[0] if n else None,
                                                C.c_uint64(n), C.byref(part)))
        return None if part.value == 0xFFFFFFFF else part.value

    def reassign_candidates(self, part):
        """lb2_index_reassign_candidates (select_reassign_candidates): the partitions whose raw rows a split of `part`
        reads, in candidate order"""
        ids, cnt = np.empty(64, np.uint32), C.c_uint32()
        check(lib().lb2_index_reassign_candidates(self._h, C.c_uint32(part), C.c_void_p(ids.ctypes.data), C.byref(cnt)))
        return ids[:cnt.value].copy()

    def _raw(self, vectors):
        if isinstance(vectors, (DeviceArray, PinnedArray)):
            return vectors
        npdt = {F32: np.float32, F16: np.float16, U8: np.uint8, BF16: np.uint16}[getattr(self, "_dt", F32)]
        d = self.info()["dimension"]
        return np.ascontiguousarray(np.asarray(vectors).reshape(-1, d), dtype=npdt)

    def split(self, part, vectors, row_ids, cand_vectors=None, cand_row_ids=None, cand_part_ids=None,
              add_vectors=None, add_row_ids=None, add_part_ids=None, add_payload=None, add_factors=None,
              remove_row_ids=None, seed=0):
        """lb2_index_split: split partition `part` (vectors / row_ids: its raw rows, ascending ids) with the raw rows of
        its reassign candidates (grouped in candidate order), composed with an optimize's add list and removals.
        Returns (new index, dict(new_centroids, dest)): dest[i] the new partition of raw row i (the partition's rows,
        then the candidates'), 0xFFFFFFFF for a candidate row that stays."""
        return self._split(part, vectors, row_ids, cand_vectors, cand_row_ids, cand_part_ids, add_vectors, add_row_ids,
                           add_part_ids, add_payload, add_factors, remove_row_ids, seed, 0)

    def _split(self, part, vectors, row_ids, cand_vectors, cand_row_ids, cand_part_ids, add_vectors, add_row_ids,
               add_part_ids, add_payload, add_factors, remove_row_ids, seed, insert_batch):
        from ._lib import SplitParams
        op, keep = self._optimize_params(add_vectors, add_row_ids, add_part_ids, add_payload, add_factors, None, None,
                                         remove_row_ids, None, seed, insert_batch)
        info = self.info()
        d = info["dimension"]
        v, r = self._raw(vectors), np.ascontiguousarray(row_ids, dtype=np.uint64)
        if cand_vectors is None:
            cv, cr, cp = self._raw(np.zeros((0, d))), np.zeros(0, np.uint64), np.zeros(0, np.uint32)
        else:
            cv, cr = self._raw(cand_vectors), np.ascontiguousarray(cand_row_ids, dtype=np.uint64)
            cp = np.ascontiguousarray(cand_part_ids, dtype=np.uint32)
        new_k = info["num_partitions"] + (1 if len(r) else 0)
        cent = np.empty((new_k, d), _model_np(getattr(self, "_dt", F32)))
        dest = np.empty(len(r) + len(cr), np.uint32)
        pz = lambda a: as_ptr(a)[0] if a.shape[0] else None  # noqa: E731
        sp = SplitParams(part, pz(v), pz(r), len(r), pz(cv), pz(cr), pz(cp), len(cr), op, pz(cent), pz(dest))
        h = C.c_void_p()
        check(lib().lb2_index_split(self._h, C.byref(sp), C.byref(h)))
        del keep
        return self._like(h), dict(new_centroids=cent, dest=dest)

    def join(self, part, vectors, row_ids, remove_row_ids=None, remap=None, seed=0):
        """lb2_index_join: delete partition `part` and send its raw rows (ascending ids) to their nearest reassign
        candidate, composed with removals and a row-id remap.  Returns (new index, dest)."""
        return self._join(part, vectors, row_ids, remove_row_ids, remap, seed, 0)

    def _join(self, part, vectors, row_ids, remove_row_ids, remap, seed, insert_batch):
        from ._lib import JoinParams
        v, r = self._raw(vectors), np.ascontiguousarray(row_ids, dtype=np.uint64)
        rm = None if remove_row_ids is None else np.sort(np.ascontiguousarray(remove_row_ids, dtype=np.uint64))
        ro, rn = self._remap_arrays(remap)
        dest = np.empty(len(r), np.uint32)
        pz = lambda a: as_ptr(a)[0] if a is not None and a.shape[0] else None  # noqa: E731
        jp = JoinParams(part, pz(v), pz(r), len(r), pz(rm), 0 if rm is None else rm.size, pz(ro), pz(rn),
                        0 if ro is None else ro.size, seed, insert_batch, pz(dest))
        h = C.c_void_p()
        check(lib().lb2_index_join(self._h, C.byref(jp), C.byref(h)))
        return self._like(h), dest

    def repartition(self):
        """lb2_index_repartition: row-sharded index -> the index of the partitions this rank owns (p % nranks == rank),
        by one device all-to-all; a copy without a communicator."""
        h = C.c_void_p()
        check(lib().lb2_index_repartition(self._h, C.byref(h)))
        out = type(self)(h)
        for a in ("_dt",):
            if hasattr(self, a):
                setattr(out, a, getattr(self, a))
        return out

    def search_sharded(self, queries, k=10, nprobes=1, out=None):
        """lb2_index_search_sharded: this index holds ONE RANK'S rows (global row ids); every rank calls with
        the same queries and gets the global top-k (per-rank lists exchanged + merged in the library)."""
        from ._lib import SearchParams
        dt = getattr(self, "_dt", F32)
        npdt = {F32: np.float32, F16: np.float16, U8: np.uint8, BF16: np.uint16}[dt]
        if not isinstance(queries, (DeviceArray, PinnedArray)):
            queries = np.ascontiguousarray(queries, dtype=npdt)
        nq = queries.shape[0]
        if out is None:
            ids, dists = np.empty((nq, k), np.uint64), np.empty((nq, k), np.float32)
        else:
            ids, dists = out
        qp, _k1 = as_ptr(queries)
        ip, _k2 = as_ptr(ids)
        dp, _k3 = as_ptr(dists)
        sp = SearchParams(k, nprobes, 0, None, 0, None, 0, 0, 0.0, 0.0)
        check(lib().lb2_index_search_sharded(self._h, qp, C.c_uint64(nq), C.byref(sp), ip, dp, None))
        return ids, dists

    def set_partition_index(self, mode, seed=0, insert_batch=1):
        """lb2_index_set_partition_index: how this index assigns rows it transforms (transform, IVF_RQ's split) and
        the rule the indexes optimize / split / join return inherit.  mode as PartitionIndex's ("exact", "auto",
        "hnsw": LANCE_USE_HNSW_SPEEDUP_INDEXING's disabled / unset / enabled); the graph over this index's centroids
        draws its levels from seed and is built with insert_batch."""
        check(lib().lb2_index_set_partition_index(self._h, C.c_int(_pi_mode(mode)), C.c_uint64(seed),
                                                  C.c_uint32(insert_batch)))

    def close(self):
        if self._h:
            lib().lb2_index_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class IvfFlatIndex(IvfPqIndex):
    """Device-resident IVFIndex<FlatIndex, FlatQuantizer> (IVF_FLAT): exact distances inside the
    probed partitions (lance-index/src/vector/flat/{index,storage}.rs)."""

    @classmethod
    def build(cls, data, distance_type="l2", num_partitions=256, max_iters=50, sample_rate=256, seed=0,
              centroids=None, row_ids=None, partition_index="exact", partition_index_batch=1, bf16=False):
        """bf16=True: `data` is a uint16 array holding bfloat16 bit patterns (numpy has no bf16 dtype)."""
        bp = FlatBuildParams()
        lib().lb2_ivfflat_build_params_default(C.byref(bp))
        keep = _ivf_fields(bp, num_partitions, max_iters, sample_rate, seed, centroids,  # noqa: F841
                           partition_index, partition_index_batch)
        return _build(cls, lib().lb2_ivfflat_build, bp, data, distance_type, row_ids, bf16)

    @classmethod
    def from_parts(cls, centroids, part_ids, vectors, row_ids=None, distance_type="l2", bf16=False):
        """The vectors keep their element type (bf16=True: uint16 bit patterns); the centroids have its model type."""
        vectors, dt = _typed(vectors, bf16)
        centroids = np.ascontiguousarray(centroids, dtype=_model_np(dt))
        k, d = centroids.shape
        h = C.c_void_p()
        check(lib().lb2_index_create_flat(C.c_void_p(centroids.ctypes.data), C.c_uint32(k), C.c_uint32(d),
                                          C.c_int(dt), C.c_int(_metric(distance_type)), C.byref(h)))
        ix = cls(h)
        ix._dt = dt
        part_ids = np.ascontiguousarray(part_ids, dtype=np.uint32)
        rid = None if row_ids is None else np.ascontiguousarray(row_ids, dtype=np.uint64)
        rp, _k = as_ptr(rid)
        vp, _k2 = as_ptr(vectors)
        check(lib().lb2_index_load_flat(h, C.c_void_p(part_ids.ctypes.data), vp, rp, C.c_uint64(part_ids.size)))
        return ix

    _STORAGE_COLUMN = "flat"

    @classmethod
    def from_storage(cls, centroids, storage, distance_type="l2", dtype=np.float32, bf16=False):
        """Open an index from its centroids (the model type of the column) and its storage columns, as
        IvfPqIndex.from_storage.  dtype / bf16: the element type of the stored rows."""
        cls._check_storage_class(storage)
        dt = BF16 if bf16 else _DTYPES[np.dtype(dtype)]
        centroids = _model_arr(centroids, dt)
        k, d = centroids.shape
        h = C.c_void_p()
        check(lib().lb2_index_create_flat(C.c_void_p(centroids.ctypes.data), C.c_uint32(k), C.c_uint32(d),
                                          C.c_int(dt), C.c_int(_metric(distance_type)), C.byref(h)))
        ix = cls(h)
        ix._dt = dt
        ix._load_storage(storage)
        return ix

    def _payload_empty(self, n):
        return np.empty((n, self.info()["dimension"]),
                        {F32: np.float32, F16: np.float16, BF16: np.uint16, U8: np.float32}[getattr(self, "_dt", F32)])

    def export(self):
        i = self.info()
        K, d, n = i["num_partitions"], i["dimension"], i["num_rows"]
        cent = np.empty((K, d), np.float32)
        off = np.empty(K + 1, np.uint64)
        # the stored vectors keep the column's element type (bf16 as uint16 bit patterns; u8 columns are held as f32)
        vec = np.empty((n, d), {F32: np.float32, F16: np.float16, BF16: np.uint16, U8: np.float32}[getattr(self, "_dt", F32)])
        rid = np.empty(n, np.uint64)
        check(lib().lb2_index_export_flat(self._h, C.c_void_p(cent.ctypes.data), C.c_void_p(off.ctypes.data),
                                          C.c_void_p(vec.ctypes.data), C.c_void_p(rid.ctypes.data)))
        return dict(centroids=cent, part_offsets=off, vectors=vec, row_ids=rid)


# ---- lance-index::vector::sq -----------------------------------------------------------------
class SQBuildParams:
    """lance_index::vector::sq::builder::SQBuildParams (sq/builder.rs:7-28)."""

    def __init__(self, num_bits=8, sample_rate=256):
        self.num_bits, self.sample_rate = num_bits, sample_rate


class ScalarQuantizer:
    """lance_index::vector::sq::ScalarQuantizer (sq.rs): 8-bit codes under the bounds [lower, upper]."""

    def __init__(self, dimension, bounds=None, num_bits=8):
        self.dimension, self.num_bits = dimension, num_bits
        self.bounds = None if bounds is None else (float(bounds[0]), float(bounds[1]))

    def build(self, data, bf16=False):
        """ScalarQuantizer::build (sq.rs:67-89,152-182): the (min, max) fold over every element -> bounds."""
        data, dt = _typed(data, bf16)
        n = int(np.prod(data.shape)) // self.dimension
        lo, hi = C.c_double(0), C.c_double(0)
        dp, _k = as_ptr(data)
        check(lib().lb2_sq_train(dp, C.c_uint64(n), C.c_uint32(self.dimension), C.c_int(dt), C.byref(lo),
                                 C.byref(hi)))
        self.bounds = (lo.value, hi.value)
        return self.bounds

    def transform(self, vectors, bf16=False):
        """ScalarQuantizer::quantize = scale_to_u8 (sq.rs:263-277) -> u8 codes [n][d]."""
        vectors, dt = _typed(vectors, bf16)
        n = int(np.prod(vectors.shape)) // self.dimension
        out = np.empty((n, self.dimension), np.uint8)
        vp, _k = as_ptr(vectors)
        check(lib().lb2_sq_encode(vp, n, self.dimension, dt, self.bounds[0], self.bounds[1],
                                  C.c_void_p(out.ctypes.data)))
        return out


class IvfSqIndex(IvfPqIndex):
    """Device-resident IVFIndex<FlatIndex, ScalarQuantizer> (IVF_SQ): 8-bit scalar codes, searched with the
    reference's exact integer distances (lance-index/src/vector/sq/storage.rs:432-468)."""

    @classmethod
    def build(cls, data, distance_type="l2", num_partitions=256, max_iters=50, sample_rate=256, seed=0,
              centroids=None, row_ids=None, partition_index="exact", partition_index_batch=1, bf16=False, sq_params=None):
        """create_index(.., "IVF_SQ"); the IVF stage equals IvfFlatIndex.build's with the same arguments.
        bf16=True: `data` is a uint16 array holding bfloat16 bit patterns."""
        sq_params = sq_params or SQBuildParams()
        bp = _CSqBuildParams()
        lib().lb2_ivfsq_build_params_default(C.byref(bp))
        keep = _ivf_fields(bp, num_partitions, max_iters, sample_rate, seed, centroids,  # noqa: F841
                           partition_index, partition_index_batch)
        bp.num_bits, bp.sample_rate = sq_params.num_bits, sq_params.sample_rate
        return _build(cls, lib().lb2_ivfsq_build, bp, data, distance_type, row_ids, bf16)

    @classmethod
    def from_parts(cls, centroids, bounds, part_ids, codes, row_ids=None, distance_type="l2", dtype=np.float32,
                   bf16=False):
        """Open a reference-built IVF_SQ index: centroids, the `lance:sq` bounds (lower, upper), and the shuffle
        output (partition ids, codes [n][d], row ids).  dtype / bf16: the element type of the queries and of the
        raw column used by refine (bf16=True: uint16 bit patterns)."""
        dt = BF16 if bf16 else _DTYPES[np.dtype(dtype)]
        centroids = _model_arr(centroids, dt)
        k, d = centroids.shape
        h = C.c_void_p()
        check(lib().lb2_index_create_sq(C.c_void_p(centroids.ctypes.data), k, d, dt, _metric(distance_type),
                                        float(bounds[0]), float(bounds[1]), C.byref(h)))
        ix = cls(h)
        ix._dt = dt
        part_ids = np.ascontiguousarray(part_ids, dtype=np.uint32)
        codes = np.ascontiguousarray(codes, dtype=np.uint8)
        rid = None if row_ids is None else np.ascontiguousarray(row_ids, dtype=np.uint64)
        rp, _k = as_ptr(rid)
        check(lib().lb2_index_load_sq(h, C.c_void_p(part_ids.ctypes.data), C.c_void_p(codes.ctypes.data), rp,
                                      C.c_uint64(part_ids.size)))
        return ix

    _STORAGE_COLUMN = "__sq_code"

    @classmethod
    def from_storage(cls, centroids, bounds, storage, distance_type="l2", dtype=np.float32, bf16=False):
        """Open an index from its centroids, the `lance:sq` bounds and its storage columns, as
        IvfPqIndex.from_storage."""
        cls._check_storage_class(storage)
        dt = BF16 if bf16 else _DTYPES[np.dtype(dtype)]
        centroids = _model_arr(centroids, dt)
        k, d = centroids.shape
        h = C.c_void_p()
        check(lib().lb2_index_create_sq(C.c_void_p(centroids.ctypes.data), k, d, dt, _metric(distance_type),
                                        float(bounds[0]), float(bounds[1]), C.byref(h)))
        ix = cls(h)
        ix._dt = dt
        ix._load_storage(storage)
        return ix

    def _payload_empty(self, n):
        return np.empty((n, self.info()["dimension"]), np.uint8)

    def export(self):
        i = self.info()
        K, d, n = i["num_partitions"], i["dimension"], i["num_rows"]
        cent = np.empty((K, d), np.float32)
        bounds = np.empty(2, np.float64)
        off = np.empty(K + 1, np.uint64)
        codes = np.empty((n, d), np.uint8)
        rid = np.empty(n, np.uint64)
        check(lib().lb2_index_export_sq(self._h, C.c_void_p(cent.ctypes.data), C.c_void_p(bounds.ctypes.data),
                                        C.c_void_p(off.ctypes.data), C.c_void_p(codes.ctypes.data),
                                        C.c_void_p(rid.ctypes.data)))
        return dict(centroids=cent, bounds=(float(bounds[0]), float(bounds[1])), part_offsets=off, codes=codes,
                    row_ids=rid)


# ---- lance-index::vector::hnsw over SQ storage (IVF_HNSW_SQ) ---------------------------------------------
class HnswBuildParams:
    """lance_index::vector::hnsw::builder::HnswBuildParams (hnsw/builder.rs:47-72), plus insert_batch: B of the
    batched build (include/lance_b200.h, IVF_HNSW_SQ): nodes are inserted in deterministic rounds of up to B
    concurrent inserts (1, 2, 4, .. then B).  1 (or 0) is the serial build; at most 65536."""

    def __init__(self, max_level=7, m=20, ef_construction=150, insert_batch=1):
        self.max_level, self.m, self.ef_construction = max_level, m, ef_construction
        self.insert_batch = insert_batch


class _HnswGraphs:
    """The graph half of IvfHnswSqIndex, IvfHnswPqIndex and IvfHnswFlatIndex: attach, export and search with ef=.
    search, search_refine, search_ex and search_probed take ef= (lb2_index_search_hnsw); the other search methods use
    k' + k' / 2."""
    _KIND = None   # "sq", "pq" or "flat": the suffix of the kind's C entry points

    @classmethod
    def _need_graph(cls, graph):
        if graph is None:
            raise ValueError(f"{cls.__name__}.from_parts needs graph= (the dict export()['graph'] returns)")

    def _attach_graph(self, graph):
        """lb2_index_load_hnsw_sq / _pq / _flat of a dict as export()["graph"] returns"""
        g = graph
        arr = {k: np.ascontiguousarray(g[k], dtype=t) for k, t in (
            ("levels", np.uint8), ("counts0", np.uint32), ("neighbors0", np.uint32), ("dists0", np.float32),
            ("counts_up", np.uint32), ("neighbors_up", np.uint32), ("dists_up", np.float32))}
        ptr = {k: C.c_void_p(v.ctypes.data) if v.size else None for k, v in arr.items()}
        check(getattr(lib(), f"lb2_index_load_hnsw_{self._KIND}")(
            self._h, C.c_uint32(g["max_level"]), C.c_uint32(g["m"]), C.c_uint32(g.get("ef_construction", 0)),
            ptr["levels"], ptr["counts0"], ptr["neighbors0"], ptr["dists0"], ptr["counts_up"], ptr["neighbors_up"],
            ptr["dists_up"]))

    def export(self, *args):
        """the parent kind's export plus "graph": the HNSW graphs in the device layout of include/lance_b200.h."""
        out = super().export(*args)
        n = self.info()["num_rows"]
        ml, m, efc, nu = C.c_uint32(), C.c_uint32(), C.c_uint32(), C.c_uint64()
        check(getattr(lib(), f"lb2_index_hnsw_{self._KIND}_info")(self._h, C.byref(ml), C.byref(m), C.byref(efc), C.byref(nu)))
        m, nu = m.value, nu.value
        g = dict(max_level=ml.value, m=m, ef_construction=efc.value, levels=np.empty(n, np.uint8),
                 counts0=np.empty(n, np.uint32), neighbors0=np.empty((n, 2 * m), np.uint32),
                 dists0=np.empty((n, 2 * m), np.float32), counts_up=np.empty(nu, np.uint32),
                 neighbors_up=np.empty((nu, m), np.uint32), dists_up=np.empty((nu, m), np.float32))
        ptr = {k: C.c_void_p(v.ctypes.data) if isinstance(v, np.ndarray) and v.size else None for k, v in g.items()}
        check(getattr(lib(), f"lb2_index_export_hnsw_{self._KIND}")(self._h, ptr["levels"], ptr["counts0"], ptr["neighbors0"], ptr["dists0"],
                                             ptr["counts_up"], ptr["neighbors_up"], ptr["dists_up"]))
        out["graph"] = g
        return out

    def optimize(self, add_vectors=None, add_row_ids=None, add_part_ids=None, add_payload=None, add_factors=None,
                 new_centroids=None, part_map=None, remove_row_ids=None, remap=None, seed=0, insert_batch=None):
        """the parent kind's optimize; insert_batch: B of the rebuilt partitions' graphs (None: the B this index was
        built with, 1 for a loaded graph).  Kept partitions keep their graphs verbatim."""
        return self._optimize(add_vectors, add_row_ids, add_part_ids, add_payload, add_factors, new_centroids, part_map,
                              remove_row_ids, remap, seed, 0 if insert_batch is None else int(insert_batch))

    def split(self, part, vectors, row_ids, cand_vectors=None, cand_row_ids=None, cand_part_ids=None,
              add_vectors=None, add_row_ids=None, add_part_ids=None, add_payload=None, add_factors=None,
              remove_row_ids=None, seed=0, insert_batch=None):
        """the parent kind's split; insert_batch as in optimize"""
        return self._split(part, vectors, row_ids, cand_vectors, cand_row_ids, cand_part_ids, add_vectors, add_row_ids,
                           add_part_ids, add_payload, add_factors, remove_row_ids, seed,
                           0 if insert_batch is None else int(insert_batch))

    def join(self, part, vectors, row_ids, remove_row_ids=None, remap=None, seed=0, insert_batch=None):
        """the parent kind's join; insert_batch as in optimize"""
        return self._join(part, vectors, row_ids, remove_row_ids, remap, seed,
                          0 if insert_batch is None else int(insert_batch))

    def _search_hnsw(self, queries, k, nprobes, ef, probe=None, allow_bitmap=None, refine_factor=0, vectors=None,
                     lower_bound=None, upper_bound=None):
        """lb2_index_search_hnsw: search_ex (probe None) or search_probed (probe = ProbeParams) with this call's ef"""
        from ._lib import SearchParams
        npdt = {F32: np.float32, F16: np.float16, U8: np.uint8, BF16: np.uint16}[getattr(self, "_dt", F32)]
        if not isinstance(queries, (DeviceArray, PinnedArray)):
            queries = np.ascontiguousarray(queries, dtype=npdt)
        if vectors is not None and not isinstance(vectors, (DeviceArray, PinnedArray)):
            vectors = np.ascontiguousarray(vectors, dtype=npdt)
        nq = queries.shape[0]
        ids, dists = np.empty((nq, k), np.uint64), np.empty((nq, k), np.float32)
        counts, nprobes_out = np.empty(nq, np.uint32), np.empty(nq, np.uint32)
        qp, _k1 = as_ptr(queries)
        vp, _k0 = as_ptr(vectors)
        bp, _k4 = as_ptr(None if allow_bitmap is None else (allow_bitmap if isinstance(allow_bitmap, (DeviceArray, PinnedArray)) else np.ascontiguousarray(allow_bitmap, dtype=np.uint64)))
        sp = SearchParams(k, nprobes, refine_factor, vp.value if vp is not None else None,
                          0 if vectors is None else vectors.shape[0], bp.value if bp is not None else None,
                          int(lower_bound is not None), int(upper_bound is not None),
                          float(lower_bound or 0.0), float(upper_bound or 0.0))
        check(lib().lb2_index_search_hnsw(self._h, qp, C.c_uint64(nq), C.byref(sp),
                                          None if probe is None else C.byref(probe), C.c_uint32(int(ef)),
                                          as_ptr(ids)[0], as_ptr(dists)[0], as_ptr(counts)[0],
                                          None if probe is None else as_ptr(nprobes_out)[0]))
        return ids, dists, counts, nprobes_out

    def search(self, queries, k=10, nprobes=1, out=None, ef=None):
        """IvfPqIndex.search; ef: the graph search's ef for this call (None: k + k / 2)."""
        if ef is None:
            return super().search(queries, k, nprobes, out)
        ids, dists, _, _ = self._search_hnsw(queries, k, nprobes, ef)
        if out is not None:
            out[0][...], out[1][...] = ids, dists
            return out
        return ids, dists

    def search_refine(self, vectors, queries, k=10, nprobes=1, refine_factor=1, out=None, ef=None):
        """IvfPqIndex.search_refine; ef as in search (None: k' + k' / 2, k' = k * refine_factor)."""
        if ef is None:
            return super().search_refine(vectors, queries, k, nprobes, refine_factor, out)
        ids, dists, _, _ = self._search_hnsw(queries, k, nprobes, ef, refine_factor=refine_factor, vectors=vectors)
        return ids, dists

    def search_ex(self, queries, k=10, nprobes=1, allow_bitmap=None, refine_factor=0, vectors=None, out=None,
                  lower_bound=None, upper_bound=None, ef=None):
        """IvfPqIndex.search_ex; ef as in search_refine."""
        if ef is None:
            return super().search_ex(queries, k, nprobes, allow_bitmap, refine_factor, vectors, out, lower_bound,
                                     upper_bound)
        ids, dists, _, _ = self._search_hnsw(queries, k, nprobes, ef, None, allow_bitmap, refine_factor, vectors,
                                             lower_bound, upper_bound)
        return ids, dists

    def search_probed(self, queries, k, minimum_nprobes=1, maximum_nprobes=None, late_width=1, allow_bitmap=None,
                      mask_ids=None, mask_max_len=None, refine_factor=0, vectors=None, lower_bound=None,
                      upper_bound=None, ef=None):
        """IvfPqIndex.search_probed; ef as in search_refine (mask_ids needs ef=None)."""
        if ef is None:
            return super().search_probed(queries, k, minimum_nprobes, maximum_nprobes, late_width, allow_bitmap,
                                         mask_ids, mask_max_len, refine_factor, vectors, lower_bound, upper_bound)
        if mask_ids is not None:
            raise ValueError("search_probed with ef: mask_ids is not supported; pass ef=None")
        from ._lib import ProbeParams
        pp = ProbeParams(minimum_nprobes, maximum_nprobes or 0, late_width, int(mask_max_len is not None),
                         int(mask_max_len or 0), None, 0)
        return self._search_hnsw(queries, k, 0, ef, pp, allow_bitmap, refine_factor, vectors, lower_bound,
                                 upper_bound)



class IvfHnswSqIndex(_HnswGraphs, IvfSqIndex):
    """Device-resident IVFIndex<HNSW, ScalarQuantizer> (IVF_HNSW_SQ): IVF_SQ's partitions, bounds and codes with an
    HNSW graph per partition over the codes (lance-index/src/vector/hnsw/builder.rs).  search, search_refine,
    search_ex and search_probed take ef= (lb2_index_search_hnsw); the other search methods use k' + k' / 2."""

    @classmethod
    def build(cls, data, distance_type="l2", num_partitions=256, max_iters=50, sample_rate=256, seed=0,
              centroids=None, row_ids=None, partition_index="exact", partition_index_batch=1, bf16=False, sq_params=None, hnsw_params=None):
        """create_index(.., "IVF_HNSW_SQ"); the IVF stage, bounds and codes equal IvfSqIndex.build's with the same
        arguments.  The graphs' level draws use `seed`."""
        sq_params = sq_params or SQBuildParams()
        bp = _CHnswSqBuildParams()
        lib().lb2_ivfhnswsq_build_params_default(C.byref(bp))
        keep = _ivf_fields(bp.sq, num_partitions, max_iters, sample_rate, seed, centroids,  # noqa: F841
                           partition_index, partition_index_batch)
        bp.sq.num_bits, bp.sq.sample_rate = sq_params.num_bits, sq_params.sample_rate
        _hnsw_fields(bp, hnsw_params)
        return _build(cls, lib().lb2_ivfhnswsq_build, bp, data, distance_type, row_ids, bf16)

    _KIND = "sq"

    @classmethod
    def from_parts(cls, centroids, bounds, part_ids, codes, row_ids=None, distance_type="l2", dtype=np.float32,
                   bf16=False, graph=None):
        """IvfSqIndex.from_parts plus `graph`: a dict as export()["graph"] returns (max_level, m, ef_construction,
        levels, counts0, neighbors0, dists0, counts_up, neighbors_up, dists_up) over the rows in partition order."""
        cls._need_graph(graph)
        ix = super().from_parts(centroids, bounds, part_ids, codes, row_ids, distance_type, dtype, bf16)
        ix._attach_graph(graph)
        return ix


class IvfHnswPqIndex(_HnswGraphs, IvfPqIndex):
    """Device-resident IVFIndex<HNSW, ProductQuantizer> (IVF_HNSW_PQ): IVF_PQ's partitions, codebook and codes with an
    HNSW graph per partition over the PQ storage (lance-index/src/vector/pq/storage.rs:600-1037).  A query scores a
    node from the IVF_PQ scan's table; a node being inserted scores others from the table of its own decoded codes,
    and the heuristic compares the decoded rows (include/lance_b200.h).  search, search_refine, search_ex and
    search_probed take ef=; the other search methods use k' + k' / 2."""
    _KIND = "pq"

    @classmethod
    def build(cls, data, distance_type="l2", params=None, hnsw_params=HnswBuildParams(), row_ids=None, bf16=False):
        """create_index(.., "IVF_HNSW_PQ"); the IVF stage, codebook and codes equal IvfPqIndex.build's with the same
        arguments.  The graphs' level draws use params.seed."""
        bp = _CHnswPqBuildParams()
        lib().lb2_ivfhnswpq_build_params_default(C.byref(bp))
        keep = _fill_build_params(bp.pq, params or IvfBuildParams())  # noqa: F841 (alive across the build)
        _hnsw_fields(bp, hnsw_params)
        return _build(cls, lib().lb2_ivfhnswpq_build, bp, data, distance_type, row_ids, bf16)

    @classmethod
    def from_parts(cls, centroids, codebook, part_ids, codes, row_ids=None, distance_type="l2", num_bits=8,
                   dtype=np.float32, bf16=False, graph=None):
        """IvfPqIndex.from_parts plus `graph` (as export()["graph"] returns).  dtype / bf16: the column's element type
        (bf16=True: uint16 bit patterns), which picks the heuristic's distance rule and the type of the queries."""
        cls._need_graph(graph)
        dt = BF16 if bf16 else _DTYPES[np.dtype(dtype)]
        centroids, codebook = _model_arr(centroids, dt), _model_arr(codebook, dt)
        k, d = centroids.shape
        M = codebook.shape[0]
        h = C.c_void_p()
        check(lib().lb2_index_create(C.c_void_p(centroids.ctypes.data), C.c_uint32(k), C.c_uint32(d),
                                     C.c_int(dt), C.c_int(_metric(distance_type)),
                                     C.c_void_p(codebook.ctypes.data), C.c_uint32(M), C.c_uint32(num_bits),
                                     C.byref(h)))
        ix = cls(h)
        ix._dt = dt
        part_ids = np.ascontiguousarray(part_ids, dtype=np.uint32)
        codes = np.ascontiguousarray(codes, dtype=np.uint8)
        rid = None if row_ids is None else np.ascontiguousarray(row_ids, dtype=np.uint64)
        rp, _k = as_ptr(rid)
        check(lib().lb2_index_load(h, C.c_void_p(part_ids.ctypes.data), C.c_void_p(codes.ctypes.data), rp,
                                   C.c_uint64(part_ids.size)))
        ix._attach_graph(graph)
        return ix


class IvfHnswFlatIndex(_HnswGraphs, IvfFlatIndex):
    """Device-resident IVFIndex<HNSW, FlatQuantizer> (IVF_HNSW_FLAT): IVF_FLAT's partitions, vectors and row ids with
    an HNSW graph per partition over the stored rows (lance-index/src/vector/flat/storage.rs).  Every distance, cosine
    included, is the one IVF_FLAT's scan computes for the pair; the heuristic's dist_between(u, v) puts the candidate
    u in the query role (include/lance_b200.h).  search, search_refine, search_ex and search_probed take ef=; the
    other search methods use k' + k' / 2."""
    _KIND = "flat"

    @classmethod
    def build(cls, data, distance_type="l2", num_partitions=256, max_iters=50, sample_rate=256, seed=0,
              centroids=None, row_ids=None, partition_index="exact", partition_index_batch=1, bf16=False, hnsw_params=None):
        """create_index(.., "IVF_HNSW_FLAT"); the IVF stage, vectors and row ids equal IvfFlatIndex.build's with the
        same arguments.  The graphs' level draws use `seed`.  bf16=True: uint16 bfloat16 bit patterns."""
        bp = _CHnswFlatBuildParams()
        lib().lb2_ivfhnswflat_build_params_default(C.byref(bp))
        keep = _ivf_fields(bp.flat, num_partitions, max_iters, sample_rate, seed, centroids,  # noqa: F841
                           partition_index, partition_index_batch)
        _hnsw_fields(bp, hnsw_params)
        return _build(cls, lib().lb2_ivfhnswflat_build, bp, data, distance_type, row_ids, bf16)

    @classmethod
    def from_parts(cls, centroids, part_ids, vectors, row_ids=None, distance_type="l2", bf16=False, graph=None):
        """IvfFlatIndex.from_parts plus `graph` (as export()["graph"] returns) over the rows in partition order.  The
        centroids may also be f32 as export() returns them for a bf16 column (their bits are kept)."""
        cls._need_graph(graph)
        centroids = _model_arr(centroids, BF16 if bf16 else _typed(vectors)[1])
        ix = super().from_parts(centroids, part_ids, vectors, row_ids, distance_type, bf16)
        ix._attach_graph(graph)
        return ix


# ---- lance-index::vector::bq (RaBitQ) -------------------------------------------------------------
class RQBuildParams:
    """lance_index::vector::bq::builder::RQBuildParams (bq/builder.rs:30-45)."""

    def __init__(self, num_bits=1):
        self.num_bits = num_bits


class RabitQuantizer:
    """lance_index::vector::bq::builder::RabitQuantizer: the rotation R [code_dim][code_dim] (code_dim = d * num_bits,
    of which the first d columns are used) and the transform of rows into sign codes and factors."""

    def __init__(self, dimension, num_bits=1, rotation=None):
        self.dimension, self.num_bits = dimension, num_bits
        self.code_dim = dimension * num_bits
        self.rotation = None if rotation is None else np.ascontiguousarray(rotation, dtype=np.float32)

    def build(self, seed=0):
        """random_orthogonal (bq/builder.rs:309-367), drawn on the device from `seed` -> rotation."""
        r = np.empty((self.code_dim, self.code_dim), np.float32)
        check(lib().lb2_rq_rotation(self.code_dim, seed, C.c_void_p(r.ctypes.data)))
        self.rotation = r
        return r

    def transform(self, centroids, vectors, distance_type="l2"):
        """The IVF_RQ transform of rows (ivf.rs:281-328, bq/transform.rs:70-220) -> dict of part_ids, codes
        [n][code_dim / 8], add_factors, scale_factors and valid (False: the row was dropped)."""
        centroids = np.ascontiguousarray(centroids, dtype=np.float32)
        vectors, dt = _typed(vectors)
        k, d = centroids.shape
        n = vectors.shape[0]
        part, valid = np.empty(n, np.uint32), np.empty(n, np.uint8)
        codes = np.empty((n, self.code_dim // 8), np.uint8)
        add, scale = np.empty(n, np.float32), np.empty(n, np.float32)
        vp, _k = as_ptr(vectors)
        check(lib().lb2_ivfrq_transform(C.c_void_p(centroids.ctypes.data), C.c_uint32(k),
                                        C.c_void_p(self.rotation.ctypes.data), C.c_uint32(d),
                                        C.c_uint32(self.num_bits), C.c_int(dt), C.c_int(_metric(distance_type)), vp,
                                        C.c_uint64(n), C.c_void_p(part.ctypes.data), C.c_void_p(codes.ctypes.data),
                                        C.c_void_p(add.ctypes.data), C.c_void_p(scale.ctypes.data),
                                        C.c_void_p(valid.ctypes.data)))
        return dict(part_ids=part, codes=codes, add_factors=add, scale_factors=scale, valid=valid.astype(bool))


class IvfRqIndex(IvfPqIndex):
    """Device-resident IVFIndex<FlatIndex, RabitQuantizer> (IVF_RQ): 1-bit codes of rotated residuals, scored from
    the reference's 4-bit distance tables (lance-index/src/vector/bq/storage.rs:160-445)."""

    @classmethod
    def build(cls, data, distance_type="l2", num_partitions=256, max_iters=50, sample_rate=256, seed=0,
              centroids=None, row_ids=None, partition_index="exact", partition_index_batch=1, rq_params=None):
        """create_index(.., "IVF_RQ"); the IVF stage equals IvfFlatIndex.build's with the same arguments, the
        rotation is drawn from seed + 1.  f32 columns."""
        bp = _CRqBuildParams()
        lib().lb2_ivfrq_build_params_default(C.byref(bp))
        keep = _ivf_fields(bp, num_partitions, max_iters, sample_rate, seed, centroids,  # noqa: F841
                           partition_index, partition_index_batch)
        bp.num_bits = (rq_params or RQBuildParams()).num_bits
        return _build(cls, lib().lb2_ivfrq_build, bp, data, distance_type, row_ids)

    @classmethod
    def from_parts(cls, centroids, rotation, part_ids, codes, add_factors, scale_factors, row_ids=None,
                   distance_type="l2", num_bits=1, dtype=np.float32):
        """Open a reference-built IVF_RQ index: centroids, the `lance:rabit` rotation [code_dim][code_dim], and the
        rows (partition ids, unpacked codes [n][code_dim / 8], add / scale factors, row ids)."""
        dt = _DTYPES[np.dtype(dtype)]
        centroids = np.ascontiguousarray(centroids, dtype=_model_np(dt))
        rotation = np.ascontiguousarray(rotation, dtype=_model_np(dt))
        k, d = centroids.shape
        h = C.c_void_p()
        check(lib().lb2_index_create_rq(C.c_void_p(centroids.ctypes.data), C.c_uint32(k), C.c_uint32(d), C.c_int(dt),
                                        C.c_int(_metric(distance_type)), C.c_void_p(rotation.ctypes.data),
                                        C.c_uint32(num_bits), C.byref(h)))
        ix = cls(h)
        ix._dt = dt
        part_ids = np.ascontiguousarray(part_ids, dtype=np.uint32)
        codes = np.ascontiguousarray(codes, dtype=np.uint8)
        add = np.ascontiguousarray(add_factors, dtype=np.float32)
        scale = np.ascontiguousarray(scale_factors, dtype=np.float32)
        rid = None if row_ids is None else np.ascontiguousarray(row_ids, dtype=np.uint64)
        rp, _k = as_ptr(rid)
        check(lib().lb2_index_load_rq(h, C.c_void_p(part_ids.ctypes.data), C.c_void_p(codes.ctypes.data),
                                      C.c_void_p(add.ctypes.data), C.c_void_p(scale.ctypes.data), rp,
                                      C.c_uint64(part_ids.size)))
        return ix

    _STORAGE_COLUMN = "__rabit_code"

    @classmethod
    def from_storage(cls, centroids, rotation, storage, distance_type="l2", num_bits=1, dtype=np.float32):
        """Open an index from its centroids, the `lance:rabit` rotation and its storage columns (the packed
        "__rabit_code", "__add_factors", "__scale_factors"), as IvfPqIndex.from_storage."""
        cls._check_storage_class(storage)
        dt = _DTYPES[np.dtype(dtype)]
        centroids = np.ascontiguousarray(centroids, dtype=_model_np(dt))
        rotation = np.ascontiguousarray(rotation, dtype=_model_np(dt))
        k, d = centroids.shape
        h = C.c_void_p()
        check(lib().lb2_index_create_rq(C.c_void_p(centroids.ctypes.data), C.c_uint32(k), C.c_uint32(d), C.c_int(dt),
                                        C.c_int(_metric(distance_type)), C.c_void_p(rotation.ctypes.data),
                                        C.c_uint32(num_bits), C.byref(h)))
        ix = cls(h)
        ix._dt = dt
        ix._load_storage(storage)
        return ix

    def _payload_empty(self, n):
        i = self.info()
        return np.empty((n, i["dimension"] * i["num_bits"] // 8), np.uint8)

    def export(self):
        i = self.info()
        K, d, nb, n = i["num_partitions"], i["dimension"], i["num_bits"], i["num_rows"]
        cd = d * nb
        cent = np.empty((K, d), np.float32)
        rot = np.empty((cd, cd), np.float32)
        off = np.empty(K + 1, np.uint64)
        codes = np.empty((n, cd // 8), np.uint8)
        add, scale = np.empty(n, np.float32), np.empty(n, np.float32)
        rid = np.empty(n, np.uint64)
        check(lib().lb2_index_export_rq(self._h, C.c_void_p(cent.ctypes.data), C.c_void_p(rot.ctypes.data),
                                        C.c_void_p(off.ctypes.data), C.c_void_p(codes.ctypes.data),
                                        C.c_void_p(add.ctypes.data), C.c_void_p(scale.ctypes.data),
                                        C.c_void_p(rid.ctypes.data)))
        return dict(centroids=cent, rotation=rot, part_offsets=off, codes=codes, add_factors=add,
                    scale_factors=scale, row_ids=rid)
