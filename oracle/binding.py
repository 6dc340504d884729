"""ctypes binding of the CPU oracle (oracle/lance_oracle.cc).

TEST INFRASTRUCTURE ONLY: importable from tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs.  The product package (lance_b200/) never imports this.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "liblance_oracle.so")

METRIC = {"l2": 0, "cosine": 1, "dot": 2}


def build(force=False):
    src = os.path.join(_HERE, "lance_oracle.cc")
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", _HERE, "all"], stdout=subprocess.DEVNULL)
    return _SO


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(_SO)
        L = _lib
        f32p, u8p, u32p, u64p = (C.POINTER(C.c_float), C.POINTER(C.c_uint8),
                                 C.POINTER(C.c_uint32), C.POINTER(C.c_uint64))
        for name in ("lo_l2_f32", "lo_dot_f32", "lo_cosine_f32"):
            getattr(L, name).restype = C.c_float
            getattr(L, name).argtypes = [f32p, f32p, C.c_uint64]
        L.lo_norm_l2_f32.restype = C.c_float
        L.lo_norm_l2_f32.argtypes = [f32p, C.c_uint64]
        L.lo_l2_u8.restype = C.c_float
        L.lo_l2_u8.argtypes = [u8p, u8p, C.c_uint64]
        L.lo_dot_u8.restype = C.c_float
        L.lo_dot_u8.argtypes = [u8p, u8p, C.c_uint64]
        for name in ("lo_l2_f16", "lo_l2_bf16", "lo_dot_f16", "lo_dot_bf16"):
            getattr(L, name).restype = C.c_float
            getattr(L, name).argtypes = [C.POINTER(C.c_uint16), C.POINTER(C.c_uint16), C.c_uint64]
        L.lo_normalize_f32.restype = C.c_float
        L.lo_kmeans_train.restype = C.c_int
        L.lo_flat_topk.restype = C.c_uint64
        L.lo_hardware_threads.restype = C.c_int
    return _lib


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t)) if a is not None else None


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def nthreads_default():
    return max(1, lib().lo_hardware_threads())


def l2(x, y):
    x, y = _f32(x), _f32(y)
    return float(lib().lo_l2_f32(_p(x, C.c_float), _p(y, C.c_float), x.size))


def dot(x, y):
    x, y = _f32(x), _f32(y)
    return float(lib().lo_dot_f32(_p(x, C.c_float), _p(y, C.c_float), x.size))


def cosine(x, y):
    x, y = _f32(x), _f32(y)
    return float(lib().lo_cosine_f32(_p(x, C.c_float), _p(y, C.c_float), x.size))


def l2_u8(x, y):
    x = np.ascontiguousarray(x, dtype=np.uint8)
    y = np.ascontiguousarray(y, dtype=np.uint8)
    return float(lib().lo_l2_u8(_p(x, C.c_uint8), _p(y, C.c_uint8), x.size))


def l2_f16(x, y):
    x = np.ascontiguousarray(x, dtype=np.float16).view(np.uint16)
    y = np.ascontiguousarray(y, dtype=np.float16).view(np.uint16)
    return float(lib().lo_l2_f16(_p(x, C.c_uint16), _p(y, C.c_uint16), x.size))


def _bits16(a, dtype):
    """16-bit elements as uint16 bit patterns: float16 arrays, or uint16 arrays holding bfloat16 patterns."""
    return np.ascontiguousarray(a, dtype=dtype).view(np.uint16)


def l2_bf16(x, y):
    """x, y: uint16 arrays of bfloat16 bit patterns (numpy has no bf16 dtype)."""
    x, y = _bits16(x, np.uint16), _bits16(y, np.uint16)
    return float(lib().lo_l2_bf16(_p(x, C.c_uint16), _p(y, C.c_uint16), x.size))


def dot_f16(x, y):
    """Dot for f16 (dot.rs:105-136 scalar fallback): 32 f32 lanes."""
    x, y = _bits16(x, np.float16), _bits16(y, np.float16)
    return float(lib().lo_dot_f16(_p(x, C.c_uint16), _p(y, C.c_uint16), x.size))


def dot_bf16(x, y):
    """Dot for bf16 (dot.rs:78-83): 32 f32 lanes; x, y are uint16 arrays of bfloat16 bit patterns."""
    x, y = _bits16(x, np.uint16), _bits16(y, np.uint16)
    return float(lib().lo_dot_bf16(_p(x, C.c_uint16), _p(y, C.c_uint16), x.size))


def dot_u8(x, y):
    """Dot for u8 (dot.rs:152-161): exact u32 sum, one conversion to f32."""
    x = np.ascontiguousarray(x, dtype=np.uint8)
    y = np.ascontiguousarray(y, dtype=np.uint8)
    return float(lib().lo_dot_u8(_p(x, C.c_uint8), _p(y, C.c_uint8), x.size))


def l2_batch(frm, to, d):
    frm, to = _f32(frm), _f32(to)
    n = to.size // d
    out = np.empty(n, np.float32)
    lib().lo_l2_batch_f32(_p(frm, C.c_float), _p(to, C.c_float), C.c_uint64(n), C.c_uint64(d),
                          _p(out, C.c_float))
    return out


def normalize_rows(x, nthreads=1):
    x = _f32(x)
    out = np.empty_like(x)
    n, d = x.shape
    lib().lo_normalize_rows_f32(_p(x, C.c_float), C.c_uint64(n), C.c_uint64(d), _p(out, C.c_float),
                                C.c_int(nthreads))
    return out


def compute_membership(centroids, data, metric="l2", balance_factor=0.0, cluster_sizes=None,
                       nthreads=1):
    centroids, data = _f32(centroids), _f32(data)
    k, d = centroids.shape
    n = data.shape[0]
    ids = np.empty(n, np.uint32)
    dists = np.empty(n, np.float32)
    valid = np.empty(n, np.uint8)
    cs = None if cluster_sizes is None else np.ascontiguousarray(cluster_sizes, dtype=np.uint64)
    lib().lo_compute_membership(_p(centroids, C.c_float), C.c_uint64(k), C.c_uint64(d),
                                _p(data, C.c_float), C.c_uint64(n), C.c_int(METRIC[metric]),
                                C.c_float(balance_factor), _p(cs, C.c_uint64), _p(ids, C.c_uint32),
                                _p(dists, C.c_float), _p(valid, C.c_uint8), C.c_int(nthreads))
    return ids, dists, valid.astype(bool)


def kmeans_train(data, k, max_iters=50, tolerance=1e-4, balance_factor=0.0, metric="l2", seed=0,
                 init_centroids=None, nthreads=1):
    """balance_factor is the post-division value (reference: params.balance_factor / n)."""
    data = _f32(data)
    n, d = data.shape
    init = None if init_centroids is None else _f32(init_centroids)
    out = np.empty((k, d), np.float32)
    loss = C.c_double(0)
    it = lib().lo_kmeans_train(_p(data, C.c_float), C.c_uint64(n), C.c_uint64(d), C.c_uint64(k),
                               C.c_int(max_iters), C.c_double(tolerance),
                               C.c_float(balance_factor), C.c_int(METRIC[metric]),
                               C.c_uint64(seed), _p(init, C.c_float), _p(out, C.c_float),
                               C.byref(loss), C.c_int(nthreads))
    return out, loss.value, it


def find_partitions(centroids, query, nprobes, metric="l2"):
    centroids, query = _f32(centroids), _f32(query)
    k, d = centroids.shape
    p = min(nprobes, k)
    ids = np.empty(p, np.uint32)
    dists = np.empty(p, np.float32)
    lib().lo_find_partitions(_p(centroids, C.c_float), C.c_uint64(k), C.c_uint64(d),
                             _p(query, C.c_float), C.c_uint64(nprobes), C.c_int(METRIC[metric]),
                             _p(ids, C.c_uint32), _p(dists, C.c_float))
    return ids, dists


def compute_residual(centroids, vectors, part_ids, nthreads=1):
    centroids, vectors = _f32(centroids), _f32(vectors)
    part_ids = np.ascontiguousarray(part_ids, dtype=np.uint32)
    n, d = vectors.shape
    out = np.empty_like(vectors)
    lib().lo_compute_residual(_p(centroids, C.c_float), C.c_uint64(d), _p(vectors, C.c_float),
                              C.c_uint64(n), _p(part_ids, C.c_uint32), _p(out, C.c_float),
                              C.c_int(nthreads))
    return out


def pq_train(data, M, nbits=8, max_iters=50, sample_rate=256, metric="l2", seed=0,
             init_codebook=None, nthreads=1):
    data = _f32(data)
    n, d = data.shape
    k = 1 << nbits
    init = None if init_codebook is None else _f32(init_codebook)
    out = np.empty((M, k, d // M), np.float32)
    iters = np.zeros(M, np.int32)
    lib().lo_pq_train(_p(data, C.c_float), C.c_uint64(n), C.c_uint64(d), C.c_uint64(M),
                      C.c_int(nbits), C.c_int(max_iters), C.c_uint64(sample_rate),
                      C.c_int(METRIC[metric]), C.c_uint64(seed), _p(init, C.c_float),
                      _p(out, C.c_float), _p(iters, C.c_int), C.c_int(nthreads))
    return out, iters


def pq_encode(codebook, vectors, nbits=8, metric="l2", nthreads=1):
    codebook, vectors = _f32(codebook), _f32(vectors)
    M = codebook.shape[0]
    n, d = vectors.shape
    bpr = M // 2 if nbits == 4 else M
    out = np.empty((n, bpr), np.uint8)
    lib().lo_pq_encode(_p(codebook, C.c_float), C.c_uint64(M), C.c_int(nbits), C.c_uint64(d),
                       C.c_int(METRIC[metric]), _p(vectors, C.c_float), C.c_uint64(n),
                       _p(out, C.c_uint8), C.c_int(nthreads))
    return out


def build_lut(codebook, query, nbits=8, metric="l2"):
    codebook, query = _f32(codebook), _f32(query)
    M = codebook.shape[0]
    d = query.size
    out = np.empty(M * (1 << nbits), np.float32)
    lib().lo_build_lut(_p(codebook, C.c_float), C.c_int(nbits), C.c_uint64(M), C.c_uint64(d),
                       C.c_int(METRIC[metric]), _p(query, C.c_float), _p(out, C.c_float))
    return out


def transpose_codes(codes):
    codes = np.ascontiguousarray(codes, dtype=np.uint8)
    n, M = codes.shape
    out = np.empty((M, n), np.uint8)
    lib().lo_transpose_codes(_p(codes, C.c_uint8), C.c_uint64(n), C.c_uint64(M), _p(out, C.c_uint8))
    return out


def pq_scan(lut, codes_t, metric="l2"):
    lut = _f32(lut)
    codes_t = np.ascontiguousarray(codes_t, dtype=np.uint8)
    M, n = codes_t.shape
    out = np.empty(n, np.float32)
    lib().lo_pq_scan(_p(lut, C.c_float), C.c_uint64(M), _p(codes_t, C.c_uint8), C.c_uint64(n),
                     C.c_int(METRIC[metric]), _p(out, C.c_float))
    return out


def flat_topk(dists, row_ids, k, lower=None, upper=None):
    dists = _f32(dists)
    n = dists.size
    rid = None if row_ids is None else np.ascontiguousarray(row_ids, dtype=np.uint64)
    oi = np.empty(k, np.uint64)
    od = np.empty(k, np.float32)
    use_range = lower is not None or upper is not None
    lo = np.finfo(np.float32).min if lower is None else lower
    hi = np.finfo(np.float32).max if upper is None else upper
    got = lib().lo_flat_topk(_p(dists, C.c_float), _p(rid, C.c_uint64), C.c_uint64(n),
                             C.c_uint64(k), C.c_int(int(use_range)), C.c_float(lo), C.c_float(hi),
                             _p(oi, C.c_uint64), _p(od, C.c_float))
    return oi[:got], od[:got]


def flat_distance_all(query, vectors, metric="l2", nthreads=1):
    query, vectors = _f32(query), _f32(vectors)
    n, d = vectors.shape
    out = np.empty(n, np.float32)
    lib().lo_flat_distance_all(_p(query, C.c_float), _p(vectors, C.c_float), C.c_uint64(n),
                               C.c_uint64(d), C.c_int(METRIC[metric]), _p(out, C.c_float),
                               C.c_int(nthreads))
    return out


def _mask_args(allow, block):
    a = None if allow is None else np.ascontiguousarray(np.sort(np.asarray(allow, dtype=np.uint64)))
    b = None if block is None else np.ascontiguousarray(np.sort(np.asarray(block, dtype=np.uint64)))
    keep = (a, b)
    return keep, [(_p(a, C.c_uint64) if a is not None and a.size else None), C.c_uint64(0 if a is None else a.size),
                  C.c_int(a is not None),
                  (_p(b, C.c_uint64) if b is not None and b.size else None), C.c_uint64(0 if b is None else b.size),
                  C.c_int(b is not None)]


def ivfpq_search(centroids, codebook, part_offsets, codes, row_ids, queries, k, nprobes,
                 metric="l2", nbits=8, nthreads=1, allow=None, block=None, lower=None, upper=None):
    centroids, codebook, queries = _f32(centroids), _f32(codebook), _f32(queries)
    K, d = centroids.shape
    M = codebook.shape[0]
    po = np.ascontiguousarray(part_offsets, dtype=np.uint64)
    codes = np.ascontiguousarray(codes, dtype=np.uint8)
    rid = np.ascontiguousarray(row_ids, dtype=np.uint64)
    nq = queries.shape[0]
    oi = np.empty((nq, k), np.uint64)
    od = np.empty((nq, k), np.float32)
    oc = np.empty(nq, np.uint32)
    if lower is not None or upper is not None:  # range branch (flat/index.rs:100-115,131-148)
        keep, margs = _mask_args(allow, block)
        lib().lo_ivfpq_search_ex(_p(centroids, C.c_float), C.c_uint64(K), C.c_uint64(d),
                                 C.c_int(METRIC[metric]), _p(codebook, C.c_float), C.c_uint64(M),
                                 C.c_int(nbits), _p(po, C.c_uint64), _p(codes, C.c_uint8),
                                 _p(rid, C.c_uint64), _p(queries, C.c_float), C.c_uint64(nq),
                                 C.c_uint64(k), C.c_uint64(nprobes), *margs,
                                 C.c_int(lower is not None), C.c_float(lower or 0.0),
                                 C.c_int(upper is not None), C.c_float(upper or 0.0), _p(oi, C.c_uint64),
                                 _p(od, C.c_float), _p(oc, C.c_uint32), C.c_int(nthreads))
        return oi, od, oc
    if allow is not None or block is not None:  # prefilter path (flat/index.rs:129-165)
        keep, margs = _mask_args(allow, block)
        lib().lo_ivfpq_search_masked(_p(centroids, C.c_float), C.c_uint64(K), C.c_uint64(d),
                                     C.c_int(METRIC[metric]), _p(codebook, C.c_float), C.c_uint64(M),
                                     C.c_int(nbits), _p(po, C.c_uint64), _p(codes, C.c_uint8),
                                     _p(rid, C.c_uint64), _p(queries, C.c_float), C.c_uint64(nq),
                                     C.c_uint64(k), C.c_uint64(nprobes), *margs, _p(oi, C.c_uint64),
                                     _p(od, C.c_float), _p(oc, C.c_uint32), C.c_int(nthreads))
        return oi, od, oc
    lib().lo_ivfpq_search(_p(centroids, C.c_float), C.c_uint64(K), C.c_uint64(d),
                          C.c_int(METRIC[metric]), _p(codebook, C.c_float), C.c_uint64(M),
                          C.c_int(nbits), _p(po, C.c_uint64), _p(codes, C.c_uint8),
                          _p(rid, C.c_uint64), _p(queries, C.c_float), C.c_uint64(nq),
                          C.c_uint64(k), C.c_uint64(nprobes), _p(oi, C.c_uint64),
                          _p(od, C.c_float), _p(oc, C.c_uint32), C.c_int(nthreads))
    return oi, od, oc


def sum_4bit_dist_table(n, code_len, codes, dist_table):
    """sum_4bit_dist_table_scalar (lance-linalg/src/simd/dist_table.rs:62-91) -> u16[n]."""
    codes = np.ascontiguousarray(codes, dtype=np.uint8)
    dist_table = np.ascontiguousarray(dist_table, dtype=np.uint8)
    out = np.zeros(n, np.uint16)
    lib().lo_sum_4bit_dist_table(C.c_uint64(n), C.c_uint64(code_len), _p(codes, C.c_uint8),
                                 _p(dist_table, C.c_uint8), _p(out, C.c_uint16))
    return out


def pq_scan_4bit(lut, codes_t, n, k_hint, metric="l2"):
    """compute_pq_distance_4bit (pq/distance.rs:147-242): lut [M][16] f32, codes_t [M/2][n] packed u8."""
    lut = _f32(lut)
    M = lut.size // 16
    codes_t = np.ascontiguousarray(codes_t, dtype=np.uint8)
    out = np.empty(n, np.float32)
    lib().lo_pq_scan_4bit(_p(lut, C.c_float), C.c_uint64(M), _p(codes_t, C.c_uint8), C.c_uint64(n),
                          C.c_uint64(k_hint), C.c_int(METRIC[metric]), _p(out, C.c_float))
    return out


def brute_force_topk(data, queries, k, metric="l2", nthreads=1):
    data, queries = _f32(data), _f32(queries)
    n, d = data.shape
    nq = queries.shape[0]
    oi = np.empty((nq, k), np.uint64)
    od = np.empty((nq, k), np.float32)
    lib().lo_brute_force_topk(_p(data, C.c_float), C.c_uint64(n), C.c_uint64(d),
                              C.c_int(METRIC[metric]), _p(queries, C.c_float), C.c_uint64(nq),
                              C.c_uint64(k), _p(oi, C.c_uint64), _p(od, C.c_float),
                              C.c_int(nthreads))
    return oi, od


def ivfflat_search(centroids, part_offsets, vectors, row_ids, queries, k, nprobes, metric="l2", nthreads=1,
                   allow=None, block=None, lower=None, upper=None):
    centroids, vectors, queries = _f32(centroids), _f32(vectors), _f32(queries)
    K, d = centroids.shape
    po = np.ascontiguousarray(part_offsets, dtype=np.uint64)
    rid = np.ascontiguousarray(row_ids, dtype=np.uint64)
    nq = queries.shape[0]
    oi = np.empty((nq, k), np.uint64)
    od = np.empty((nq, k), np.float32)
    oc = np.empty(nq, np.uint32)
    if lower is not None or upper is not None:
        keep, margs = _mask_args(allow, block)
        lib().lo_ivfflat_search_ex(_p(centroids, C.c_float), C.c_uint64(K), C.c_uint64(d), C.c_int(METRIC[metric]),
                                   _p(po, C.c_uint64), _p(vectors, C.c_float), _p(rid, C.c_uint64),
                                   _p(queries, C.c_float), C.c_uint64(nq), C.c_uint64(k), C.c_uint64(nprobes),
                                   *margs, C.c_int(lower is not None), C.c_float(lower or 0.0),
                                   C.c_int(upper is not None), C.c_float(upper or 0.0), _p(oi, C.c_uint64),
                                   _p(od, C.c_float), _p(oc, C.c_uint32), C.c_int(nthreads))
        return oi, od, oc
    if allow is not None or block is not None:
        keep, margs = _mask_args(allow, block)
        lib().lo_ivfflat_search_masked(_p(centroids, C.c_float), C.c_uint64(K), C.c_uint64(d), C.c_int(METRIC[metric]),
                                       _p(po, C.c_uint64), _p(vectors, C.c_float), _p(rid, C.c_uint64),
                                       _p(queries, C.c_float), C.c_uint64(nq), C.c_uint64(k), C.c_uint64(nprobes),
                                       *margs, _p(oi, C.c_uint64), _p(od, C.c_float), _p(oc, C.c_uint32),
                                       C.c_int(nthreads))
        return oi, od, oc
    lib().lo_ivfflat_search(_p(centroids, C.c_float), C.c_uint64(K), C.c_uint64(d), C.c_int(METRIC[metric]),
                            _p(po, C.c_uint64), _p(vectors, C.c_float), _p(rid, C.c_uint64),
                            _p(queries, C.c_float), C.c_uint64(nq), C.c_uint64(k), C.c_uint64(nprobes),
                            _p(oi, C.c_uint64), _p(od, C.c_float), _p(oc, C.c_uint32), C.c_int(nthreads))
    return oi, od, oc


def hierarchical_kmeans(data, k, max_iters=50, tolerance=1e-4, balance_factor=0.0, metric="l2", hk=16, seed=0, nthreads=1):
    data = _f32(data)
    n, d = data.shape
    out = np.zeros((k, d), np.float32)
    got = lib().lo_hierarchical_kmeans(_p(data, C.c_float), C.c_uint64(n), C.c_uint64(d), C.c_uint64(k),
                                       C.c_int(max_iters), C.c_double(tolerance), C.c_float(balance_factor),
                                       C.c_int(METRIC[metric]), C.c_uint64(hk), C.c_uint64(seed),
                                       _p(out, C.c_float), C.c_int(nthreads))
    return out, got
