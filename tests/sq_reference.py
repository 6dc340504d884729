"""IVF_SQ restated from the reference for the tests (no product code).

The scalar quantizer is integer and f64 arithmetic plus three f32 roundings, all of which numpy performs exactly as
the reference's Rust does (element-wise IEEE operations, round to nearest even, no contraction):
  - bounds:   ScalarQuantizer::update_bounds (lance-index/src/vector/sq.rs:67-89)
  - encode:   scale_to_u8 (sq.rs:263-277)
  - distance: SQDistCalculator (sq/storage.rs:404-468) with l2_distance_uint_scalar (lance-linalg/src/distance/
              l2.rs:44-49), the u8 dot (dot.rs:152-161) and inverse_scalar_dist (sq.rs:279-287)
The search is FlatIndex::search (flat/index.rs:82-177) through the CPU oracle's restated heap (oracle/binding.py
flat_topk), and the global merge by (_distance, _rowid) (rust/lance/src/dataset/scanner.rs:3450-3466).
"""
import numpy as np

from oracle import binding as ob


def bf16_to_f32(bits):
    """uint16 bfloat16 bit patterns -> their exact f32 values"""
    return (np.asarray(bits, np.uint16).astype(np.uint32) << 16).view(np.float32)


def sq_bounds(values):
    """the fold from (f64::MAX, f64::MIN) with f64::min / f64::max over every element: NaN is ignored"""
    v = np.asarray(values, np.float64).ravel()
    v = v[~np.isnan(v)]
    lo, hi = float(np.finfo(np.float64).max), float(np.finfo(np.float64).min)
    if v.size:
        lo, hi = min(lo, float(v.min())), max(hi, float(v.max()))
    return lo, hi


def sq_encode(values, lower, upper):
    """((v - start) * 255.0 / range) in f64, then `as u8`: truncation toward zero, saturating, NaN -> 0"""
    v = np.asarray(values, np.float64)
    if lower == upper:
        return np.zeros(v.shape, np.uint8)
    rng = np.float64(upper) - np.float64(lower)
    with np.errstate(all="ignore"):
        x = (v - np.float64(lower)) * 255.0 / rng
    out = np.zeros(v.shape, np.uint8)
    ok = ~np.isnan(x)
    out[ok] = np.clip(np.trunc(x[ok]), 0.0, 255.0).astype(np.uint8)
    return out


def sq_distance_all(qcode, codes, lower, upper, metric="l2"):
    """u32 sum over the code bytes (L2 / cosine: squared differences; dot: 1 - products), as f32, rescaled"""
    q = np.asarray(qcode, np.int64).ravel()
    c = np.asarray(codes, np.int64).reshape(-1, q.size)
    if metric == "dot":
        f = np.float32(1.0) - (c * q).sum(axis=1).astype(np.float32)
    else:
        f = ((c - q) ** 2).sum(axis=1).astype(np.float32)
    rf = np.float32(np.float64(upper) - np.float64(lower))
    return (f * (rf * rf)) / np.float32(65025.0)


def _total_key(d):
    b = np.asarray(d, np.float32).view(np.int32).astype(np.int64)
    return np.where(b < 0, b ^ 0x7FFFFFFF, b)


def ivfsq_search(centroids, bounds, part_offsets, codes, row_ids, queries, k, nprobes, metric="l2", allow=None,
                 block=None, lower=None, upper=None):
    """IVFIndex::search over an IVF_SQ index held as CSR-by-partition arrays -> ([nq][k] ids, dists, counts).
    queries: f32 values (f16 / bf16 queries converted exactly first).  allow / block: RowIdMask lists; with a mask
    the partition is visited row by row and unselected rows never reach the heap (flat/index.rs:129-165)."""
    cent = np.ascontiguousarray(centroids, np.float32)
    K = cent.shape[0]
    offs = np.asarray(part_offsets, np.int64)
    codes = np.asarray(codes, np.uint8)
    row_ids = np.asarray(row_ids, np.uint64)
    queries = np.ascontiguousarray(queries, np.float32)
    if metric == "cosine":
        queries = ob.normalize_rows(queries)                      # knn.rs:497-499
    cmetric = "dot" if metric == "dot" else "l2"
    masked = allow is not None or block is not None
    allow_set = None if allow is None else set(np.asarray(allow, np.uint64).tolist())
    block_set = set() if block is None else set(np.asarray(block, np.uint64).tolist())
    nq = queries.shape[0]
    oi = np.full((nq, k), np.iinfo(np.uint64).max, np.uint64)
    od = np.full((nq, k), np.inf, np.float32)
    oc = np.zeros(nq, np.uint32)
    for qi in range(nq):
        q = queries[qi]
        qc = sq_encode(q, *bounds)                                # sq/storage.rs:404-430: codes, not a residual
        pids, _ = ob.find_partitions(cent, q, min(nprobes, K), metric=cmetric)
        cid, cd = [], []
        for p in pids:
            a, b = offs[p], offs[p + 1]
            if a == b:
                continue
            dist = sq_distance_all(qc, codes[a:b], *bounds, metric=metric)
            rid = row_ids[a:b]
            if masked:
                sel = np.array([(allow_set is None or r in allow_set) and r not in block_set for r in rid.tolist()],
                               dtype=bool)
                dist, rid = dist[sel], rid[sel]
            ids, ds = ob.flat_topk(dist, rid, k, lower, upper)
            cid.append(ids)
            cd.append(ds)
        if not cid:
            continue
        ids, ds = np.concatenate(cid), np.concatenate(cd)
        order = np.lexsort((ids, _total_key(ds)))[:k]
        oi[qi, :order.size], od[qi, :order.size], oc[qi] = ids[order], ds[order], order.size
    return oi, od, oc
