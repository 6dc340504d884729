"""flat_knn restated in numpy (test infrastructure): the plan of a nearest() query without an index, and the unindexed
half of knn_combined (rust/lance/src/dataset/scanner.rs:3336-3411, 2912-3027).

Every row is scored with compute_distance's function for the key's element type (lance-index/src/vector/flat.rs:94-150),
the refine plan's rule:
  * f32 L2 / dot, f16 L2, bf16 L2 / dot: 16 f32 lanes (l2.rs:57-91, dot.rs:30-58): the d % 16 tail summed first,
    lane accumulators over the full chunks, folded 0..15; the reference refuses bf16 keys here, so bf16 takes the
    product's rule, the 16-lane f32 loop over the converted values;
  * f16 dot: dot_scalar::<f16, f32, 32> (dot.rs:133): the same with 32 lanes;
  * u8 L2 / dot: the exact u32 sum (wrapping), converted to f32 once (l2.rs:44-49, dot.rs:152-161).
numpy rounds every f32 operation on its own (no contraction), so these are the oracle's per-row functions
(`oracle/binding.py`: l2, dot, l2_f16, dot_f16, l2_bf16, l2_u8, dot_u8) vectorised over queries and rows;
tests/test_flat_search.py pins them to those functions.  Then the rows whose allow bit is clear are dropped,
`_distance >= lower AND _distance < upper` is applied (a NaN fails both), and SortExec(_distance, _rowid).fetch(k)
orders by the f32 total order, ties by row id."""
import numpy as np

BLOCK = 1 << 22   # f32 elements of one block of partial sums


def _f32(a, dt):
    a = np.asarray(a)
    if dt == "bf16":
        return (a.astype(np.uint32) << 16).view(np.float32)
    return a.astype(np.float32)


def _lanes(Q, X, lanes, metric):
    """[nq, n] distances of the lane rule; Q [nq, d], X [n, d] f32"""
    nq, d = Q.shape
    n = X.shape[0]
    full = d // lanes * lanes

    def term(a, b):
        return (a - b) * (a - b) if metric == "l2" else a * b

    out = np.empty((nq, n), np.float32)
    step = max(1, BLOCK // max(1, n * lanes))
    for q0 in range(0, nq, step):
        q = Q[q0:q0 + step]
        s = np.zeros((len(q), n), np.float32)
        for i in range(full, d):
            s = s + term(q[:, i, None], X[None, :, i])
        acc = np.zeros((len(q), n, lanes), np.float32)
        for c in range(0, full, lanes):
            acc = acc + term(q[:, None, c:c + lanes], X[None, :, c:c + lanes])
        t = np.zeros((len(q), n), np.float32)
        for lane in range(lanes):
            t = t + acc[:, :, lane]
        out[q0:q0 + step] = s + t
    return out if metric == "l2" else (np.float32(1.0) - out).astype(np.float32)


def _u8(Q, X, metric):
    """[nq, n] u8 distances: the int64 sum mod 2^32 is the wrapping u32 sum; through f64 (exact) to one f32 rounding"""
    Q, X = np.asarray(Q, np.int64), np.asarray(X, np.int64)
    nq, d = Q.shape
    n = X.shape[0]
    out = np.empty((nq, n), np.float32)
    step = max(1, BLOCK // max(1, n * d))
    for q0 in range(0, nq, step):
        q = Q[q0:q0 + step]
        if metric == "l2":
            s = ((q[:, None, :] - X[None]) ** 2).sum(-1)
        else:
            s = (q[:, None, :] * X[None]).sum(-1)
        out[q0:q0 + step] = (s & 0xFFFFFFFF).astype(np.float64).astype(np.float32)
    return out if metric == "l2" else (np.float32(1.0) - out).astype(np.float32)


def distances(queries, vectors, metric, dt):
    """[nq, n]: compute_distance's value for every (query, row) pair, L2 or dot"""
    if metric not in ("l2", "dot"):
        raise ValueError("the restatement covers L2 and dot; cosine is checked against f64")
    if dt == "u8":
        return _u8(queries, vectors, metric)
    lanes = 32 if (dt == "f16" and metric == "dot") else 16
    return _lanes(_f32(queries, dt), _f32(vectors, dt), lanes, metric)


def total_order_key(d):
    """f32::total_cmp as an int64 key"""
    b = np.ascontiguousarray(d, np.float32).view(np.int32).astype(np.int64)
    return np.where(b < 0, b ^ 0x7FFFFFFF, b)


def flat_search(vectors, queries, k, metric="l2", dtype="f32", row_ids=None, allow=None, lower=None, upper=None):
    """(ids [nq][k], dists [nq][k], counts [nq]); unused slots (2**64 - 1, +inf).  allow: uint64 words, bit i = row i."""
    vectors, queries = np.asarray(vectors), np.asarray(queries)
    n, nq = vectors.shape[0], queries.shape[0]
    rid = np.arange(n, dtype=np.uint64) if row_ids is None else np.asarray(row_ids, np.uint64)
    ok = np.ones(n, bool)
    if allow is not None:
        bits = np.unpackbits(np.asarray(allow, np.uint64).view(np.uint8), bitorder="little")
        ok = bits[:n].astype(bool)
    ids = np.full((nq, k), ~np.uint64(0), np.uint64)
    dists = np.full((nq, k), np.inf, np.float32)
    counts = np.zeros(nq, np.uint32)
    if n == 0:
        return ids, dists, counts
    D = distances(queries, vectors, metric, dtype)
    for i in range(nq):
        keep = ok.copy()
        with np.errstate(invalid="ignore"):
            if lower is not None:
                keep &= D[i] >= np.float32(lower)
            if upper is not None:
                keep &= D[i] < np.float32(upper)
        di, ri = D[i][keep], rid[keep]
        order = np.lexsort((ri, total_order_key(di)))[:k]
        ids[i, :len(order)], dists[i, :len(order)], counts[i] = ri[order], di[order], len(order)
    return ids, dists, counts
