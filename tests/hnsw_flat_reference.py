"""IVF_HNSW_FLAT restated from the reference for the tests (no product code).

The graph engine is hnsw_reference's (RHeap, _greedy, _beam, _prune, node_levels), driven as hnsw_pq_reference drives
it; only the distances differ.  FlatFloatStorage (lance-index/src/vector/flat/storage.rs:31-185,345-410) holds the
stored rows as they are and keeps the index's distance type, cosine included (builder.rs:841, flat/storage.rs:108-158,
353-366), so one matrix serves all three distances:
  - P[u][v]: the IVF_FLAT scan's rule with row u in the query role and row v as the stored row.  It is node u's
    distance to v while u is inserted (dist_calculator_from_id), what u's lists store, and the heuristic's
    dist_between(u, v) with u the candidate (hnsw.rs:82); at search time the (normalised) query takes the query role.
  - L2 and dot: flat_reference's 16-lane rule on the stored values as f32 (u8 columns are stored as f32).
  - cosine: the device's COSINE rule restated bit for bit: 16 f32 FMA lanes for <q, y> and <y, y> (element e to lane
    e % 16), the xor tree (offsets 8, 4, 2, 1), |q| from the same 16 FMA lanes over q, then 1 - xy / |q| / sqrt(yy).
    fmaf is emulated exactly (fma32).  The two norms round separately, so P is not symmetric under cosine.
"""
import numpy as np

import flat_reference as fr
from hnsw_pq_reference import build_partition
from hnsw_reference import MAX_KEY, MIN_KEY, RHeap, _beam, _graph_of, _greedy, node_levels
from oracle import binding as ob
from sq_reference import _total_key


def fma32(a, b, c):
    """fmaf(a, b, c) on f32 arrays, correctly rounded: the f64 product of two f32 values is exact; it is added to c in
    f64 with round-to-odd (the TwoSum error decides: a nonzero error with an even last mantissa bit steps one ulp
    towards it), then rounded to f32.  Round-to-odd at 53 bits followed by one rounding to 24 bits is the correct
    rounding because 53 >= 24 + 2."""
    a, b, c = (np.asarray(v, np.float32).astype(np.float64) for v in (a, b, c))
    p = a * b
    s = p + c
    bv = s - p
    err = (p - (s - bv)) + (c - bv)
    even = (s.view(np.int64) & 1) == 0
    fix = (err != 0) & even & np.isfinite(s)
    s = np.where(fix, np.nextafter(s, np.where(err > 0, np.inf, -np.inf)), s)
    return s.astype(np.float32)


def tree16(parts):
    """the xor-shuffle tree over the last axis (16 lane partials): at offset o lane i adds lane i + o"""
    v = np.array(parts, np.float32, copy=True)
    for off in (8, 4, 2, 1):
        v[..., :off] = v[..., :off] + v[..., off:2 * off]
    return v[..., 0]


def cosine_rule(Q, X):
    """[nq, n]: the COSINE rule with Q [nq, d] in the query role and X [n, d] the stored rows, both f32"""
    Q, X = np.asarray(Q, np.float32), np.asarray(X, np.float32)
    nq, d = Q.shape
    n = X.shape[0]
    xy = np.zeros((nq, n, 16), np.float32)
    yy = np.zeros((n, 16), np.float32)
    qq = np.zeros((nq, 16), np.float32)
    for c in range(0, d, 16):
        w = min(16, d - c)
        q, x = Q[:, c:c + w], X[:, c:c + w]
        xy[:, :, :w] = fma32(q[:, None, :], x[None, :, :], xy[:, :, :w])
        yy[:, :w] = fma32(x, x, yy[:, :w])
        qq[:, :w] = fma32(q, q, qq[:, :w])
    q_norm = np.sqrt(tree16(qq))
    return (np.float32(1.0) - tree16(xy) / q_norm[:, None] / np.sqrt(tree16(yy))[None, :]).astype(np.float32)


def distances(Q, X, metric):
    """[nq, n]: the IVF_FLAT scan's distance of every (query role, row) pair over f32 values"""
    Q, X = np.asarray(Q, np.float32), np.asarray(X, np.float32)
    if Q.shape[0] == 0 or X.shape[0] == 0:
        return np.zeros((Q.shape[0], X.shape[0]), np.float32)
    if metric == "cosine":
        return cosine_rule(Q, X)
    return fr._lanes(Q, X, 16, metric)


def stored_f32(vectors, dt):
    """IVF_FLAT's stored rows (as export()["vectors"] returns them) as f32: bf16 bit patterns widened, u8 columns are
    already stored as f32"""
    return fr._f32(vectors, "bf16" if dt == "bf16" else "f32")


def pair_matrix(X, metric):
    """P[u][v] = distances(X[u], X[v]): u in the query role"""
    return distances(X, X, metric)


def build(vectors, part_offsets, metric, dt="f32", m=20, max_level=7, efc=150, seed=0):
    """the graphs of every partition in the device layout: dict as IvfHnswFlatIndex.export()["graph"] (unused list
    slots zero); vectors as export()["vectors"] returns them"""
    X = stored_f32(vectors, dt)
    offs = np.asarray(part_offsets, np.int64)
    n = int(offs[-1])
    levels = np.zeros(n, np.uint8)
    c0 = np.zeros(n, np.uint32)
    n0 = np.zeros((n, 2 * m), np.uint32)
    d0 = np.zeros((n, 2 * m), np.float32)
    cu, nu, du = [], [], []
    for p in range(len(offs) - 1):
        a, b = int(offs[p]), int(offs[p + 1])
        lv = node_levels(seed, p, b - a, m, max_level)
        P = pair_matrix(X[a:b], metric)
        g = build_partition(P, P, lv, m, max_level, efc)
        for i in range(b - a):
            levels[a + i] = lv[i]
            lst = g.lists[i][0]
            c0[a + i] = len(lst)
            for j, (nid, _, f) in enumerate(lst):
                n0[a + i, j], d0[a + i, j] = nid, f
            for level in range(1, lv[i]):
                row_n, row_d = np.zeros(m, np.uint32), np.zeros(m, np.float32)
                for j, (nid, _, f) in enumerate(g.lists[i][level]):
                    row_n[j], row_d[j] = nid, f
                cu.append(len(g.lists[i][level]))
                nu.append(row_n)
                du.append(row_d)
    return dict(max_level=max_level, m=m, ef_construction=efc, levels=levels, counts0=c0, neighbors0=n0, dists0=d0,
                counts_up=np.asarray(cu, np.uint32), neighbors_up=np.asarray(nu, np.uint32).reshape(-1, m),
                dists_up=np.asarray(du, np.float32).reshape(-1, m))


def search(centroids, part_offsets, vectors, row_ids, graph, queries, k, nprobes, metric="l2", dt="f32", ef=None,
           allow_bits=None, lower=None, upper=None):
    """IVFIndex::search over IVF_HNSW_FLAT -> ([nq][k] ids, dists, counts); k is k' (k * refine_factor).  queries: the
    query values as f32; allow_bits: bool per storage position (the prefilter bitmap), or None."""
    cent = np.ascontiguousarray(centroids, np.float32)
    K = cent.shape[0]
    offs = np.asarray(part_offsets, np.int64)
    X = stored_f32(vectors, dt)
    row_ids = np.asarray(row_ids, np.uint64)
    queries = np.ascontiguousarray(queries, np.float32)
    if metric == "cosine":
        queries = ob.normalize_rows(queries)
    ef = k + k // 2 if ef is None else ef
    lo = MIN_KEY if lower is None else int(_total_key(np.float32(lower)))
    hi = MAX_KEY if upper is None else int(_total_key(np.float32(upper)))
    graphs = {}
    nq = queries.shape[0]
    oi = np.full((nq, k), np.iinfo(np.uint64).max, np.uint64)
    od = np.full((nq, k), np.inf, np.float32)
    oc = np.zeros(nq, np.uint32)
    for qi in range(nq):
        pids, _ = ob.find_partitions(cent, queries[qi], min(nprobes, K), metric="dot" if metric == "dot" else "l2")
        cid, cd = [], []
        for p in pids:
            a, b = int(offs[p]), int(offs[p + 1])
            if a == b:
                continue
            dq = distances(queries[qi:qi + 1], X[a:b], metric)[0]
            kq = _total_key(dq)
            allow = None if allow_bits is None else np.asarray(allow_bits[a:b], bool)
            if allow is not None and int(allow.sum()) < (b - a) * 10 // 100:
                heap = RHeap()
                for j in np.flatnonzero(allow).tolist():
                    key = int(kq[j])
                    if key <= lo or key > hi:
                        continue
                    if len(heap) < k:
                        heap.push(key, j)
                    elif key < heap.k[0]:
                        heap.pop()
                        heap.push(key, j)
                res = heap.into_sorted()
            else:
                if p not in graphs:
                    graphs[p] = _graph_of(graph, a, b)
                g = graphs[p]
                ep, ek = 0, int(kq[0])
                for level in range(graph["max_level"] - 1, -1, -1):
                    ep, ek = _greedy(g, dq, kq, level, ep, ek)
                res = _beam(g, kq, 0, ep, ek, ef, allow, lo, hi)[:k]
            for key, j in res:
                cid.append(row_ids[a + j])
                cd.append(dq[j])
        if not cid:
            continue
        ids, ds = np.asarray(cid, np.uint64), np.asarray(cd, np.float32)
        order = np.lexsort((ids, _total_key(ds)))[:k]
        oi[qi, :order.size], od[qi, :order.size], oc[qi] = ids[order], ds[order], order.size
    return oi, od, oc
