"""IVF_HNSW_PQ restated from the reference for the tests (no product code).

The graph engine is hnsw_reference's (RHeap, _greedy, _beam, _prune, _Graph, node_levels); only the distances differ.
ProductQuantizationStorage (lance-index/src/vector/pq/storage.rs:600-1037) gives a PQ graph two of them:
  - D[i][j]: PQDistCalculator::distance (:891-919) of node j on the table of node i's decoded codes
    (dist_calculator_from_id, :675-749).  It scores every candidate of node i's insertion and is what its lists store;
    at search time the same sum runs on the table of the (residual) query.  The table is the oracle's build_lut, the
    IVF_PQ scan's table.  8-bit codes: the m-ascending f32 sum of table[m][code[m]]; 4-bit codes: the byte-ordered
    sum of table[2i][lo] + table[2i+1][hi]; dot subtracts M - 1.  Rust's f32 Sum starts from -0.0, numpy from +0.0:
    the two differ only for a sum of -0.0 terms alone, and no table entry is -0.0 (L2 entries are sums of squares
    from +0.0, dot entries 1 - x).
  - H[u][v]: dist_between (:751-841), distance_type.func() over the two decoded rows: flat_reference's lane rules
    (16 f32 lanes; 32 lanes for 16-bit dot, dot.rs:78-83,133).
The storage's distance type is L2 under cosine (pq/storage.rs:465-468), so cosine is L2 on the normalised rows.
"""
import numpy as np

import flat_reference as fr
from hnsw_reference import MAX_KEY, MIN_KEY, INF_KEY, RHeap, _beam, _graph_of, _greedy, _Graph, _prune, node_levels
from oracle import binding as ob
from sq_reference import _total_key


def _pq_metric(metric):
    return "dot" if metric == "dot" else "l2"


def unpack(codes, nbits):
    """[n][M] code indices of [n][cw] code bytes (4-bit: low nibble = sub-vector 2i, pq.rs:168-173)"""
    codes = np.asarray(codes, np.uint8)
    if nbits == 8:
        return codes.astype(np.int64)
    c = np.empty((codes.shape[0], 2 * codes.shape[1]), np.int64)
    c[:, 0::2] = codes & 0xF
    c[:, 1::2] = codes >> 4
    return c


def decode(codebook, codes, nbits):
    """get_centroids / get_centroids_4bit: the codewords of every row concatenated, [n][d] f32"""
    cb = np.asarray(codebook, np.float32)
    c = unpack(codes, nbits)
    return cb[np.arange(cb.shape[0])[None, :], c].reshape(c.shape[0], cb.shape[0] * cb.shape[2])


def table(codebook, q, nbits, metric):
    """the [M][2^nbits] table of the query q (build_distance_table_l2 / _dot as the oracle's build_lut restates it)"""
    cb = np.asarray(codebook, np.float32)
    return ob.build_lut(cb, np.asarray(q, np.float32), nbits=nbits, metric=_pq_metric(metric)).reshape(cb.shape[0], -1)


def table_distances(tab, codes, nbits, metric):
    """PQDistCalculator::distance of every row of `codes` on the table `tab`"""
    M = tab.shape[0]
    c = unpack(codes, nbits)
    dist = np.zeros(c.shape[0], np.float32)
    if nbits == 8:
        for m in range(M):
            dist = dist + tab[m, c[:, m]]
    else:
        for i in range(M // 2):
            dist = dist + (tab[2 * i, c[:, 2 * i]] + tab[2 * i + 1, c[:, 2 * i + 1]])
    if metric == "dot":
        dist = np.where(dist == dist, dist - np.float32(M - 1), dist).astype(np.float32)
    return dist


def node_matrix(codebook, codes, nbits, metric):
    """D: D[i][j] = node j's distance on node i's table (the distances of node i's insertion)"""
    X = decode(codebook, codes, nbits)
    return np.stack([table_distances(table(codebook, X[i], nbits, metric), codes, nbits, metric)
                     for i in range(X.shape[0])]) if X.shape[0] else np.zeros((0, 0), np.float32)


def between_matrix(codebook, codes, nbits, metric, dtype):
    """H: H[u][v] = dist_between(u, v), the lane rule of the column type on the decoded rows"""
    X = decode(codebook, codes, nbits)
    if X.shape[0] == 0:
        return np.zeros((0, 0), np.float32)
    lanes = 32 if (metric == "dot" and dtype in ("f16", "bf16")) else 16
    return fr._lanes(X, X, lanes, _pq_metric(metric))


def build_partition(D, H, levels, m, max_level, efc):
    """HNSW::index_vectors over one partition: the traversal and the lists on D, the heuristic on H"""
    n = len(levels)
    g = _Graph(levels)
    if n < 2:
        return g
    KD, KH = _total_key(D), _total_key(H)
    for i in range(1, n):
        target = levels[i] - 1
        dq, kq = D[i], KD[i]
        ep, ek = 0, int(kq[0])
        for level in range(max_level - 1, target, -1):
            ep, ek = _greedy(g, dq, kq, level, ep, ek)
        for level in range(target, -1, -1):
            res = _beam(g, kq, level, ep, ek, efc)
            m_max = 2 * m if level == 0 else m
            g.lists[i][level] = _prune([(nid, key, float(dq[nid])) for key, nid in res], m_max, KH)
            ek, ep = res[0]
        for level in range(target + 1):
            m_max = 2 * m if level == 0 else m
            for (eid, ekey, ef_) in g.lists[i][level]:
                other = g.lists[eid][level]
                cutoff = INF_KEY if len(other) < m_max else other[-1][1]
                if ekey < cutoff:
                    g.lists[eid][level] = _prune(other + [(i, ekey, ef_)], m_max, KH)
    return g


def build(codes, part_offsets, codebook, nbits, metric, dtype="f32", m=20, max_level=7, efc=150, seed=0):
    """the graphs of every partition in the device layout: dict as IvfHnswPqIndex.export()["graph"] (unused list
    slots zero)"""
    offs = np.asarray(part_offsets, np.int64)
    codes = np.asarray(codes, np.uint8)
    n = int(offs[-1])
    levels = np.zeros(n, np.uint8)
    c0 = np.zeros(n, np.uint32)
    n0 = np.zeros((n, 2 * m), np.uint32)
    d0 = np.zeros((n, 2 * m), np.float32)
    cu, nu, du = [], [], []
    for p in range(len(offs) - 1):
        a, b = int(offs[p]), int(offs[p + 1])
        lv = node_levels(seed, p, b - a, m, max_level)
        pc = codes[a:b]
        g = build_partition(node_matrix(codebook, pc, nbits, metric), between_matrix(codebook, pc, nbits, metric, dtype),
                            lv, m, max_level, efc)
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


def search(centroids, codebook, nbits, part_offsets, codes, row_ids, graph, queries, k, nprobes, metric="l2", ef=None,
           allow_bits=None, lower=None, upper=None):
    """IVFIndex::search over IVF_HNSW_PQ -> ([nq][k] ids, dists, counts); k is k' (k * refine_factor).
    allow_bits: bool per storage position (the prefilter bitmap), or None."""
    cent = np.ascontiguousarray(centroids, np.float32)
    K = cent.shape[0]
    offs = np.asarray(part_offsets, np.int64)
    codes = np.asarray(codes, np.uint8)
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
        pids, _ = ob.find_partitions(cent, queries[qi], min(nprobes, K), metric=_pq_metric(metric))
        cid, cd = [], []
        for p in pids:
            a, b = int(offs[p]), int(offs[p + 1])
            if a == b:
                continue
            qr = queries[qi] if metric == "dot" else (queries[qi] - cent[p]).astype(np.float32)  # ivf/v2.rs:316-332
            dq = table_distances(table(codebook, qr, nbits, metric), codes[a:b], nbits, metric)
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
