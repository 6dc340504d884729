"""IVF_HNSW_SQ restated from the reference for the tests (no product code).

Every distance is the SQ distance of sq_reference (query-to-row and row-to-row, sq/storage.rs:387-444,
storage.rs:102-105), precomputed per partition as an f32 matrix; comparisons use f32::total_cmp order keys where the
reference compares OrderedFloat (the heuristic's sort included), and plain f32 `<` where it compares f32
(greedy_search).
  - heaps:   Rust's BinaryHeap (push = sift_up; pop = swap with the last, sift_down_to_bottom, sift_up;
             into_sorted_vec = the heap sort with sift_down_range), on (key, node) with the key alone compared
  - build:   HNSW::index_vectors (hnsw/builder.rs:742-775) with the nodes inserted 1 .. n - 1 in order, insert
             (:396-463), prune (:491-507), select_neighbors_heuristic (hnsw.rs:60-88) with a stable sort,
             GraphBuilderNode::cutoff (graph/builder.rs:50-57), beam_search / greedy_search (graph.rs:275-409)
  - levels:  node 0 max_level levels; node i >= 1: 1 + #{l in 1 .. max_level - 1 : u < 2^32 // m^l}, u the
             splitmix64 draw keyed by (seed, partition, node)
  - search:  HNSW::search (builder.rs:678-739): the flat branch below 10 % allowed rows, search_inner otherwise
"""
import numpy as np

from oracle import binding as ob
from sq_reference import _total_key, sq_distance_all, sq_encode

MASK64 = (1 << 64) - 1
INF_KEY = int(_total_key(np.float32(np.inf)))
MIN_KEY = int(_total_key(np.float32(np.finfo(np.float32).min)))
MAX_KEY = int(_total_key(np.float32(np.finfo(np.float32).max)))


def thresholds(m, max_level):
    return [(1 << 32) // (m ** l) for l in range(max_level)]


def level_draw(seed, p, i):
    x = (seed + (((p << 32) | i) * 0x9E3779B97F4A7C15)) & MASK64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & MASK64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & MASK64
    x ^= x >> 31
    return x >> 32


def node_levels(seed, p, n, m, max_level):
    thr = thresholds(m, max_level)
    lv = [max_level] * min(n, 1)
    for i in range(1, n):
        u = level_draw(seed, p, i)
        lv.append(1 + sum(1 for l in range(1, max_level) if u < thr[l]))
    return lv


class RHeap:
    """std::collections::BinaryHeap (a max-heap) over (key, value), the key alone compared"""

    def __init__(self):
        self.k, self.v = [], []

    def __len__(self):
        return len(self.k)

    def _sift_up(self, start, pos):
        k, v = self.k, self.v
        ek, ev = k[pos], v[pos]
        while pos > start:
            parent = (pos - 1) // 2
            if ek <= k[parent]:
                break
            k[pos], v[pos] = k[parent], v[parent]
            pos = parent
        k[pos], v[pos] = ek, ev

    def push(self, key, val):
        self.k.append(key)
        self.v.append(val)
        self._sift_up(0, len(self.k) - 1)

    def pop(self):
        k, v = self.k, self.v
        key, val = k.pop(), v.pop()
        if k:
            key, k[0] = k[0], key
            val, v[0] = v[0], val
            end, pos = len(k), 0
            ek, ev = k[0], v[0]
            child = 1
            while child <= end - 2:
                if k[child] <= k[child + 1]:
                    child += 1
                k[pos], v[pos] = k[child], v[child]
                pos, child = child, 2 * child + 1
            if child == end - 1:
                k[pos], v[pos] = k[child], v[child]
                pos = child
            k[pos], v[pos] = ek, ev
            self._sift_up(0, pos)
        return key, val

    def into_sorted(self):
        k, v = self.k, self.v
        end = len(k)
        while end > 1:
            end -= 1
            k[0], k[end] = k[end], k[0]
            v[0], v[end] = v[end], v[0]
            pos, child = 0, 1
            ek, ev = k[0], v[0]
            placed = False
            while child <= end - 2:
                if k[child] <= k[child + 1]:
                    child += 1
                if ek >= k[child]:
                    placed = True
                    break
                k[pos], v[pos] = k[child], v[child]
                pos, child = child, 2 * child + 1
            if not placed and child == end - 1 and ek < k[child]:
                k[pos], v[pos] = k[child], v[child]
                pos = child
            k[pos], v[pos] = ek, ev
        return list(zip(k, v))


def pair_distances(codes, bounds, metric):
    """[n][n] f32 SQ distances between the code rows (cosine: L2 on the codes)"""
    c = np.asarray(codes, np.int64)
    if metric == "dot":
        f = np.float32(1.0) - (c @ c.T).astype(np.float32)
    else:
        sq = (c * c).sum(axis=1)
        f = (sq[:, None] + sq[None, :] - 2 * (c @ c.T)).astype(np.float32)
    rf = np.float32(np.float64(bounds[1]) - np.float64(bounds[0]))
    return (f * (rf * rf)) / np.float32(65025.0)


class _Graph:
    def __init__(self, levels):
        self.levels = levels
        self.lists = [[[] for _ in range(L)] for L in levels]   # entries (node, key, f32 distance)


def _greedy(g, dq, kq, level, cur, ckey):
    cf = float(dq[cur])
    while True:
        nxt = None
        for (nid, _, _) in g.lists[cur][level]:
            f = float(dq[nid])
            if f < cf:
                cf, ckey, nxt = f, int(kq[nid]), nid
        if nxt is None:
            return cur, ckey
        cur = nxt


def _beam(g, kq, level, ep, ek, ef, allow=None, lo=MIN_KEY, hi=MAX_KEY):
    visited = {ep}
    cand, res = RHeap(), RHeap()
    cand.push(-ek, ep)
    if (allow is None or allow[ep]) and lo <= ek < hi:
        res.push(ek, ep)
    while len(cand):
        ck, cur = cand.pop()
        ck = -ck
        furthest = res.k[0] if len(res) else INF_KEY
        if ck > furthest and len(res) == ef:
            break
        unvisited = [nid for (nid, _, _) in g.lists[cur][level] if nid not in visited]
        for nid in unvisited:
            visited.add(nid)
            key = int(kq[nid])
            if key <= furthest or len(res) < ef:
                if (allow is None or allow[nid]) and lo <= key < hi:
                    if len(res) < ef:
                        res.push(key, nid)
                    elif key < res.k[0]:
                        res.pop()
                        res.push(key, nid)
                cand.push(-key, nid)
    return res.into_sorted()


def _prune(entries, m_max, K):
    if len(entries) <= m_max:
        return list(entries)
    order = sorted(range(len(entries)), key=lambda j: entries[j][1])   # total_cmp order, stable: ties keep their order
    out = []
    for j in order:
        if len(out) >= m_max:
            break
        uid, ukey, _ = entries[j]
        if not out or all(ukey < K[uid, vid] for (vid, _, _) in out):
            out.append(entries[j])
    return out


def build_partition(codes, bounds, metric, levels, m, max_level, efc):
    """HNSW::index_vectors over one partition's codes -> _Graph"""
    n = len(levels)
    g = _Graph(levels)
    if n < 2:
        return g
    D = pair_distances(codes, bounds, metric)
    K = _total_key(D)
    for i in range(1, n):
        target = levels[i] - 1
        dq, kq = D[i], K[i]
        ep, ek = 0, int(kq[0])
        for level in range(max_level - 1, target, -1):
            ep, ek = _greedy(g, dq, kq, level, ep, ek)
        for level in range(target, -1, -1):
            res = _beam(g, kq, level, ep, ek, efc)
            m_max = 2 * m if level == 0 else m
            g.lists[i][level] = _prune([(nid, key, float(dq[nid])) for key, nid in res], m_max, K)
            ek, ep = res[0]
        for level in range(target + 1):
            m_max = 2 * m if level == 0 else m
            for (eid, ekey, ef_) in g.lists[i][level]:
                other = g.lists[eid][level]
                cutoff = INF_KEY if len(other) < m_max else other[-1][1]
                if ekey < cutoff:
                    g.lists[eid][level] = _prune(other + [(i, ekey, ef_)], m_max, K)
    return g


def build(codes, part_offsets, bounds, metric, m=20, max_level=7, efc=150, seed=0):
    """the graphs of every partition in the device layout: dict as IvfHnswSqIndex.export()["graph"] (unused list
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
        g = build_partition(codes[a:b], bounds, metric, lv, m, max_level, efc)
        for i in range(b - a):
            levels[a + i] = lv[i]
            lst = g.lists[i][0]
            c0[a + i] = len(lst)
            for j, (nid, _, f) in enumerate(lst):
                n0[a + i, j], d0[a + i, j] = nid, f
            for level in range(1, lv[i]):
                lst = g.lists[i][level]
                row_n, row_d = np.zeros(m, np.uint32), np.zeros(m, np.float32)
                for j, (nid, _, f) in enumerate(lst):
                    row_n[j], row_d[j] = nid, f
                cu.append(len(lst))
                nu.append(row_n)
                du.append(row_d)
    return dict(max_level=max_level, m=m, ef_construction=efc, levels=levels, counts0=c0, neighbors0=n0, dists0=d0,
                counts_up=np.asarray(cu, np.uint32), neighbors_up=np.asarray(nu, np.uint32).reshape(-1, m),
                dists_up=np.asarray(du, np.float32).reshape(-1, m))


def _graph_of(graph, a, b):
    """the _Graph of rows [a, b) from the device layout"""
    lv = [int(x) for x in graph["levels"][a:b]]
    up = np.concatenate([[0], np.cumsum(np.asarray(graph["levels"], np.int64) - 1)])
    g = _Graph(lv)
    for i in range(b - a):
        r = a + i
        g.lists[i][0] = [(int(graph["neighbors0"][r, j]), None, None) for j in range(int(graph["counts0"][r]))]
        for level in range(1, lv[i]):
            u = int(up[r]) + level - 1
            g.lists[i][level] = [(int(graph["neighbors_up"][u, j]), None, None)
                                 for j in range(int(graph["counts_up"][u]))]
    return g


def search(centroids, bounds, part_offsets, codes, row_ids, graph, queries, k, nprobes, metric="l2", ef=None,
           allow_bits=None, lower=None, upper=None):
    """IVFIndex::search over IVF_HNSW_SQ -> ([nq][k] ids, dists, counts); k is k' (k * refine_factor).
    allow_bits: bool per storage position (the prefilter bitmap), or None."""
    cent = np.ascontiguousarray(centroids, np.float32)
    K = cent.shape[0]
    offs = np.asarray(part_offsets, np.int64)
    codes = np.asarray(codes, np.uint8)
    row_ids = np.asarray(row_ids, np.uint64)
    queries = np.ascontiguousarray(queries, np.float32)
    if metric == "cosine":
        queries = ob.normalize_rows(queries)
    cmetric = "dot" if metric == "dot" else "l2"
    ef = k + k // 2 if ef is None else ef
    lo = MIN_KEY if lower is None else int(_total_key(np.float32(lower)))
    hi = MAX_KEY if upper is None else int(_total_key(np.float32(upper)))
    graphs = {}
    nq = queries.shape[0]
    oi = np.full((nq, k), np.iinfo(np.uint64).max, np.uint64)
    od = np.full((nq, k), np.inf, np.float32)
    oc = np.zeros(nq, np.uint32)
    for qi in range(nq):
        qc = sq_encode(queries[qi], *bounds)
        pids, _ = ob.find_partitions(cent, queries[qi], min(nprobes, K), metric=cmetric)
        cid, cd = [], []
        for p in pids:
            a, b = int(offs[p]), int(offs[p + 1])
            if a == b:
                continue
            dq = sq_distance_all(qc, codes[a:b], *bounds, metric=metric)
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
