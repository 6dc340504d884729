"""The batched HNSW build (insert_batch B, include/lance_b200.h) restated for the tests (no product code).

The engine is hnsw_reference's (_greedy, _beam, _prune, _Graph, node_levels) and the distance matrices are those of
the three kinds' restatements; only the insertion order differs.  A partition of n >= 2 nodes is built in rounds: the
first starts at s = 1, a round starting at s inserts nodes s .. e - 1 with e = min(n, s + min(B, s)), the next starts
at e.  Each round:
  1. every node of the round searches the graph as it stood at s (no list names a node >= s yet, so running the
     round's searches one after the other sees the same graph) and takes its pruned results as its own lists;
  2. the back-links of the round's nodes, i ascending, level 0 .. top, entries in list order, each with the serial
     rule (cutoff at the last entry of a full list, append, prune).
With B = 1 this is the serial build step for step.
"""
import numpy as np

import hnsw_flat_reference as hf
import hnsw_pq_reference as hp
import hnsw_reference as hr
from hnsw_reference import INF_KEY, _beam, _Graph, _greedy, _prune, node_levels
from sq_reference import _total_key


def rounds(n, batch):
    """[(s, e)] of every round of an n-node partition"""
    out, s = [], 1
    while s < n:
        e = min(n, s + min(batch, s))
        out.append((s, e))
        s = e
    return out


def build_partition_batched(D, H, levels, m, max_level, efc, batch):
    """the batched build over one partition: the traversal and the lists on D, the heuristic on H -> _Graph"""
    n = len(levels)
    g = _Graph(levels)
    if n < 2:
        return g
    KD, KH = _total_key(D), _total_key(H)
    for s, e in rounds(n, batch):
        for i in range(s, e):                       # 1. the searches, over the graph as it stood at s
            target = levels[i] - 1
            dq, kq = D[i], KD[i]
            ep, ek = 0, int(kq[0])
            for level in range(max_level - 1, target, -1):
                ep, ek = _greedy(g, dq, kq, level, ep, ek)
            for level in range(target, -1, -1):
                res = _beam(g, kq, level, ep, ek, efc)
                assert all(nid < s for _, nid in res)
                m_max = 2 * m if level == 0 else m
                g.lists[i][level] = _prune([(nid, key, float(dq[nid])) for key, nid in res], m_max, KH)
                ek, ep = res[0]
        for i in range(s, e):                       # 2. the back-links, i ascending
            for level in range(levels[i]):
                m_max = 2 * m if level == 0 else m
                for (eid, ekey, ef_) in g.lists[i][level]:
                    other = g.lists[eid][level]
                    cutoff = INF_KEY if len(other) < m_max else other[-1][1]
                    if ekey < cutoff:
                        g.lists[eid][level] = _prune(other + [(i, ekey, ef_)], m_max, KH)
    return g


def _layout(part_offsets, m, max_level, efc, seed, graph_of):
    """the device layout of every partition's graph (unused list slots zero); graph_of(p, a, b, levels) -> _Graph"""
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
        g = graph_of(p, a, b, lv)
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


def build_sq(codes, part_offsets, bounds, metric, m=20, max_level=7, efc=150, seed=0, batch=1):
    """as hnsw_reference.build, inserted in rounds of `batch`"""
    codes = np.asarray(codes, np.uint8)

    def graph_of(p, a, b, lv):
        D = hr.pair_distances(codes[a:b], bounds, metric) if b > a else np.zeros((0, 0), np.float32)
        return build_partition_batched(D, D, lv, m, max_level, efc, batch)
    return _layout(part_offsets, m, max_level, efc, seed, graph_of)


def build_pq(codes, part_offsets, codebook, nbits, metric, dtype="f32", m=20, max_level=7, efc=150, seed=0, batch=1):
    """as hnsw_pq_reference.build, inserted in rounds of `batch`"""
    codes = np.asarray(codes, np.uint8)

    def graph_of(p, a, b, lv):
        pc = codes[a:b]
        return build_partition_batched(hp.node_matrix(codebook, pc, nbits, metric),
                                       hp.between_matrix(codebook, pc, nbits, metric, dtype), lv, m, max_level, efc,
                                       batch)
    return _layout(part_offsets, m, max_level, efc, seed, graph_of)


def build_flat(vectors, part_offsets, metric, dt="f32", m=20, max_level=7, efc=150, seed=0, batch=1):
    """as hnsw_flat_reference.build, inserted in rounds of `batch`"""
    X = hf.stored_f32(vectors, dt)

    def graph_of(p, a, b, lv):
        P = hf.pair_matrix(X[a:b], metric)
        return build_partition_batched(P, P, lv, m, max_level, efc, batch)
    return _layout(part_offsets, m, max_level, efc, seed, graph_of)
