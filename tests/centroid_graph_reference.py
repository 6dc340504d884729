"""The reference's SimpleIndex restated for the tests (no product code): the HNSW graph over the IVF centroids and the
row assignment through it (lance-index/src/vector/utils.rs:26-108, ivf/transform.rs:48-68,112-124).

  - mode:    may_train_index (utils.rs:67-91): "exact" never, "auto" when k * d >= 1 000 000, "hnsw" always; only an
             f32 model has a graph (u8 columns have f32 models, f16 / bf16 models never do)
  - graph:   HNSW::index_vectors over FlatFloatStorage of the centroids with max_level 7, m 12, ef_construction 15:
             hnsw_flat_reference's graph (serial) or hnsw_batch_reference's (insert_batch >= 2) of ONE partition
             holding the k centroids, levels from the draw of (seed, partition 0, node i)
  - search:  search_basic (hnsw/builder.rs:164-235) with k = 1, ef = 15, no bounds: entry node 0, greedy_search at
             every level from max_level - 1 down to 0, beam_search at level 0 (results kept only when
             f32::MIN <= dist < f32::MAX, graph.rs:290-291), the first of into_sorted_vec.  Distances are the f32
             16-lane rule (flat_reference._lanes); every NaN takes one positive bit pattern, as the device's arithmetic
             produces, so that the total-order keys agree.
  - rows:    a row with a non-finite element (KeepFiniteVectors drops it) and a row whose search keeps no result
             (the reference's res[0] panics there) are part 0, dist NaN, valid False.
"""
import numpy as np

import flat_reference as fr
import hnsw_batch_reference as hb
from hnsw_reference import MAX_KEY, MIN_KEY, _beam, _graph_of, _greedy
from sq_reference import _total_key

MAX_LEVEL, M, EFC, EF = 7, 12, 15, 15


def uses_graph(k, d, dtype, mode):
    """may_train_index's decision for a k x d model over a column of dtype "f32", "f16", "bf16" or "u8" """
    if mode == "exact" or (mode == "auto" and k * d < 1_000_000):
        return False
    return dtype in ("f32", "u8")


def build(centroids, metric, seed=0, batch=1):
    """the graph as PartitionIndex.export() returns it"""
    X = np.ascontiguousarray(centroids, np.float32)
    return hb.build_flat(X, [0, X.shape[0]], metric, "f32", m=M, max_level=MAX_LEVEL, efc=EFC, seed=seed,
                         batch=max(batch, 1))


def distances(rows, centroids, metric):
    """[n, k] f32 16-lane distances, NaN canonical"""
    D = fr._lanes(np.asarray(rows, np.float32), np.asarray(centroids, np.float32), 16, metric)
    return np.where(np.isnan(D), np.float32(np.nan), D).astype(np.float32)


def assign(graph, centroids, rows, metric):
    """SimpleIndex::search of every row -> (part u32[n], dist f32[n], valid bool[n])"""
    X = np.ascontiguousarray(centroids, np.float32)
    R = np.ascontiguousarray(rows, np.float32)
    n = R.shape[0]
    part = np.zeros(n, np.uint32)
    dist = np.full(n, np.nan, np.float32)
    valid = np.zeros(n, bool)
    g = _graph_of(graph, 0, X.shape[0])
    live = np.flatnonzero(np.isfinite(R).all(axis=1))
    for b0 in range(0, live.size, 256):
        blk = live[b0:b0 + 256]
        D = distances(R[blk], X, metric)
        for t, i in enumerate(blk.tolist()):
            dq = D[t]
            kq = _total_key(dq)
            ep, ek = 0, int(kq[0])
            for level in range(graph["max_level"] - 1, -1, -1):
                ep, ek = _greedy(g, dq, kq, level, ep, ek)
            res = _beam(g, kq, 0, ep, ek, EF, None, MIN_KEY, MAX_KEY)
            if res:
                j = res[0][1]
                part[i], dist[i], valid[i] = j, dq[j], True
    return part, dist, valid
