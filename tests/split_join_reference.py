"""numpy restatement of the reference's partition split and join decisions (rust/lance/src/index/vector/builder.rs):
should_split (:1152-1176), should_join (:1343-1394), select_reassign_candidates_impl (:1788-1814), assign_vectors
(:1690-1749), reassign_vectors (:1754-1785) and join_partition_impl (:1476-1530).

Distances come from a caller's `dist(from, to)` -- the oracle's pinned per-type functions (oracle/binding.py), never the
device -- in the reference's orientation: d0 / d1 / d2 = dist(centroid, row), candidate distances dist(row, centroid)
and the candidate ranking dist(c0, centroid)."""
import numpy as np

REASSIGN_RANGE = 64
MAX_PARTITION_SIZE_FACTOR = 4
MIN_PARTITION_SIZE_PERCENT = 25
STAYS = 0xFFFFFFFF
# IndexType::target_partition_size (lance-index/src/lib.rs:284-295)
TARGET = {"flat": 4096, "pq": 8192, "sq": 8192, "rq": 8192, "hnsw_sq": 1 << 20, "hnsw_pq": 1 << 20, "hnsw_flat": 1 << 20}


def should_split(sizes, target):
    """the largest partition strictly above MAX_PARTITION_SIZE_FACTOR x target (the first of equal sizes), or None"""
    best, part = 0, None
    for p, n in enumerate(sizes):
        if n > best and n > MAX_PARTITION_SIZE_FACTOR * target:
            best, part = n, p
    return part


def should_join(sizes, target):
    """the smallest partition strictly below MIN_PARTITION_SIZE_PERCENT x target / 100 (the first of equal sizes), or
    None; never with one partition"""
    if len(sizes) <= 1:
        return None
    best, part = None, None
    for p, n in enumerate(sizes):
        if (best is None or n < best) and n < MIN_PARTITION_SIZE_PERCENT * target // 100:
            best, part = n, p
    return part


def _total_key(x):
    """f32::total_cmp as an integer key"""
    b = np.float32(x).view(np.int32).astype(np.int64)
    return b ^ ((b >> 31) & 0x7FFFFFFF)


def select_reassign_candidates(centroid_dists, part):
    """the first min(REASSIGN_RANGE + 1, K) centroids by (distance, id), `part` dropped, min(65, K) - 1 kept"""
    k = len(centroid_dists)
    rng = min(REASSIGN_RANGE + 1, k)
    order = sorted(range(k), key=lambda j: (_total_key(centroid_dists[j]), j))[:rng]
    return [j for j in order if j != part][:max(rng - 1, 0)]


def first_min(dists):
    """position_min_by(total_cmp): the first minimum, or None for no candidates"""
    best = None
    for j, v in enumerate(dists):
        if best is None or _total_key(v) < _total_key(dists[best]):
            best = j
    return best


def reassign_vector(cand_dists, cand_ids, d12, part, k_old):
    """reassign_vectors with Some((d1, d2)): the candidate minimum when it is <= d1 and <= d2, else c1 / c2"""
    d1, d2 = d12
    j = first_min(cand_dists)
    if j is not None and cand_dists[j] <= d1 and cand_dists[j] <= d2:
        return cand_ids[j]
    return part if d1 <= d2 else k_old


def assign_vectors(d0, d1, d2, part, k_old, deleted_original_partition, cand_dists_of_row=None, cand_ids=()):
    """destinations of one partition's rows: the split partition's (deleted_original_partition, cand_dists_of_row(i)
    gives row i's candidate distances) or a candidate partition's (STAYS for a row whose own centroid is nearest)"""
    out = []
    for i in range(len(d0)):
        if d0[i] <= d1[i] and d0[i] <= d2[i]:
            if not deleted_original_partition:
                out.append(STAYS)
                continue
            out.append(reassign_vector(cand_dists_of_row(i), cand_ids, (d1[i], d2[i]), part, k_old))
        else:
            out.append(part if d1[i] <= d2[i] else k_old)
    return np.array(out, np.uint32)


def join_destinations(cand_dists, cand_ids, part):
    """join_partition_impl: each row to its first-minimum candidate, ids above `part` shifted down by one"""
    out = []
    for ds in cand_dists:
        c = cand_ids[first_min(ds)]
        out.append(c if c < part else c - 1)
    return np.array(out, np.uint32)


def split_decisions(dist, centroids, part, c1, c2, rows, cand_rows, cand_parts):
    """every destination of a split: the split partition's rows, then the candidate partitions' rows (grouped in
    candidate order); returns (candidate ids, destinations)"""
    k = len(centroids)
    c0 = centroids[part]
    cands = select_reassign_candidates([dist(c0, c) for c in centroids], part)
    d0 = [dist(c0, r) for r in rows]
    d1 = [dist(c1, r) for r in rows]
    d2 = [dist(c2, r) for r in rows]
    dest = [assign_vectors(d0, d1, d2, part, k, True, lambda i: [dist(rows[i], centroids[c]) for c in cands], cands)]
    for q in cands:
        sel = np.flatnonzero(np.asarray(cand_parts) == q)
        rq = [cand_rows[i] for i in sel]
        dest.append(assign_vectors([dist(centroids[q], r) for r in rq], [dist(c1, r) for r in rq],
                                   [dist(c2, r) for r in rq], part, k, False))
    return np.array(cands, np.uint32), np.concatenate(dest).astype(np.uint32)


def join_decisions(dist, centroids, part, rows):
    """(candidate ids, destinations) of a join of `part`"""
    cands = select_reassign_candidates([dist(centroids[part], c) for c in centroids], part)
    return np.array(cands, np.uint32), join_destinations([[dist(r, centroids[c]) for c in cands] for r in rows], cands,
                                                         part)


# ---- the per-pair distance rules in numpy f32, to show that a case tells rules apart ---------------------------------
# Every operation rounds to f32 (numpy float32 arithmetic, no FMA).  x, y: f32 arrays [..., d] holding the elements'
# exact f32 values; the result is dist(x, y) per leading index.
def _terms(x, y, metric):
    x, y = np.asarray(x, np.float32), np.asarray(y, np.float32)
    if metric == "dot":
        return x * y
    t = x - y
    return t * t


def rule_sum(x, y, metric, lanes=16, tail="first", fold=None):
    """lanes f32 accumulators, lane l owning elements l, l + lanes, ...; tail="first": the d % lanes tail summed
    sequentially first and added last (the reference's dot_scalar / l2 shape), tail="lanes": the tail walked into the
    lanes like any other element; fold: the order the lanes are folded in (default 0 .. lanes - 1).  dot: 1 - sum."""
    t = _terms(x, y, metric)
    d = t.shape[-1]
    n = d // lanes * lanes
    s = np.zeros(t.shape[:-1], np.float32)
    acc = np.zeros(t.shape[:-1] + (lanes,), np.float32)
    for c in range(0, n, lanes):
        acc += t[..., c:c + lanes]
    if tail == "first":
        for e in range(n, d):
            s += t[..., e]
    else:
        for e in range(n, d):
            acc[..., e - n] += t[..., e]
    tot = np.zeros(t.shape[:-1], np.float32)
    for lane in (range(lanes) if fold is None else fold):
        tot += acc[..., lane]
    out = s + tot
    return np.float32(1) - out if metric == "dot" else out


def lanes16(x, y, metric):
    """LANES16: l2 / dot of f32 rows and 16-bit l2 (l2.rs:57-91, dot.rs:30-58 with 16 lanes)"""
    return rule_sum(x, y, metric, 16)


def dot32(x, y, metric="dot"):
    """DOT32: 16-bit dot, dot_scalar::<T, f32, 32> (dot.rs:30-58)"""
    return rule_sum(x, y, metric, 32)


def tail_in_lanes(x, y, metric):
    """wrong: 16 lanes with the tail walked into the lanes"""
    return rule_sum(x, y, metric, 16, tail="lanes")


def dot32_b_first(x, y, metric="dot"):
    """wrong: DOT32 with accumulators 16..31 folded before 0..15"""
    return rule_sum(x, y, metric, 32, fold=list(range(16, 32)) + list(range(16)))


def batch_rule(metric, dt):
    """lb2_distance_batch's rule for l2 / dot: DOT32 for 16-bit dot, LANES16 otherwise"""
    return dot32 if metric == "dot" and dt != "f32" else lanes16


def matrix(rule, metric):
    """D(A, B)[i, j] = rule(A[i], B[j]) (A in the `from` role)"""
    return lambda A, B: rule(np.asarray(A, np.float32)[:, None, :], np.asarray(B, np.float32)[None, :, :], metric)


def decisions(D, centroids, part, rows, c12=None, cand_rows=None, cand_parts=None, Dc=None):
    """split_decisions (c12 = (c1, c2)) or join_decisions over matrix distances D(from_rows, to_rows) -> (candidates,
    destinations); Dc: the distances of the candidate scan, dist(row, candidate centroid) (default D)"""
    Dc = Dc or D
    centroids = np.asarray(centroids, np.float32)
    rows = np.asarray(rows, np.float32)
    k = len(centroids)
    cands = select_reassign_candidates(D(centroids[part:part + 1], centroids)[0], part)
    cid = np.asarray(cands, np.int64)

    def first_min(rs):
        dc = Dc(rs, centroids[cid])
        j = np.argmin(_total_key(dc), axis=1)
        return cid[j], dc[np.arange(len(rs)), j]
    if c12 is None:
        ids, _ = first_min(rows)
        return cands, np.where(ids < part, ids, ids - 1).astype(np.uint32)
    c1, c2 = (np.asarray(c, np.float32) for c in c12)
    d0, d1, d2 = D(np.stack([centroids[part], c1, c2]), rows)
    out = np.where(d1 <= d2, part, k).astype(np.int64)
    want = (d0 <= d1) & (d0 <= d2)
    if len(cands) and want.any():
        ids, best = first_min(rows[want])
        take = (best <= d1[want]) & (best <= d2[want])
        out[want] = np.where(take, ids, out[want])
    dest = [out]
    cand_rows = np.asarray(cand_rows, np.float32).reshape(-1, centroids.shape[1])
    for q in cands:
        rq = cand_rows[np.asarray(cand_parts) == q]
        e0 = D(centroids[q:q + 1], rq)[0]
        e1, e2 = D(np.stack([c1, c2]), rq)
        dest.append(np.where((e0 <= e1) & (e0 <= e2), STAYS, np.where(e1 <= e2, part, k)))
    return cands, np.concatenate(dest).astype(np.uint32)
