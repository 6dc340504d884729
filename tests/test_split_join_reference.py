"""tests/split_join_reference.py on the reference's own split and join scenarios (rust/lance/src/index/vector/ivf/v2.rs:
2223-2470) and on constructed rows, with the oracle's distances.  No GPU."""
import numpy as np

import split_join_reference as sj
from oracle import binding as ob

DIM = 16


def test_choice_rules_thresholds_and_ties():
    t = sj.TARGET["flat"]
    assert sj.should_split([16384, 100], t) is None                  # not strictly above 4 x 4096
    assert sj.should_split([16385, 16386, 16386], t) == 1            # the largest, the first of equal sizes
    assert sj.should_join([1024, 5000], t) is None                   # not strictly below 25% of 4096
    assert sj.should_join([1023, 7, 7], t) == 1
    assert sj.should_join([0], t) is None                            # one partition always stays
    assert sj.TARGET["pq"] == sj.TARGET["sq"] == sj.TARGET["rq"] == 8192 and sj.TARGET["hnsw_pq"] == 1 << 20


def test_candidate_cut_and_ties():
    # K <= 65: every other centroid; equal distances by id
    assert sj.select_reassign_candidates([0.0, 1.0, 1.0, 0.5], 0) == [3, 1, 2]
    # K = 100: min(65, K) ranked, `part` dropped, 64 kept
    dists = np.arange(100, dtype=np.float32)[::-1].copy()
    c = sj.select_reassign_candidates(dists, 99)
    assert len(c) == 64 and c[0] == 98 and c[-1] == 35
    c = sj.select_reassign_candidates(dists, 0)                      # part outside the first 65: 64 of them kept
    assert len(c) == 64 and c[0] == 99 and 0 not in c


def test_decision_ties():
    # d1 == d2 -> c1; d0 == min(d1, d2) of a candidate row -> stays; a candidate minimum equal to d1 -> the candidate;
    # equal candidate distances -> the first
    assert sj.assign_vectors([2.0], [1.0], [1.0], 4, 9, True)[0] == 4
    assert sj.assign_vectors([1.0], [1.0], [3.0], 4, 9, False)[0] == sj.STAYS
    assert sj.assign_vectors([1.0], [1.0], [3.0], 4, 9, True, lambda i: [5.0, 1.0, 1.0], [7, 2, 3])[0] == 2
    assert sj.assign_vectors([0.5], [1.0], [3.0], 4, 9, True, lambda i: [1.5], [7])[0] == 4
    assert sj.assign_vectors([np.nan], [2.0], [1.0], 4, 9, True)[0] == 9   # NaN follows the comparisons
    assert sj.join_destinations([[3.0, 2.0, 2.0]], [0, 5, 6], 4).tolist() == [4]


def _l2(a, b):
    return ob.l2(np.asarray(a, np.float32), np.asarray(b, np.float32))


def _layout(k_new, old_part, old_ids, raw_ids, dest, dropped_part=None, shift=None):
    """(rows per new partition, every row id of the new index): old rows not moved keep their partition (shifted by
    `shift` after a join), the moved rows go to dest, the partition `dropped_part` keeps none of its old rows"""
    moved = dest != sj.STAYS
    gone = np.isin(old_ids, raw_ids[moved])
    if dropped_part is not None:
        gone |= old_part == dropped_part
    keep_part = old_part[~gone] if shift is None else shift(old_part[~gone])
    parts = np.concatenate([keep_part, dest[moved]]).astype(np.int64)
    return np.bincount(parts, minlength=k_new), np.concatenate([old_ids[~gone], raw_ids[moved]])


def test_partition_split_on_append():
    """ivf/v2.rs:2223-2298: IVF_PQ with 2 partitions over two clusters of 2048 rows (e0, e1; DIM 32), 50 000 rows
    identical to e0 appended, optimize -> 3 partitions"""
    dim, stored, appended = 32, 2048, 50_000
    e0, e1 = np.eye(dim, dtype=np.float32)[:2]
    cent = np.stack([e0, e1])                        # the IVF model two tight clusters train
    ids = np.arange(2 * stored + appended, dtype=np.uint64)
    rows = np.concatenate([np.repeat(e0[None], stored, 0), np.repeat(e1[None], stored, 0),
                           np.repeat(e0[None], appended, 0)])
    part_of, _, _ = ob.compute_membership(cent, rows)   # the appended rows transform into partition 0
    sizes = np.bincount(part_of, minlength=2)
    part = sj.should_split(sizes.tolist(), sj.TARGET["pq"])
    assert sizes.tolist() == [stored + appended, stored] and part == 0
    # split_partition_impl: k = 2 on the first 512 of the partition's raw rows (ascending ids)
    own = np.flatnonzero(part_of == part)
    c12, _, _ = ob.kmeans_train(rows[own[:512]], 2, max_iters=50, seed=0)
    cand = np.flatnonzero(part_of == 1)
    cands, dest = sj.split_decisions(_l2, cent, part, c12[0], c12[1], rows[own], rows[cand], part_of[cand])
    assert cands.tolist() == [1]
    new_cent = np.concatenate([cent, c12[1:2]])
    new_cent[part] = c12[0]
    counts, placed = _layout(len(new_cent), part_of, ids, ids[np.concatenate([own, cand])], dest, dropped_part=part)
    assert len(new_cent) == 3 and counts.sum() == len(ids)            # 2 -> 3 partitions, no row lost
    assert np.array_equal(np.sort(placed), ids)                      # every row exactly once
    assert (dest[len(own):] == sj.STAYS).all()                       # the e1 rows stay where they are
    assert counts[1] == stored and counts[0] + counts[2] == stored + appended


def test_join_partition_on_delete():
    """ivf/v2.rs:2301-2470: 100 / 3000 / 3000 rows around centroids 0, 10, 20 on the first axis; all but one row of
    partition 0 deleted and compacted away; optimize -> 2 partitions, the kept row in the old partition 1"""
    sizes = [100, 3000, 3000]
    cent = np.zeros((3, DIM), np.float32)
    cent[:, 0] = [0.0, 10.0, 20.0]
    rows, rid = [], 0
    for c, n in enumerate(sizes):
        for _ in range(n):
            rid += 1
            v = np.full(DIM, (rid % 50) * 0.01, np.float32)
            v[0] = c * 10.0 + (rid % 100) * 0.005
            rows.append(v)
    rows = np.array(rows)
    ids = np.arange(len(rows), dtype=np.uint64)
    part_of, _, _ = ob.compute_membership(cent, rows)
    p0 = np.flatnonzero(part_of == 0)
    assert len(p0) == 100
    mapping = {int(i): None for i in ids[p0[1:]]}                    # the compaction's remap: deleted rows -> None
    left = [int(sum(1 for i in ids[part_of == p] if int(i) not in mapping)) for p in range(3)]
    part = sj.should_join(left, sj.TARGET["pq"])
    assert left == [1, 3000, 3000] and part == 0
    kept = p0[:1]
    cands, dest = sj.join_decisions(_l2, cent, part, rows[kept])
    assert cands.tolist() == [1, 2] and dest.tolist() == [0]          # to old partition 1, now 0
    alive = np.array([int(i) not in mapping for i in ids])
    counts, placed = _layout(2, part_of[alive], ids[alive], ids[kept], dest, dropped_part=part,
                             shift=lambda p: np.where(p > part, p - 1, p))
    assert counts.tolist() == [3001, 3000]                           # 3 -> 2 partitions
    assert np.array_equal(np.sort(placed), ids[alive])


def test_constructed_rows_land_exactly_once():
    rng = np.random.default_rng(7)
    K, d = 9, 8
    cent = rng.normal(0, 2, (K, d)).astype(np.float32)
    part_of = rng.integers(0, K, 600)
    rows = (cent[part_of] + rng.normal(0, 1.5, (600, d))).astype(np.float32)
    ids = np.arange(600, dtype=np.uint64)
    part = 3
    c1, c2 = cent[part] + 0.7, cent[part] - 0.7
    cands = sj.select_reassign_candidates([_l2(cent[part], c) for c in cent], part)
    split_rows = rows[part_of == part]
    order = np.concatenate([np.flatnonzero(part_of == q) for q in cands])
    got_cands, dest = sj.split_decisions(_l2, cent, part, c1, c2, split_rows, rows[order], part_of[order])
    assert got_cands.tolist() == cands
    raw_ids = np.concatenate([ids[part_of == part], ids[order]])
    moved = dest != sj.STAYS
    assert moved[:len(split_rows)].all()                              # the split partition keeps no row of its own
    kept_old = ids[(part_of != part) & ~np.isin(ids, raw_ids[moved])]
    placed = np.concatenate([kept_old, raw_ids[moved]])
    assert np.array_equal(np.sort(placed), ids)
    assert set(dest[moved].tolist()) <= set(cands) | {part, K}
