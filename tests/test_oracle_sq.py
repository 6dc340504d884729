"""CPU checks of the IVF_SQ restatement (tests/sq_reference.py) against the reference's own SQ tests."""
import numpy as np

from oracle import binding as ob
from sq_reference import ivfsq_search, sq_bounds, sq_distance_all, sq_encode


def test_sq8_literals_of_the_reference():
    # test_f16_sq8 / test_f32_sq8 / test_f64_sq8 (sq.rs:296-370): 0..16 -> bounds (0, 15), codes i * 17
    for dt in (np.float16, np.float32, np.float64):
        v = np.arange(16).astype(dt)
        lo, hi = sq_bounds(v)
        assert (lo, hi) == (0.0, 15.0)
        assert np.array_equal(sq_encode(v, lo, hi), (np.arange(16) * 17).astype(np.uint8))
    # test_scale_to_u8_with_nan (sq.rs:372-389)
    assert sq_encode(np.array([0.0, 1.0, 2.0, 3.0, np.nan]), 0.0, 3.0).tolist() == [0, 85, 170, 255, 0]


def test_bounds_fold_and_encode_edges():
    assert sq_bounds([np.nan, np.nan]) == (np.finfo(np.float64).max, np.finfo(np.float64).min)
    assert sq_bounds([np.inf, 1.0]) == (1.0, np.inf)        # f64::MAX.min(inf) is f64::MAX
    assert sq_bounds([-np.inf, 1.0]) == (-np.inf, 1.0)
    assert sq_encode(np.array([-5.0, 0.2, 9.0, np.inf, -np.inf]), 0.0, 1.0).tolist() == [0, 51, 255, 255, 0]
    assert sq_encode(np.array([3.0, np.nan, -1.0]), 2.0, 2.0).tolist() == [0, 0, 0]
    # u32 sums: 512 dimensions at opposite ends round above 2^24 as f32 (s as f32)
    d = 512
    f = sq_distance_all(np.zeros(d, np.uint8), np.full((1, d), 255, np.uint8), 0.0, 255.0)[0]
    assert f == np.float32(d * 255 * 255) * np.float32(65025.0) / np.float32(65025.0)


def _oracle_sq_recall(metric, seed):
    """test_build_ivf_sq (ivf/v2.rs:1403-1421) through the restatement: 512 x 32 uniform [0, 1) rows, nlist 4,
    query = row 0, k = 100, nprobes = nlist, recall against brute force."""
    rng = np.random.default_rng(seed)
    n, d, nlist, k = 512, 32, 4, 100
    data = rng.random((n, d), dtype=np.float32)
    stored = ob.normalize_rows(data) if metric == "cosine" else data
    part_metric = "dot" if metric == "dot" else "l2"
    cent, _, _ = ob.kmeans_train(stored, nlist, max_iters=50, metric=part_metric, seed=seed,
                                 balance_factor=float(np.float32(1.0) / np.float32(n)))
    part, _, valid = ob.compute_membership(cent, stored, metric=part_metric)
    assert valid.all()
    order = np.argsort(part, kind="stable")
    offs = np.concatenate([[0], np.cumsum(np.bincount(part, minlength=nlist))]).astype(np.uint64)
    bounds = sq_bounds(stored)                       # every row is in the 65 536-row SQ sample
    codes = sq_encode(stored[order], *bounds)
    q = data[:1]
    gt, _ = ob.brute_force_topk(data, q, k, metric=metric)
    ids, _, cnt = ivfsq_search(cent, bounds, offs, codes, order.astype(np.uint64), q, k, nlist, metric=metric)
    assert int(cnt[0]) == k
    return len(set(ids[0].tolist()) & set(gt[0].tolist())) / k


def test_reference_recall_floors_ivf_sq():
    # test_build_ivf_sq (v2.rs:1403-1421): >= 0.85 / 0.85 / 0.75
    for metric, floor in (("l2", 0.85), ("cosine", 0.85), ("dot", 0.75)):
        for seed in (1, 2):
            r = _oracle_sq_recall(metric, seed)
            assert r >= floor, (metric, seed, r)
