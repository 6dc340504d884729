"""Flat KNN over a vector column (`lb2_flat_search`: flat_knn, scanner.rs:3336-3411) and the combined search of an
index with the rows it does not cover (`lb2_index_search_combined`: knn_combined, scanner.rs:2946-3027).

CPU: the numpy restatement of flat_knn (`tests/flat_reference.py`) pinned to the oracle's per-type distance functions,
and against an f64 brute force, its tie rule, bitmap and range.
GPU: ids, distances and counts bit for bit against that restatement for L2 / dot at every element type; cosine within the
f64 bound of test_exact_search_variants; ties that overflow the k-th place (smallest row ids win, not the heap's
choice); host and device columns across staged chunks; and the combined search of all four index kinds against the
(distance, row id) merge of its two halves."""
import ctypes as C

import numpy as np
import pytest

import lance_b200 as lb
from lance_b200 import _lib
import flat_reference as fr
from oracle import binding as ob
from test_exact_search_variants import _bf16_f32, _cosine64, _cosine_bound, _f32, _native

NT = 16
NONE = np.uint64(~np.uint64(0))
SEARCH_SLAB = 32768


def _bitmap(mask):
    """bool per row -> uint64 words, bit i = row i"""
    bits = np.zeros((len(mask) + 63) // 64 * 64, np.uint8)
    bits[:len(mask)] = mask
    return np.packbits(bits, bitorder="little").view(np.uint64)


def _column(rng, n, d, dt, nq, clusters=8):
    """n rows and nq queries near the same cluster centres, in element type dt (u8: integer levels)"""
    if dt == "u8":
        lvl = rng.integers(0, 256, (clusters, d))
        x = np.clip(lvl[rng.integers(0, clusters, n)] + rng.integers(-40, 41, (n, d)), 0, 255).astype(np.uint8)
        q = np.clip(lvl[rng.integers(0, clusters, nq)] + rng.integers(-40, 41, (nq, d)), 0, 255).astype(np.uint8)
        return x, q
    cent = rng.standard_normal((clusters, d)).astype(np.float32) * 2
    x = cent[rng.integers(0, clusters, n)] + rng.standard_normal((n, d)).astype(np.float32)
    q = cent[rng.integers(0, clusters, nq)] + rng.standard_normal((nq, d)).astype(np.float32)
    if d >= 64:  # dot: rows of similar norm keep the products in a modest range
        x *= np.float32(0.25)
        q *= np.float32(0.25)
    return _native(x, dt), _native(q, dt)


def _assert_same(got, want, what):
    gi, gd, gc = got
    wi, wd, wc = want
    assert np.array_equal(gc, wc), (what, np.flatnonzero(gc != wc)[:5])
    for i in range(len(wi)):
        if not (np.array_equal(gi[i], wi[i]) and np.array_equal(gd[i], wd[i], equal_nan=True)):
            r = next(j for j in range(len(wi[i])) if gi[i, j] != wi[i, j] or not
                     (gd[i, j] == wd[i, j] or (np.isnan(gd[i, j]) and np.isnan(wd[i, j]))))
            raise AssertionError(f"{what}: query {i}, rank {r}: got ({gi[i, r]}, {gd[i, r]!r}), "
                                 f"want ({wi[i, r]}, {wd[i, r]!r})")


def _profiled(fn):
    lb.profile.reset()
    lb.profile.enable(True)
    try:
        out = fn()
    finally:
        lb.profile.enable(False)
    return out, lb.profile.dump()


# ---- CPU: the restatement ---------------------------------------------------------------------------------------------
def _f64_dists(x, q, metric):
    x64, q64 = x.astype(np.float64), q.astype(np.float64)
    if metric == "l2":
        return ((q64[:, None, :] - x64[None]) ** 2).sum(-1)
    return 1.0 - q64 @ x64.T


_PER_ROW = {("f32", "l2"): ob.l2, ("f16", "l2"): ob.l2_f16, ("bf16", "l2"): ob.l2_bf16, ("u8", "l2"): ob.l2_u8,
            ("f32", "dot"): ob.dot, ("f16", "dot"): ob.dot_f16, ("u8", "dot"): ob.dot_u8,
            # bf16 dot: the product's 16-lane f32 rule (the reference has no bf16 key in refine)
            ("bf16", "dot"): lambda a, b: ob.dot(_bf16_f32(a), _bf16_f32(b))}


@pytest.mark.parametrize("metric", ["l2", "dot"])
@pytest.mark.parametrize("dt", ["f32", "f16", "bf16", "u8"])
def test_restatement_is_the_oracles_per_row_distance(dt, metric):
    """tests/flat_reference.py's vectorised distances equal the oracle's per-row functions bit for bit"""
    rng = np.random.default_rng(6900 + len(dt) + (metric == "dot"))
    for d in (1, 5, 16, 17, 31, 32, 33, 100, 140, 1040):
        x, q = _column(rng, 30, d, dt, 3)
        got = fr.distances(q, x, metric, dt)
        f = _PER_ROW[dt, metric]
        want = np.array([[f(q[i], x[j]) for j in range(len(x))] for i in range(len(q))], np.float32)
        if metric == "dot":
            want = (np.float32(1.0) - want).astype(np.float32)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (dt, metric, d)
    if dt == "f16" and metric == "dot":   # the restatement tells f16 dot's 32 lanes from 16
        x, q = _column(rng, 300, 128, "f16", 2)
        lanes16 = fr._lanes(q.astype(np.float32), x.astype(np.float32), 16, "dot")
        assert np.sum(fr.distances(q, x, "dot", "f16") != lanes16) > 20


@pytest.mark.parametrize("metric", ["l2", "dot"])
@pytest.mark.parametrize("dt", ["f32", "f16", "bf16", "u8"])
def test_oracle_flat_search_agrees_with_f64_where_the_gap_allows(dt, metric):
    rng = np.random.default_rng(7000 + len(dt) + (metric == "dot"))
    n, d, nq, k = 3000, 40, 12, 20
    x, q = _column(rng, n, d, dt, nq)
    oi, od, oc = fr.flat_search(x, q, k, metric, dt)
    assert np.all(oc == k)
    x32, q32 = _f32(x, dt), _f32(q, dt)
    ex = _f64_dists(x32, q32, metric)
    scale = np.abs(x32.astype(np.float64)).max() * np.abs(q32.astype(np.float64)).max() * d + 1.0
    bound = 4 * (d + 2) * 2.0 ** -24 * (scale if metric == "dot" else ex.max())
    for i in range(nq):
        order = np.argsort(ex[i], kind="stable")
        kth, nxt = ex[i, order[k - 1]], ex[i, order[k]]
        got = set(oi[i].astype(np.int64).tolist())
        if nxt - kth > 2 * bound:   # the f64 top-k set is unambiguous under the f32 rounding bound
            assert got == set(order[:k].tolist()), (dt, metric, i)
        assert np.all(np.abs(od[i].astype(np.float64) - ex[i, oi[i].astype(np.int64)]) <= bound), (dt, metric, i)
        assert all(od[i, j] <= od[i, j + 1] for j in range(k - 1))


def test_oracle_flat_search_ties_go_to_the_smallest_row_ids():
    rng = np.random.default_rng(7100)
    n, d = 500, 16
    x = rng.standard_normal((n, d)).astype(np.float32)
    dup = x[3].copy()
    rows = rng.choice(n, 40, replace=False)
    x[rows] = dup                                             # 40 (+1) rows at distance 0 of the query
    rid = rng.permutation(n * 7)[:n].astype(np.uint64)        # distinct, shuffled
    for k in (1, 5, 41, 60):
        oi, od, oc = fr.flat_search(x, dup[None], k, "l2", row_ids=rid)
        tied = np.sort(rid[np.flatnonzero((x == dup).all(1))])
        m = min(k, len(tied))
        assert np.array_equal(oi[0, :m], tied[:m]) and np.all(od[0, :m] == 0), k


def test_oracle_flat_search_bitmap_and_range():
    rng = np.random.default_rng(7200)
    n, d, nq, k = 1000, 24, 6, 30
    x, q = _column(rng, n, d, "f32", nq)
    allow = rng.random(n) < 0.3
    oi, od, oc = fr.flat_search(x, q, k, "l2", allow=_bitmap(allow))
    for i in range(nq):
        assert np.all(allow[oi[i, :oc[i]].astype(np.int64)])
    full_i, full_d, _ = fr.flat_search(x, q, n, "l2")
    lo, hi = float(np.median(full_d[:, 50])), float(np.median(full_d[:, 200]))
    ri, rd, rc = fr.flat_search(x, q, k, "l2", lower=lo, upper=hi, allow=_bitmap(allow))
    for i in range(nq):
        keep = allow[full_i[i].astype(np.int64)] & (full_d[i] >= np.float32(lo)) & (full_d[i] < np.float32(hi))
        want = full_i[i][keep][:k]
        assert rc[i] == len(want) and np.array_equal(ri[i, :rc[i]], want), i
        assert np.all(ri[i, rc[i]:] == NONE) and np.all(np.isinf(rd[i, rc[i]:]))
    # all clear: nothing returned
    ci, cd, cc = fr.flat_search(x, q, k, "l2", allow=_bitmap(np.zeros(n, bool)))
    assert np.all(cc == 0) and np.all(ci == NONE)


# ---- GPU: flat search against the oracle ---------------------------------------------------------------------------
CASES = [(dt, d) for dt in ("f32", "f16", "bf16", "u8") for d in (1, 36, 128, 140, 1536)]


@pytest.mark.gpu
@pytest.mark.parametrize("metric", ["l2", "dot"])
@pytest.mark.parametrize("dt,d", CASES, ids=[f"{t}-d{d}" for t, d in CASES])
def test_flat_search_matches_oracle_bit_for_bit(dt, d, metric):
    rng = np.random.default_rng(7300 + d + 3 * len(dt) + (metric == "dot"))
    n, nq = (2500, 21) if d < 1536 else (700, 5)
    x, q = _column(rng, n, d, dt, nq)
    bf = dt == "bf16"
    for k in (1, 10, 100, 1024):
        got, prof = _profiled(lambda: lb.flat_search(x, q, k, metric, bf16=bf))
        _assert_same(got, fr.flat_search(x, q, k, metric, dt), (dt, d, metric, k))
        assert prof.get("flat_search:scan", (0,))[0] == 1 and prof.get("flat_search:merge", (0,))[0] >= 1, prof
    # n < k, and shuffled row ids with a bitmap and a range
    got = lb.flat_search(x[:7], q, 10, metric, bf16=bf)
    _assert_same(got, fr.flat_search(x[:7], q, 10, metric, dt), ("n < k", dt, d))
    rid = rng.permutation(5 * n)[:n].astype(np.uint64)
    allow = _bitmap(rng.random(n) < 0.5)
    _, full_d, _ = fr.flat_search(x, q, 200, metric, dt)
    lo, hi = float(np.median(full_d[:, 5])), float(np.median(full_d[:, 150]))
    got = lb.flat_search(x, q, 50, metric, row_ids=rid, allow_bitmap=allow, lower_bound=lo, upper_bound=hi, bf16=bf)
    _assert_same(got, fr.flat_search(x, q, 50, metric, dt, row_ids=rid, allow=allow, lower=lo, upper=hi),
                 ("filtered", dt, d))


@pytest.mark.gpu
@pytest.mark.parametrize("dt,d", [("f32", 128), ("f32", 36), ("f16", 140), ("bf16", 128), ("u8", 36)])
def test_flat_search_cosine_within_the_f64_bound(dt, d):
    rng = np.random.default_rng(7400 + d + len(dt))
    n, nq, k = 3000, 9, 50
    x, q = _column(rng, n, d, dt, nq)
    ids, dists, cnt = lb.flat_search(x, q, k, "cosine", bf16=dt == "bf16")
    x32, q32 = _f32(x, dt), _f32(q, dt)
    assert np.all(cnt == k)
    for i in range(nq):
        got, gd = ids[i].astype(np.int64), dists[i].astype(np.float64)
        assert np.all(np.abs(gd - _cosine64(q32[i], x32[got])) <= _cosine_bound(q32[i], x32[got])), i
        assert all(gd[j] < gd[j + 1] or (gd[j] == gd[j + 1] and got[j] < got[j + 1]) for j in range(k - 1)), i
        ex = _cosine64(q32[i], x32)
        b2 = 2 * float(np.max(_cosine_bound(q32[i], x32)))
        kth = np.sort(ex)[k - 1]
        assert set(np.flatnonzero(ex < kth - b2).tolist()) <= set(got.tolist()), i


@pytest.mark.gpu
@pytest.mark.parametrize("metric", ["l2", "dot"])
def test_flat_search_many_row_ranges_ties_and_nan(metric):
    """n = 60 000 rows split over many CTAs (so more lists per query than one rank merge takes at k = 100 and 1024);
    one row duplicated 300 times under shuffled row ids: the query equal to it ties 301 rows at the best distance,
    and the smallest row ids must win.  Rows holding NaN have NaN distances, which sort after +inf."""
    rng = np.random.default_rng(7500 + (metric == "dot"))
    n, d = 60000, 36
    x, q = _column(rng, n, d, "f32", 6)
    dup = x[11].copy()
    x[rng.choice(n, 300, replace=False)] = dup
    x[5 + rng.choice(n - 5, 50, replace=False), 3] = np.nan
    q[0] = dup
    q[1] = dup
    rid = rng.permutation(n * 3)[:n].astype(np.uint64)
    for k in (1, 10, 100, 1024):
        got = lb.flat_search(x, q, k, metric, row_ids=rid)
        _assert_same(got, fr.flat_search(x, q, k, metric, row_ids=rid), (metric, k))
    # every row tied and shuffled: the k smallest row ids
    same = np.repeat(dup[None], 5000, axis=0)
    rid5 = rng.permutation(10 ** 6)[:5000].astype(np.uint64)
    gi, gd, gc = lb.flat_search(same, dup[None], 100, metric, row_ids=rid5)
    assert np.array_equal(gi[0], np.sort(rid5)[:100]) and gc[0] == 100
    # NaN rows only: returned after everything else, ascending by row id
    nan_rows = np.flatnonzero(np.isnan(x).any(1))
    allow = np.zeros(n, bool)
    allow[nan_rows] = True
    allow[:5] = True
    gi, gd, gc = lb.flat_search(x, q[2:3], 60, metric, row_ids=rid, allow_bitmap=_bitmap(allow))
    assert gc[0] == 55 and np.all(np.isnan(gd[0, 5:55])) and np.all(np.diff(gi[0, 5:55].astype(np.int64)) > 0)
    # an all-clear bitmap: count 0, padded outputs
    gi, gd, gc = lb.flat_search(x, q, 10, metric, allow_bitmap=_bitmap(np.zeros(n, bool)))
    assert np.all(gc == 0) and np.all(gi == NONE) and np.all(np.isposinf(gd))


@pytest.mark.gpu
def test_flat_search_more_queries_than_a_slab():
    rng = np.random.default_rng(7600)
    n, d, nq = 300, 8, SEARCH_SLAB + 77
    x, q = _column(rng, n, d, "f32", nq)
    got = lb.flat_search(x, q, 10, "l2")
    _assert_same(got, fr.flat_search(x, q, 10, "l2"), "slab")


def _pinned(a):
    p = lb.PinnedArray(a.shape, a.dtype)
    p.array[...] = a
    return p


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["f32", "f16", "u8"])
def test_flat_search_host_and_device_columns_across_chunks(dt, monkeypatch):
    """LB2_CHUNK_ROWS = 1000: a pageable or pinned host column of 4321 rows is staged in five chunks, each contributing
    its own lists; a device column is read in place in one launch."""
    rng = np.random.default_rng(7700 + len(dt))
    n, d, nq = 4321, 36, 40
    x, q = _column(rng, n, d, dt, nq)
    want = fr.flat_search(x, q, 30, "l2", dt)
    dev = lb.DeviceArray.from_numpy(x)
    pin = _pinned(x)
    try:
        monkeypatch.setenv("LB2_CHUNK_ROWS", "1000")
        for kind, col, scans in (("numpy", x, 5), ("pinned", pin, 5), ("device", dev, 1)):
            got, prof = _profiled(lambda: lb.flat_search(col, q, 30, "l2"))
            _assert_same(got, want, (dt, kind))
            assert prof.get("flat_search:scan", (0,))[0] == scans, (kind, prof)
            if kind != "device":
                assert prof.get("flat_search:stage_rows", (0,))[0] == 5, (kind, prof)
        monkeypatch.delenv("LB2_CHUNK_ROWS")
        got = lb.flat_search(dev, lb.DeviceArray.from_numpy(q), 30, "l2")
        _assert_same(got, want, (dt, "device queries"))
    finally:
        pin.free()


@pytest.mark.gpu
def test_flat_search_refusals():
    x = np.zeros((10, 8), np.float32)
    with pytest.raises(lb.LanceB200Error) as e:
        lb.flat_search(x, x[:1], 0)
    assert e.value.status == _lib.INVALID_ARG
    with pytest.raises(lb.LanceB200Error) as e:
        lb.flat_search(x, x[:1], 1025)
    assert e.value.status == _lib.UNSUPPORTED
    big = np.zeros((2, 8192), np.float32)
    with pytest.raises(lb.LanceB200Error) as e:
        lb.flat_search(big, big[:1], 1)
    assert e.value.status == _lib.UNSUPPORTED


# ---- GPU: the combined search ---------------------------------------------------------------------------------------
KINDS = ["pq", "flat", "sq", "rq"]


def _build(kind, data, K, metric):
    if kind == "pq":
        p = lb.IvfBuildParams(num_partitions=K, num_sub_vectors=8, max_iters=4, pq_max_iters=4)
        return lb.IvfPqIndex.build(data, metric, p)
    b = {"flat": lb.IvfFlatIndex, "sq": lb.IvfSqIndex, "rq": lb.IvfRqIndex}[kind]
    return b.build(data, metric, num_partitions=K, max_iters=4)


def _merge(a, b, k):
    """the (distance, row id) merge of two result lists per query"""
    ai, ad, ac = a
    bi, bd, bc = b
    nq = len(ac)
    ids, dists, cnt = np.full((nq, k), NONE, np.uint64), np.full((nq, k), np.inf, np.float32), np.zeros(nq, np.uint32)
    for i in range(nq):
        ci = np.concatenate([ai[i, :ac[i]], bi[i, :bc[i]]])
        cd = np.concatenate([ad[i, :ac[i]], bd[i, :bc[i]]])
        key = cd.view(np.int32).astype(np.int64)
        key = np.where(key < 0, key ^ 0x7FFFFFFF, key)
        order = np.lexsort((ci, key))[:k]
        ids[i, :len(order)], dists[i, :len(order)], cnt[i] = ci[order], cd[order], len(order)
    return ids, dists, cnt


def _search_ex(ix, q, k, nprobes, rf, vectors, bm=None):
    ids, dists = ix.search_ex(q, k=k, nprobes=nprobes, refine_factor=rf, vectors=vectors, allow_bitmap=bm)
    return ids, dists, np.sum(ids != NONE, axis=1).astype(np.uint32)


@pytest.mark.gpu
@pytest.mark.parametrize("metric", ["l2", "dot"])
@pytest.mark.parametrize("kind", KINDS)
def test_combined_search_is_the_merge_of_its_halves(kind, metric):
    rng = np.random.default_rng(7800 + KINDS.index(kind) + 10 * (metric == "dot"))
    n_ix, n_new, d, K, k = 6000, 900, 32, 16, 20
    x, q = _column(rng, n_ix + n_new, d, "f32", 14)
    ix = _build(kind, x[:n_ix], K, metric)
    new, new_id = x[n_ix:], np.arange(n_ix, n_ix + n_new, dtype=np.uint64)
    allow_new = _bitmap(rng.random(n_new) < 0.6)
    bm = ix.row_mask(rng.choice(n_ix, 3000, replace=False), None)
    for rf in (0, 3):
        kr = max(1, rf)
        # u->n == 0 is the index search with refine factor max(1, rf), bit for bit
        ci, cd, cc, _ = ix.search_combined(q, k, x, new[:0], new_id[:0], nprobes=4, refine_factor=rf)
        ei, ed, ec = _search_ex(ix, q, k, 4, kr, x)
        _assert_same((ci, cd, cc), (ei, ed, ec), (kind, "empty", rf))
        for allow_ix, allow_u in ((None, None), (bm, allow_new)):
            got, prof = _profiled(lambda: ix.search_combined(q, k, x, new, new_id, nprobes=4, refine_factor=rf,
                                                             allow_bitmap=allow_ix, unindexed_allow_bitmap=allow_u))
            want = _merge(_search_ex(ix, q, k, 4, kr, x, allow_ix),
                          lb.flat_search(new, q, k, metric, row_ids=new_id, allow_bitmap=allow_u), k)
            _assert_same(got[:3], want, (kind, rf, allow_ix is None))
            assert prof.get("search:merge_combined", (0,))[0] == 1 and prof.get("flat_search:scan", (0,))[0] == 1
        # minimum / maximum nprobes
        pi, pd, pc, pn = ix.search_combined(q, k, x, new, new_id, minimum_nprobes=2, maximum_nprobes=8,
                                            refine_factor=rf)
        si, sd, sc, sn = ix.search_probed(q, k, minimum_nprobes=2, maximum_nprobes=8, refine_factor=kr, vectors=x)
        want = _merge((si, sd, sc), lb.flat_search(new, q, k, metric, row_ids=new_id), k)
        _assert_same((pi, pd, pc), want, (kind, "probed", rf))
        assert np.array_equal(pn, sn)


def _oracle_index(kind, ix, metric, q, kc, nprobes):
    from test_probed_search import _oracle
    e = ix.export()
    if kind == "pq":
        return ob.ivfpq_search(e["centroids"], e["codebook"], e["part_offsets"], e["codes"], e["row_ids"], q, kc,
                               nprobes, metric=metric, nthreads=NT)
    return _oracle(kind, e, metric, q, kc, nprobes)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_combined_search_against_the_oracle_composition(kind):
    """oracle index search with k * rf candidates, the oracle's exact re-rank, the flat_knn restatement over the new
    rows, merge"""
    rng = np.random.default_rng(7900 + KINDS.index(kind))
    n_ix, n_new, d, K, k, rf, nprobes = 5000, 700, 32, 12, 10, 4, 3
    x, q = _column(rng, n_ix + n_new, d, "f32", 10)
    ix = _build(kind, x[:n_ix], K, "l2")
    new_id = np.arange(n_ix, n_ix + n_new, dtype=np.uint64)
    got = ix.search_combined(q, k, x, x[n_ix:], new_id, nprobes=nprobes, refine_factor=rf)
    oi, _, oc = _oracle_index(kind, ix, "l2", q, k * rf, nprobes)
    ri, rd, rc = (np.full((len(q), k), NONE, np.uint64), np.full((len(q), k), np.inf, np.float32),
                  np.zeros(len(q), np.uint32))
    for i in range(len(q)):
        cand = oi[i, :oc[i]].astype(np.int64)
        ex = np.array([ob.l2(q[i], x[c]) for c in cand], np.float32)
        order = np.lexsort((cand, ex))[:k]
        ri[i, :len(order)], rd[i, :len(order)], rc[i] = cand[order], ex[order], len(order)
    want = _merge((ri, rd, rc), fr.flat_search(x[n_ix:], q, k, "l2", row_ids=new_id), k)
    _assert_same(got[:3], want, kind)


@pytest.mark.gpu
@pytest.mark.parametrize("metric", ["l2", "dot"])
def test_combined_search_over_all_partitions_is_flat_search_over_all_rows(metric):
    """IVF_FLAT over the first 80 % of the rows, the last 20 % unindexed: with nprobes = K every indexed row is scored
    exactly, so the combined search is the flat search over the whole column"""
    rng = np.random.default_rng(8000 + (metric == "dot"))
    n, d, K = 10000, 48, 20
    x, q = _column(rng, n, d, "f32", 25)
    m = n * 8 // 10
    ix = lb.IvfFlatIndex.build(x[:m], metric, num_partitions=K, max_iters=4)
    rid = np.arange(m, n, dtype=np.uint64)
    for k, rf in ((10, 0), (100, 2), (1, 1)):
        got = ix.search_combined(q, k, x, x[m:], rid, nprobes=K, refine_factor=rf)
        _assert_same(got[:3], lb.flat_search(x, q, k, metric), (metric, k, rf))


@pytest.mark.gpu
def test_knn_with_new_data():
    """scanner.rs:4443 restated: k = 20 is more than the new rows, refine(3), with and without a filter; the closest
    new row comes first"""
    rng = np.random.default_rng(8100)
    n, d, n_new = 4000, 32, 10
    x = rng.standard_normal((n, d)).astype(np.float32)
    q = rng.standard_normal((1, d)).astype(np.float32)
    new = np.concatenate([q + np.float32(0.01), rng.standard_normal((n_new - 1, d)).astype(np.float32) * 5])
    col = np.concatenate([x, new])
    new_id = np.arange(n, n + n_new, dtype=np.uint64)
    ix = lb.IvfPqIndex.build(x, "l2", lb.IvfBuildParams(num_partitions=8, num_sub_vectors=8, max_iters=4,
                                                        pq_max_iters=4))
    ids, dists, cnt, _ = ix.search_combined(q, 20, col, new, new_id, nprobes=8, refine_factor=3)
    assert cnt[0] == 20 and ids[0, 0] == n and np.all(np.diff(dists[0]) >= 0)
    # a filter (the even row ids) over both halves
    even = np.arange(0, n + n_new, 2, dtype=np.uint64)
    bm = ix.row_mask(even, None)
    allow_new = _bitmap(new_id % 2 == 0)
    ids, dists, cnt, _ = ix.search_combined(q, 20, col, new, new_id, nprobes=8, refine_factor=3, allow_bitmap=bm,
                                            unindexed_allow_bitmap=allow_new)
    assert cnt[0] == 20 and ids[0, 0] == n and np.all(ids[0] % 2 == 0)


@pytest.mark.gpu
def test_combined_search_refusals():
    rng = np.random.default_rng(8200)
    x = rng.standard_normal((2000, 16)).astype(np.float32)
    ix = lb.IvfFlatIndex.build(x, "l2", num_partitions=4, max_iters=2)
    q = x[:2]
    sp = _lib.SearchParams(10, 2, 0, x.ctypes.data, len(x), None, 0, 0, 0.0, 0.0)
    rid = np.arange(5, dtype=np.uint64)
    u = _lib.UnindexedRows(x.ctypes.data, 5, rid.ctypes.data, None)
    out = np.empty((2, 10), np.uint64), np.empty((2, 10), np.float32)
    call = lambda sp, pp, u, npo=None: _lib.lib().lb2_index_search_combined(  # noqa: E731
        ix._h, C.c_void_p(q.ctypes.data), C.c_uint64(2), C.byref(sp), pp, u, C.c_void_p(out[0].ctypes.data),
        C.c_void_p(out[1].ctypes.data), None, npo)
    assert call(sp, None, None) == _lib.INVALID_ARG
    assert call(_lib.SearchParams(10, 2, 0, None, 0, None, 0, 0, 0.0, 0.0), None, C.byref(u)) == _lib.INVALID_ARG
    assert call(_lib.SearchParams(0, 2, 0, x.ctypes.data, len(x), None, 0, 0, 0.0, 0.0), None, C.byref(u)) == \
        _lib.INVALID_ARG
    assert call(sp, None, C.byref(_lib.UnindexedRows(x.ctypes.data, 5, None, None))) == _lib.INVALID_ARG
    npo = np.empty(2, np.uint32)
    assert call(sp, None, C.byref(u), C.c_void_p(npo.ctypes.data)) == _lib.INVALID_ARG
    assert call(_lib.SearchParams(1025, 2, 0, x.ctypes.data, len(x), None, 0, 0, 0.0, 0.0), None, C.byref(u)) == \
        _lib.UNSUPPORTED
    assert call(sp, None, C.byref(u)) == _lib.OK
