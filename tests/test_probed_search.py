"""lb2_index_search_probed on the device against the restated probe rule (tests/probe_rule.py) followed by each index
kind's reference search with the query's own nprobes, plus the shortcut rows.  Ids, distance bits, counts and the
number of partitions searched must all match."""
import ctypes as C

import numpy as np
import pytest

import lance_b200 as lb
from lance_b200 import _lib
from oracle import binding as ob
from probe_rule import probe_count
from rq_reference import ivfrq_search
from sq_reference import ivfsq_search

pytestmark = pytest.mark.gpu

KINDS = ["pq8", "pq4", "flat", "sq", "rq"]


def _build(kind, data, K, metric="l2", seed=0):
    if kind in ("pq8", "pq4"):
        p = lb.IvfBuildParams(num_partitions=K, num_sub_vectors=8, num_bits=8 if kind == "pq8" else 4, max_iters=4,
                              pq_max_iters=4, seed=seed)
        return lb.IvfPqIndex.build(data, metric, p)
    b = {"flat": lb.IvfFlatIndex, "sq": lb.IvfSqIndex, "rq": lb.IvfRqIndex}[kind]
    return b.build(data, metric, num_partitions=K, max_iters=4, seed=seed)


def _oracle(kind, e, metric, q, k, nprobes, allow=None, lower=None, upper=None):
    kw = dict(allow=allow, lower=lower, upper=upper)
    if kind in ("pq8", "pq4"):
        return ob.ivfpq_search(e["centroids"], e["codebook"], e["part_offsets"], e["codes"], e["row_ids"], q, k,
                               nprobes, metric=metric, nbits=8 if kind == "pq8" else 4, **kw)
    if kind == "flat":
        return ob.ivfflat_search(e["centroids"], e["part_offsets"], e["vectors"], e["row_ids"], q, k, nprobes,
                                 metric=metric, **kw)
    if kind == "sq":
        return ivfsq_search(e["centroids"], e["bounds"], e["part_offsets"], e["codes"], e["row_ids"], q, k, nprobes,
                            metric=metric, **kw)
    return ivfrq_search(e["centroids"], e["rotation"], e["part_offsets"], e["codes"], e["add_factors"],
                        e["scale_factors"], e["row_ids"], q, k, nprobes, metric=metric, **kw)


def _allowed_per_partition(e, allow):
    off = np.asarray(e["part_offsets"], np.int64)
    ok = np.ones(len(e["row_ids"]), bool) if allow is None else np.isin(e["row_ids"], np.asarray(allow, np.uint64))
    return np.array([ok[off[p]:off[p + 1]].sum() for p in range(len(off) - 1)], np.int64)


def _expected(kind, e, metric, q, k, minimum=1, maximum=None, late_width=1, allow=None, max_len=None, mask_ids=None):
    """the restated rule per query, then the reference search with that nprobes, then the shortcut rows"""
    K = e["centroids"].shape[0]
    L = K if maximum is None else min(maximum, K)
    allowed = _allowed_per_partition(e, allow)
    nq = q.shape[0]
    ids, dists = np.full((nq, k), ~np.uint64(0), np.uint64), np.full((nq, k), np.inf, np.float32)
    counts, nps = np.zeros(nq, np.uint32), np.zeros(nq, np.uint32)
    for i in range(nq):
        pids, pd = ob.find_partitions(e["centroids"], q[i], L, "dot" if metric == "dot" else "l2")
        c = np.minimum(k, allowed[pids])
        n, sc, _ = probe_count(pd, c, k, minimum, maximum, late_width, max_len, mask_ids is not None)
        oi, od, oc = _oracle(kind, e, metric, q[i:i + 1], k, n, allow=allow)
        ri, rd = list(oi[0, :oc[0]]), list(od[0, :oc[0]])
        if sc:
            extra = sorted(set(int(x) for x in mask_ids) - set(int(x) for x in ri))
            ri += extra
            rd += [np.float32(np.inf)] * len(extra)
        keys = [(lb_key(d_), int(r)) for d_, r in zip(rd, ri)]
        order = sorted(range(len(ri)), key=lambda j: keys[j])[:k]
        counts[i], nps[i] = len(order), n
        ids[i, :len(order)] = [ri[j] for j in order]
        dists[i, :len(order)] = [rd[j] for j in order]
    return ids, dists, counts, nps


def lb_key(d):
    b = np.array([d], np.float32).view(np.int32)[0]
    return int(b ^ ((b >> 31) & 0x7fffffff))


def _same(got, want):
    gi, gd, gc, gn = got
    wi, wd, wc, wn = want
    assert np.array_equal(gn, wn), (gn, wn)
    assert np.array_equal(gc, wc), (gc, wc)
    for i in range(len(gc)):
        n = int(gc[i])
        assert np.array_equal(gi[i, :n], wi[i, :n]), i
        assert np.array_equal(gd[i, :n].view(np.uint32), wd[i, :n].view(np.uint32)), i


def _data(n, d, seed, clusters=32):
    rng = np.random.default_rng(seed)
    base = rng.standard_normal((clusters, d)).astype(np.float32) * 4
    return (base[rng.integers(0, clusters, n)] + rng.standard_normal((n, d)).astype(np.float32)).astype(np.float32)


@pytest.fixture(scope="module", params=KINDS)
def small(request):
    kind = request.param
    d, n, K = 16, 3000, 48
    data = _data(n, d, 7)
    ix = _build(kind, data, K)
    q = _data(24, d, 8)
    return kind, ix, ix.export(), data, q


# ---- min == max == p is lb2_index_search_ex with nprobes = p ------------------------------------------------------
@pytest.mark.parametrize("variant", ["plain", "mask", "range", "refine"])
def test_fixed_equals_search_ex(small, variant):
    kind, ix, e, data, q = small
    rng = np.random.default_rng(3)
    kw = {}
    if variant == "mask":
        kw = {"allow_bitmap": ix.row_mask(rng.choice(e["row_ids"], 700, replace=False), None)}
    elif variant == "range":
        pl = ix.search_ex(q, k=10, nprobes=4)[1]
        kw = {"lower_bound": float(np.median(pl[:, 1])), "upper_bound": float(np.median(pl[:, 8]))}
    elif variant == "refine":
        kw = {"refine_factor": 3, "vectors": data}
    for p in (1, 4, 48, 60):
        want = ix.search_ex(q, k=10, nprobes=p, **kw)
        gi, gd, gc, gn = ix.search_probed(q, 10, minimum_nprobes=p, maximum_nprobes=p, **kw)
        assert np.array_equal(gi, want[0]) and np.array_equal(gd.view(np.uint32), want[1].view(np.uint32)), p
        assert (gn == min(p, 48)).all()


# ---- the default query and filters against the restated rule + the reference search -------------------------------
def test_default_query(small):
    kind, ix, e, data, q = small
    for k in (1, 5, 10, 40):
        _same(ix.search_probed(q, k), _expected(kind, e, "l2", q, k))


@pytest.mark.parametrize("frac", [0.5, 0.05, 0.003, 0.0])
@pytest.mark.parametrize("width", [1, 3, 64])
@pytest.mark.parametrize("maximum", [None, 20])
def test_filters(small, frac, width, maximum):
    kind, ix, e, data, q = small
    rng = np.random.default_rng(int(frac * 1000) + width)
    allow = rng.choice(e["row_ids"], int(len(e["row_ids"]) * frac), replace=False)
    bm = ix.row_mask(allow, None)
    k = 10
    got = ix.search_probed(q, k, minimum_nprobes=2, maximum_nprobes=maximum, late_width=width, allow_bitmap=bm,
                           mask_max_len=len(allow))
    _same(got, _expected(kind, e, "l2", q, k, 2, maximum, width, allow=allow, max_len=len(allow)))
    # iterable: the shortcut answers whenever max_len <= k
    got = ix.search_probed(q, k, minimum_nprobes=2, maximum_nprobes=maximum, late_width=width, allow_bitmap=bm,
                           mask_max_len=len(allow), mask_ids=allow)
    _same(got, _expected(kind, e, "l2", q, k, 2, maximum, width, allow=allow, max_len=len(allow), mask_ids=allow))


def test_block_list_only(small):
    kind, ix, e, data, q = small
    block = e["row_ids"][::3]
    bm = ix.row_mask(None, block)
    allow = np.setdiff1d(e["row_ids"], block)
    _same(ix.search_probed(q, 20, allow_bitmap=bm), _expected(kind, e, "l2", q, 20, allow=allow))


def test_range_with_late_search(small):
    kind, ix, e, data, q = small
    k = 10
    pl = ix.search_ex(q, k=k, nprobes=48)[1]
    lo, hi = float(np.median(pl[:, 0])), float(np.median(pl[:, 3]))
    for maximum in (None, 12):
        got = ix.search_probed(q, k, maximum_nprobes=maximum, lower_bound=lo, upper_bound=hi)
        # c_p from the reference's own range search of each partition
        K = e["centroids"].shape[0]
        L = K if maximum is None else maximum
        for i in range(q.shape[0]):
            pids, pd = ob.find_partitions(e["centroids"], q[i], L, "l2")
            c = [_range_count(kind, e, p, q[i:i + 1], k, lo, hi) for p in pids]
            n, _, _ = probe_count(pd, c, k, 1, maximum, 1)
            assert got[3][i] == n, i
            oi, od, oc = _oracle(kind, e, "l2", q[i:i + 1], k, n, lower=lo, upper=hi)
            assert got[2][i] == oc[0]
            assert np.array_equal(got[0][i, :oc[0]], oi[0, :oc[0]])
            assert np.array_equal(got[1][i, :oc[0]].view(np.uint32), od[0, :oc[0]].view(np.uint32))


def _range_count(kind, e, p, q1, k, lo, hi):
    """rows partition p returns to a range search: the reference search over an index whose other partitions are
    empty"""
    off = np.asarray(e["part_offsets"], np.uint64)
    po = np.where(np.arange(len(off)) <= p, off[p], off[p + 1]).astype(np.uint64)
    K = e["centroids"].shape[0]
    oi, od, oc = _oracle(kind, dict(e, part_offsets=po), "l2", q1, k, K, lower=lo, upper=hi)
    return int(oc[0])


def test_refine_factor_counts_kc_per_partition(small):
    kind, ix, e, data, q = small
    k, rf = 10, 4
    got = ix.search_probed(q, k, refine_factor=rf, vectors=data)
    want_np = []
    K = e["centroids"].shape[0]
    allowed = _allowed_per_partition(e, None)
    for i in range(q.shape[0]):
        pids, pd = ob.find_partitions(e["centroids"], q[i], K, "l2")
        want_np.append(probe_count(pd, np.minimum(k * rf, allowed[pids]), k)[0])
    assert np.array_equal(got[3], want_np)
    for n in set(want_np):
        sel = np.array(want_np) == n
        ref = ix.search_ex(q[sel], k=k, nprobes=n, refine_factor=rf, vectors=data)
        assert np.array_equal(got[0][sel], ref[0])
        assert np.array_equal(got[1][sel].view(np.uint32), ref[1].view(np.uint32))


def test_shortcut_variants(small):
    kind, ix, e, data, _ = small
    q = e["centroids"][:24]     # a query on a centroid prunes to few partitions, so the shortcut has room to act
    rng = np.random.default_rng(11)
    allow = rng.choice(e["row_ids"], 6, replace=False)
    outside = np.array([10 ** 9, 10 ** 9 + 7], np.uint64)
    bm = ix.row_mask(allow, None)
    for ids in (allow, np.concatenate([allow, outside])):
        got = ix.search_probed(q, 10, minimum_nprobes=1, maximum_nprobes=None, allow_bitmap=bm, mask_ids=ids,
                               mask_max_len=len(ids))
        _same(got, _expected(kind, e, "l2", q, 10, allow=allow, max_len=len(ids), mask_ids=ids))
        assert (got[2] == len(ids)).any()           # some queries took the shortcut
        # refine: the shortcut rows get exact distances (ids outside the column get NaN, ordered last)
        gr = ix.search_probed(q, 10, allow_bitmap=bm, mask_ids=ids, mask_max_len=len(ids), refine_factor=1,
                              vectors=data)
        assert np.array_equal(gr[2], got[2])
        assert np.isfinite(gr[1][:, :len(allow)]).all()
    # found0 == max_len: every allowed row is found in the initial search, nothing is added
    got = ix.search_probed(q, 10, minimum_nprobes=48, allow_bitmap=bm, mask_ids=allow, mask_max_len=len(allow))
    _same(got, _expected(kind, e, "l2", q, 10, minimum=48, allow=allow, max_len=len(allow), mask_ids=allow))
    assert np.isfinite(got[1][:, :len(allow)]).all()


# ---- shapes -----------------------------------------------------------------------------------------------------
def test_small_and_empty_partitions():
    d, K = 8, 64
    rng = np.random.default_rng(1)
    cent = rng.standard_normal((K, d)).astype(np.float32)
    sizes = rng.integers(0, 4, K)
    sizes[::5] = 0
    part = np.repeat(np.arange(K, dtype=np.uint32), sizes)
    vec = (cent[part] + 0.01 * rng.standard_normal((len(part), d))).astype(np.float32)
    ix = lb.IvfFlatIndex.from_parts(cent, part, vec)
    e = ix.export()
    q = rng.standard_normal((16, d)).astype(np.float32)
    for k in (1, 10, 50):
        for w in (1, 3):
            _same(ix.search_probed(q, k, late_width=w), _expected("flat", e, "l2", q, k, late_width=w))


def test_ranking_past_shared_memory():
    d, K = 4, 9000   # above RANK_TILE = 8192: tiles merged in global memory
    rng = np.random.default_rng(2)
    cent = rng.standard_normal((K, d)).astype(np.float32)
    part = rng.integers(0, K, 2000).astype(np.uint32)
    vec = (cent[part] + 0.01 * rng.standard_normal((len(part), d))).astype(np.float32)
    ix = lb.IvfFlatIndex.from_parts(cent, part, vec)
    e = ix.export()
    q = rng.standard_normal((6, d)).astype(np.float32)
    for k in (1, 30):
        _same(ix.search_probed(q, k), _expected("flat", e, "l2", q, k))
    got = ix.search_probed(q, 5, minimum_nprobes=K, maximum_nprobes=K)
    want = ix.search_ex(q, k=5, nprobes=K)
    assert np.array_equal(got[0], want[0]) and (got[3] == K).all()


@pytest.mark.parametrize("metric", ["dot", "cosine"])
def test_metrics_fixed_and_default(metric):
    data = _data(2000, 16, 21)
    ix = _build("flat", data, 32, metric)
    q = _data(16, 16, 22)
    for p in (1, 7):
        got = ix.search_probed(q, 10, minimum_nprobes=p, maximum_nprobes=p)
        want = ix.search_ex(q, k=10, nprobes=p)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1].view(np.uint32), want[1].view(np.uint32))
    if metric == "dot":
        _same(ix.search_probed(q, 10), _expected("flat", ix.export(), "dot", q, 10))


def test_more_queries_than_one_slab_and_empty_inputs():
    data = _data(1000, 8, 31, clusters=8)
    ix = _build("flat", data, 8)
    q = _data(33000, 8, 32, clusters=8)
    got = ix.search_probed(q, 5, minimum_nprobes=2, maximum_nprobes=2)
    want = ix.search_ex(q, k=5, nprobes=2)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1].view(np.uint32), want[1].view(np.uint32))
    g = ix.search_probed(q, 5)
    sel = np.r_[0:8, 32760:32776, 32992:33000]
    _same(tuple(a[sel] for a in g), _expected("flat", ix.export(), "l2", q[sel], 5))
    got = ix.search_probed(q[:0], 5)
    assert got[0].shape == (0, 5)
    cent = np.eye(4, dtype=np.float32)
    empty = lb.IvfFlatIndex.from_parts(cent, np.zeros(0, np.uint32), np.zeros((0, 4), np.float32))
    gi, gd, gc, gn = empty.search_probed(np.ones((3, 4), np.float32), 4)
    assert (gc == 0).all() and (gn == 4).all()


def test_invalid_arguments(small):
    kind, ix, e, data, q = small
    bm = ix.row_mask(e["row_ids"][:5], None)
    bad = [dict(minimum_nprobes=0), dict(minimum_nprobes=5, maximum_nprobes=4), dict(late_width=0),
           dict(mask_ids=e["row_ids"][:5]), dict(mask_max_len=5)]
    for kw in bad:
        with pytest.raises(lb.LanceB200Error) as ei:
            ix.search_probed(q, 10, **kw)
        assert ei.value.status == _lib.INVALID_ARG, kw
    # sp->nprobes != 0
    sp = _lib.SearchParams(10, 3, 0, None, 0, None, 0, 0, 0.0, 0.0)
    pp = _lib.ProbeParams(1, 0, 1, 0, 0, None, 0)
    qq = np.ascontiguousarray(q, np.float32)
    out_i, out_d = np.empty((len(q), 10), np.uint64), np.empty((len(q), 10), np.float32)
    st = _lib.lib().lb2_index_search_probed(ix._h, C.c_void_p(qq.ctypes.data), C.c_uint64(len(q)), C.byref(sp),
                                            C.byref(pp), C.c_void_p(out_i.ctypes.data), C.c_void_p(out_d.ctypes.data),
                                            None, None)
    assert st == _lib.INVALID_ARG
    del bm


def test_fixed_path_launches_no_new_kernels(small):
    kind, ix, e, data, q = small
    new = ("rank_probes", "partition_counts", "probe_cutoff", "gather_probes", "probe_shortcut")
    lb.profile.enable(True)
    try:
        lb.profile.reset()
        ix.search_ex(q, k=10, nprobes=5)
        names = lb.profile.dump()
        assert not any(n in key for key in names for n in new), names
        lb.profile.reset()
        ix.search_probed(q, 10)
        names = lb.profile.dump()
        assert any("rank_probes" in key for key in names) and any("probe_cutoff" in key for key in names), names
    finally:
        lb.profile.enable(False)


# ---- NprobesTestFixture (knn.rs:1605-1702) restated ------------------------------------------------------------
@pytest.fixture(scope="module")
def nprobes_fixture():
    K = 100
    # RadialStepGenerator: angle = (step as f32) / (steps as f32) * 2.0 * PI, all in f32, then cos / sin of it.
    # Mirror-image centroids (1 and 99, ...) are not exact ties in f32, which fixes the probe order.
    ang = (np.arange(K, dtype=np.float32) / np.float32(K) * np.float32(2.0) * np.float32(np.pi)).astype(np.float32)
    cent = np.stack([np.cos(ang.astype(np.float64)), np.sin(ang.astype(np.float64))], 1).astype(np.float32)
    n = 10000
    rng = np.random.default_rng(0)
    jit = rng.standard_normal((n, 2)).astype(np.float32)
    jit *= np.float32(0.0001) / np.linalg.norm(jit, axis=1, keepdims=True).astype(np.float32)
    vec = (cent[np.arange(n) % K] + jit).astype(np.float32)
    part = ob.compute_membership(cent, vec, nthreads=8)[0].astype(np.uint32)
    rowid = ((np.arange(n, dtype=np.uint64) // 100) << np.uint64(32)) | (np.arange(n, dtype=np.uint64) % 100)
    codebook = rng.random((2, 256, 1)).astype(np.float32)
    codes = rng.integers(0, 256, (n, 2)).astype(np.uint8)
    ix = lb.IvfPqIndex.from_parts(cent, codebook, part, codes, row_ids=rowid)
    label = np.arange(n) % 61
    # the same index with row id = row number, so that the raw column can be indexed by row id for refine
    ix_rows = lb.IvfPqIndex.from_parts(cent, codebook, part, codes)
    return ix, cent, vec, rowid, label, ix_rows


def test_reference_nprobes_scenarios(nprobes_fixture):
    ix, cent, vec, rowid, label, ix_rows = nprobes_fixture
    q = cent[:1]
    sel = np.sort(rowid[label == 17])
    bm = ix.row_mask(sel, None)
    # test_no_max_nprobes
    i, d, c, n = ix.search_probed(q, 50, minimum_nprobes=10, allow_bitmap=bm, mask_ids=sel, mask_max_len=len(sel))
    assert c[0] == 50 and n[0] < 100
    # test_no_prefilter_results
    none = np.zeros(0, np.uint64)
    i, d, c, n = ix.search_probed(q, 50, minimum_nprobes=10, allow_bitmap=ix.row_mask(none, None), mask_ids=none,
                                  mask_max_len=0)
    assert c[0] == 0 and n[0] == 10
    # test_some_max_nprobes
    for p, rows in ((10, 16), (20, 33), (30, 48)):
        i, d, c, n = ix.search_probed(q, 50, minimum_nprobes=p, maximum_nprobes=p, allow_bitmap=bm, mask_ids=sel,
                                      mask_max_len=len(sel))
        assert (c[0], n[0]) == (rows, p)
    # userid < 20: 5 rows found in the first 10 partitions, the other 15 at +inf
    few = np.sort(rowid[:20])
    bm20 = ix.row_mask(few, None)
    i, d, c, n = ix.search_probed(q, 50, minimum_nprobes=10, allow_bitmap=bm20, mask_ids=few, mask_max_len=20)
    assert (n[0], c[0]) == (10, 20)
    assert int(np.isinf(d[0, :c[0]]).sum()) == 15
    few = np.arange(20, dtype=np.uint64)
    i, d, c, n = ix_rows.search_probed(q, 50, minimum_nprobes=10, allow_bitmap=ix_rows.row_mask(few, None),
                                       mask_ids=few, mask_max_len=20, refine_factor=1, vectors=vec)
    assert c[0] == 20 and int(np.isinf(d[0, :c[0]]).sum()) == 0
