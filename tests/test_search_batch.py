"""lb2_index_search_batch: a batch whose queries each carry their own k, probes, refine factor, range, prefilter and
ef.  Row q must be bit for bit the single-parameter call of query q alone (lb2_index_search_ex, or
lb2_index_search_hnsw with the query's ef): ids, distance bits, counts and nprobes_out."""
import ctypes as C
import os

import numpy as np
import pytest

import lance_b200 as lb
from lance_b200 import _lib

pytestmark = pytest.mark.gpu

U64MAX = np.uint64(0xFFFFFFFFFFFFFFFF)


def _data(n, d, seed, clusters=12, dup=0.05):
    rng = np.random.default_rng(seed)
    base = rng.standard_normal((clusters, d)).astype(np.float32) * 4
    x = (base[rng.integers(0, clusters, n)] + rng.standard_normal((n, d)).astype(np.float32)).astype(np.float32)
    nd = int(n * dup)  # duplicate rows: ties at the k-th distance reach the tie replay under per-query k
    x[rng.choice(n, nd, replace=False)] = x[rng.choice(n, nd, replace=False)]
    return x


def _build(kind, data, K, metric):
    hp = lb.HnswBuildParams(m=8, ef_construction=40) if kind.startswith("hnsw") else None
    if kind in ("pq8", "pq4"):
        M = 16 if data.shape[1] == 128 else 8
        p = lb.IvfBuildParams(num_partitions=K, num_sub_vectors=M, num_bits=8 if kind == "pq8" else 4, max_iters=4,
                              pq_max_iters=4, seed=1)
        return lb.IvfPqIndex.build(data, metric, p)
    if kind == "flat_f16":
        return lb.IvfFlatIndex.build(data.astype(np.float16), metric, num_partitions=K, max_iters=4, seed=1)
    if kind == "flat_bf16":
        bits = (data.view(np.uint32) >> 16).astype(np.uint16)
        return lb.IvfFlatIndex.build(bits, metric, num_partitions=K, max_iters=4, seed=1, bf16=True)
    if kind == "hnsw_pq":
        p = lb.IvfBuildParams(num_partitions=K, num_sub_vectors=8, num_bits=8, max_iters=4, pq_max_iters=4, seed=1)
        return lb.IvfHnswPqIndex.build(data, metric, p, hp)
    b = {"flat": lb.IvfFlatIndex, "sq": lb.IvfSqIndex, "rq": lb.IvfRqIndex, "hnsw_sq": lb.IvfHnswSqIndex,
         "hnsw_flat": lb.IvfHnswFlatIndex}[kind]
    kw = {"hnsw_params": hp} if hp is not None else {}
    return b.build(data, metric, num_partitions=K, max_iters=4, seed=1, **kw)


def _queries(ix, q):
    dt = getattr(ix, "_dt", lb.F32)
    if dt == lb.BF16:
        return np.ascontiguousarray((q.view(np.uint32) >> 16).astype(np.uint16))
    return np.ascontiguousarray(q, dtype={lb.F32: np.float32, lb.F16: np.float16}[dt])


def _single(ix, qv, k, nprobes, rf, vectors, bitmap, lo, hi, ef):
    """the single-parameter call of one query: (ids [k], dists [k], count)"""
    ids, dists, cnt = np.empty((1, k), np.uint64), np.empty((1, k), np.float32), np.empty(1, np.uint32)
    vp = None if vectors is None else C.c_void_p(vectors.ctypes.data)
    sp = _lib.SearchParams(k, nprobes, rf, vp.value if rf else None, 0 if vectors is None else vectors.shape[0],
                           None if bitmap is None else bitmap.ctypes.data, int(lo is not None), int(hi is not None),
                           float(lo or 0.0), float(hi or 0.0))
    args = (ix._h, C.c_void_p(qv.ctypes.data), C.c_uint64(1), C.byref(sp))
    outs = (C.c_void_p(ids.ctypes.data), C.c_void_p(dists.ctypes.data), C.c_void_p(cnt.ctypes.data))
    if ef is not None:
        _lib.check(_lib.lib().lb2_index_search_hnsw(*args, None, C.c_uint32(ef), *outs, None))
    else:
        _lib.check(_lib.lib().lb2_index_search_ex(*args, *outs))
    return ids[0], dists[0], int(cnt[0])


def _filters(ix, e, rng):
    rid = e["row_ids"]
    return [ix.row_mask(None, rng.choice(rid, len(rid) // 3, replace=False)),         # a block list
            ix.row_mask(rng.choice(rid, len(rid) // 2, replace=False), None),         # an allow list, ~50 %
            ix.row_mask(rng.choice(rid, 40, replace=False), None),                    # a selective allow list
            ix.row_mask(np.zeros(0, np.uint64), None)]                                # an empty allow list


def _random_params(nq, K, rng, hnsw, pl):
    k = rng.integers(1, 101, nq)
    rf = np.where(rng.random(nq) < 0.4, rng.integers(1, 11, nq), 0)
    rf = np.where(k * np.maximum(rf, 1) > 1024, 0, rf)
    big = rng.choice(nq, 4, replace=False)  # a few queries at k' = 1024
    k[big[:2]], rf[big[:2]] = 1024, 0
    k[big[2:]], rf[big[2:]] = 128, 8
    nprobes = rng.integers(1, K + 3, nq)
    fof = rng.integers(-1, 4, nq)
    lo = np.where(rng.random(nq) < 0.15, np.float32(np.quantile(pl, 0.02)), np.nan).astype(np.float32)
    hi = np.where(rng.random(nq) < 0.15, np.float32(np.quantile(pl, 0.6)), np.nan).astype(np.float32)
    ef = np.zeros(nq, np.int64)
    if hnsw:
        kc = k * np.maximum(rf, 1)
        ef = np.where(rng.random(nq) < 0.5, kc + rng.integers(0, 40, nq), 0)
    return k, nprobes, rf, fof, lo, hi, ef


def _check_rows(ix, q, data, filters, got, params, k_stride):
    k, nprobes, rf, fof, lo, hi, ef = params
    K = ix.info()["num_partitions"]
    gi, gd, gc, gn = got
    vec = _queries(ix, data) if rf.any() else None
    for i in range(len(q)):
        qi = _queries(ix, q[i:i + 1])
        li = None if np.isnan(lo[i]) else float(lo[i])
        hi_ = None if np.isnan(hi[i]) else float(hi[i])
        bm = None if fof[i] < 0 else np.ascontiguousarray(filters[fof[i]], np.uint64)
        wi, wd, wc = _single(ix, qi, int(k[i]), int(nprobes[i]), int(rf[i]), vec, bm, li, hi_,
                             int(ef[i]) if ef[i] else None)
        ki = int(k[i])
        assert np.array_equal(gi[i, :ki], wi), i
        assert np.array_equal(gd[i, :ki].view(np.uint32), wd.view(np.uint32)), i
        assert gc[i] == wc and gn[i] == min(int(nprobes[i]), K), i
        assert (gi[i, ki:k_stride] == U64MAX).all() and np.isinf(gd[i, ki:k_stride]).all(), i


CASES = [(kind, m) for kind in ("pq8", "pq4", "flat", "flat_f16", "flat_bf16", "sq", "rq")
         for m in ("l2", "cosine", "dot")] + \
        [(kind, m) for kind in ("hnsw_sq", "hnsw_pq", "hnsw_flat") for m in ("l2", "cosine", "dot")]


@pytest.fixture(scope="module", params=CASES, ids=lambda c: f"{c[0]}-{c[1]}")
def case(request):
    kind, metric = request.param
    d = 128 if kind == "pq8" else 16
    data = _data(4000, d, 7)
    K = 24
    ix = _build(kind, data, K, metric)
    return kind, metric, ix, ix.export(), data


def _run_case(case, scan=None):
    kind, metric, ix, e, data = case
    rng = np.random.default_rng(11)
    nq = 300
    q = _data(nq, data.shape[1], 8)
    filters = _filters(ix, e, rng)
    pl = ix.search_ex(_queries(ix, q[:16]), k=10, nprobes=4)[1]
    params = _random_params(nq, ix.info()["num_partitions"], rng, kind.startswith("hnsw"), pl[np.isfinite(pl)])
    k, nprobes, rf, fof, lo, hi, ef = params
    old = os.environ.get("LB2_SCAN")
    if scan:
        os.environ["LB2_SCAN"] = scan
    try:
        got = ix.search_batch(_queries(ix, q), k, nprobes=nprobes, refine_factor=rf, vectors=_queries(ix, data),
                              filters=filters, filter_of=fof, lower_bound=lo, upper_bound=hi,
                              ef=ef if kind.startswith("hnsw") else None)
        _check_rows(ix, q, data, filters, got, params, int(k.max()))
    finally:
        if scan:
            if old is None:
                os.environ.pop("LB2_SCAN", None)
            else:
                os.environ["LB2_SCAN"] = old


def test_rows_equal_single_calls(case):
    if case[0] == "pq8":
        for scan in ("classic", "skew"):
            _run_case(case, scan)
    else:
        _run_case(case)


def test_uniform_batch_equals_search_ex(case):
    kind, metric, ix, e, data = case
    q = _queries(ix, _data(200, data.shape[1], 9))
    want = ix.search_ex(q, k=10, nprobes=5)
    gi, gd, gc, gn = ix.search_batch(q, 10, nprobes=5)
    assert np.array_equal(gi, want[0]) and np.array_equal(gd.view(np.uint32), want[1].view(np.uint32))
    assert (gn == 5).all()


def test_past_one_query_slab():
    data = _data(1500, 8, 3)
    ix = _build("flat", data, 8, "l2")
    nq = 32768 + 5
    q = _data(nq, 8, 4)
    k = np.where(np.arange(nq) % 2 == 0, 5, 12)
    nprobes = np.where(np.arange(nq) % 3 == 0, 2, 6)
    gi, gd, gc, gn = ix.search_batch(q, k, nprobes=nprobes)
    for kk in (5, 12):
        for p in (2, 6):
            sel = np.nonzero((k == kk) & (nprobes == p))[0]
            wi, wd = ix.search_ex(q[sel], k=kk, nprobes=p)
            assert np.array_equal(gi[sel, :kk], wi) and np.array_equal(gd[sel, :kk].view(np.uint32), wd.view(np.uint32))
            assert (gi[sel, kk:] == U64MAX).all()


@pytest.mark.parametrize("kfast", [True, False])
def test_launches_do_not_grow_with_parameter_sets(kfast):
    data = _data(6000, 128, 5)
    ix = _build("pq8", data, 32, "l2")
    e = ix.export()
    rng = np.random.default_rng(2)
    nq = 512
    q = _data(nq, 128, 6)
    filters = [ix.row_mask(rng.choice(e["row_ids"], 3000, replace=False), None) for _ in range(nq)]
    k = rng.integers(1, 16, nq) if kfast else rng.integers(16, 120, nq)
    k[0] = 15 if kfast else 119  # the shared batch takes the largest k, so both use the same merge
    nprobes = rng.integers(1, 11, nq)
    nprobes[0] = 10
    L = _lib.lib()
    n0, n1 = C.c_uint64(), C.c_uint64()
    _lib.check(L.lb2_launch_count(C.byref(n0), 1))
    ix.search_batch(q, k, nprobes=nprobes, filters=filters, filter_of=np.arange(nq))
    _lib.check(L.lb2_launch_count(C.byref(n0), 1))
    ix.search_batch(q, int(k.max()), nprobes=10, filters=filters[:1], filter_of=0)
    _lib.check(L.lb2_launch_count(C.byref(n1), 1))
    assert n0.value == n1.value, (n0.value, n1.value)


def test_refusals_leave_outputs_untouched():
    data = _data(2000, 16, 1)
    ix = _build("flat", data, 8, "l2")
    hx = _build("hnsw_sq", data, 8, "l2")
    q = _data(4, 16, 2)
    bm = ix.row_mask(np.arange(100, dtype=np.uint64), None)

    def call(index, k, nprobes=3, **kw):
        out = (np.full((4, kw.pop("k_stride", 20)), 7, np.uint64), np.full((4, 20), 3.0, np.float32))
        with pytest.raises(lb.LanceB200Error) as ei:
            index.search_batch(q, k, nprobes=nprobes, out=out, **kw)
        assert (out[0] == 7).all() and (out[1] == 3.0).all()
        return ei.value.status

    def last_error():
        buf = C.create_string_buffer(2048)
        _lib.lib().lb2_last_error(buf, 2048)
        return buf.value.decode()

    def raw(index, params, filters=(), vectors=None, k_stride=20):
        ids, dists = np.full((4, max(k_stride, 1)), 7, np.uint64), np.full((4, max(k_stride, 1)), 3.0, np.float32)
        cp = (_lib.QueryParams * 4)(*params)
        cf = (_lib.QueryFilter * max(1, len(filters)))(*filters)
        qq = np.ascontiguousarray(q)
        st = _lib.lib().lb2_index_search_batch(index._h, C.c_void_p(qq.ctypes.data), C.c_uint64(4), cp, cf,
                                                C.c_uint32(len(filters)), vectors, C.c_uint64(0), C.c_uint32(1),
                                                C.c_uint32(k_stride), C.c_void_p(ids.ctypes.data),
                                                C.c_void_p(dists.ctypes.data), None, None)
        assert (ids == 7).all() and (dists == 3.0).all()
        if params[3] is not params[0]:  # a refusal of query 3's own parameters names it
            assert "query 3" in last_error(), last_error()
        return st

    ok = _lib.QueryParams(5, 3, 0, 0, 0, 0xFFFFFFFF, 0, 0, 0, 0.0, 0.0)
    assert raw(ix, [ok] * 4, k_stride=4) == _lib.INVALID_ARG                           # k_stride below the largest k
    assert raw(ix, [ok] * 3 + [_lib.QueryParams(5, 3, 0, 0, 0, 2, 0, 0, 0, 0.0, 0.0)]) == _lib.INVALID_ARG  # filter
    assert raw(ix, [ok] * 3 + [_lib.QueryParams(5, 3, 0, 0, 0, 0xFFFFFFFF, 9, 0, 0, 0.0, 0.0)]) == _lib.INVALID_ARG
    assert raw(ix, [ok] * 3 + [_lib.QueryParams(5, 3, 0, 0, 2, 0xFFFFFFFF, 0, 0, 0, 0.0, 0.0)]) == _lib.INVALID_ARG
    assert raw(ix, [ok] * 3 + [_lib.QueryParams(0, 3, 0, 0, 0, 0xFFFFFFFF, 0, 0, 0, 0.0, 0.0)]) == _lib.INVALID_ARG
    assert raw(ix, [ok] * 3 + [_lib.QueryParams(5, 0, 0, 0, 0, 0xFFFFFFFF, 0, 0, 0, 0.0, 0.0)]) == _lib.INVALID_ARG
    assert raw(ix, [ok] * 3 + [_lib.QueryParams(5, 0, 4, 3, 0, 0xFFFFFFFF, 0, 0, 0, 0.0, 0.0)]) == _lib.INVALID_ARG
    no_bitmap = [_lib.QueryFilter(None, 1, 5, None, 0)]  # max_len without an allow bitmap
    assert raw(ix, [ok] * 3 + [_lib.QueryParams(5, 0, 1, 0, 0, 0, 0, 0, 0, 0.0, 0.0)], filters=no_bitmap) == \
        _lib.INVALID_ARG
    big = _lib.QueryParams(600, 3, 0, 0, 2, 0xFFFFFFFF, 0, 0, 0, 0.0, 0.0)
    vec = C.c_void_p(np.ascontiguousarray(data).ctypes.data)
    assert raw(ix, [ok] * 3 + [big], vectors=vec, k_stride=600) == _lib.UNSUPPORTED      # k * refine_factor > 1024
    low_ef = _lib.QueryParams(20, 3, 0, 0, 0, 0xFFFFFFFF, 10, 0, 0, 0.0, 0.0)
    assert raw(hx, [ok] * 3 + [low_ef]) == _lib.INVALID_ARG                               # ef < k'
    assert call(ix, 5, filters=[bm], filter_of=0, ef=8) == _lib.INVALID_ARG
    del bm


def _single_probed(ix, qv, k, minimum, maximum, rf, vectors, filt, lo, hi, ef, late_width):
    """lb2_index_search_probed (or lb2_index_search_hnsw with probe parameters) of one query: ids, dists, count, nprobes"""
    ids, dists = np.empty((1, k), np.uint64), np.empty((1, k), np.float32)
    cnt, nps = np.empty(1, np.uint32), np.empty(1, np.uint32)
    bm, max_len, mask = filt if filt is not None else (None, None, None)
    keep = None if mask is None else (np.ascontiguousarray(mask, np.uint64) if len(mask) else np.zeros(1, np.uint64))
    sp = _lib.SearchParams(k, 0, rf, vectors.ctypes.data if rf else None, vectors.shape[0] if rf else 0,
                           None if bm is None else bm.ctypes.data, int(lo is not None), int(hi is not None),
                           float(lo or 0.0), float(hi or 0.0))
    pp = _lib.ProbeParams(minimum, maximum, late_width, int(max_len is not None), int(max_len or 0),
                          None if keep is None else keep.ctypes.data, 0 if mask is None else len(mask))
    args = (ix._h, C.c_void_p(qv.ctypes.data), C.c_uint64(1), C.byref(sp), C.byref(pp))
    outs = tuple(C.c_void_p(a.ctypes.data) for a in (ids, dists, cnt, nps))
    if ef is not None:
        _lib.check(_lib.lib().lb2_index_search_hnsw(*args, C.c_uint32(ef), *outs))
    else:
        _lib.check(_lib.lib().lb2_index_search_probed(*args, *outs))
    return ids[0], dists[0], int(cnt[0]), int(nps[0])


PROBED = [("pq8", "l2"), ("pq4", "dot"), ("flat", "cosine"), ("sq", "l2"), ("rq", "l2"), ("hnsw_sq", "l2"),
          ("hnsw_flat", "dot")]


@pytest.mark.parametrize("kind,metric", PROBED)
@pytest.mark.parametrize("ranged", [False, True])
def test_probe_rule_rows_equal_search_probed(kind, metric, ranged):
    """min / max nprobes queries mixed with fixed ones: each row equals its own lb2_index_search_probed, nprobes_out
    included, through early pruning, late search (late_width 2) and the allow-list shortcut"""
    data = _data(4000, 16, 7)
    ix = _build(kind, data, 24, metric)
    e = ix.export()
    rng = np.random.default_rng(5)
    nq = 160
    q = _data(nq, 16, 8)
    rid = e["row_ids"]
    sel = np.sort(rng.choice(rid, 30, replace=False))
    half = np.sort(rng.choice(rid, len(rid) // 2, replace=False))
    filters = [(ix.row_mask(None, rng.choice(rid, len(rid) // 3, replace=False)), None, None),  # a block list
               (ix.row_mask(half, None), len(half), half),                                    # ~50 %, iterable
               (ix.row_mask(sel, None), len(sel), sel),                                       # selective: shortcut
               (ix.row_mask(sel, None), len(sel), None),                                      # selective, not iterable
               (ix.row_mask(np.zeros(0, np.uint64), None), 0, np.zeros(0, np.uint64))]        # empty allow list
    k = rng.integers(1, 60, nq)
    rf = np.where(rng.random(nq) < 0.3, rng.integers(1, 6, nq), 0)
    nprobes = np.where(rng.random(nq) < 0.7, 0, rng.integers(1, 27, nq))  # 0: the probe rule
    mins = rng.integers(1, 6, nq)
    maxs = np.where(rng.random(nq) < 0.5, 0, mins + rng.integers(0, 20, nq))
    fof = rng.integers(-1, len(filters), nq)
    pl = ix.search_ex(_queries(ix, q[:16]), k=10, nprobes=4)[1]
    pl = pl[np.isfinite(pl)]
    lo = np.full(nq, np.nan, np.float32)
    hi = np.where(rng.random(nq) < 0.4, np.float32(np.quantile(pl, 0.5)), np.nan).astype(np.float32) if ranged \
        else np.full(nq, np.nan, np.float32)
    hnsw = kind.startswith("hnsw")
    ef = np.where(rng.random(nq) < 0.5, k * np.maximum(rf, 1) + 7, 0) if hnsw else np.zeros(nq, np.int64)
    vec = _queries(ix, data)
    gi, gd, gc, gn = ix.search_batch(_queries(ix, q), k, nprobes=nprobes, minimum_nprobes=mins,
                                     maximum_nprobes=maxs, refine_factor=rf, vectors=vec, filters=filters,
                                     filter_of=fof, lower_bound=lo, upper_bound=hi, ef=ef if hnsw else None,
                                     late_width=2)
    K = 24
    for i in range(nq):
        qi = _queries(ix, q[i:i + 1])
        h = None if np.isnan(hi[i]) else float(hi[i])
        f = None if fof[i] < 0 else filters[fof[i]]
        ki = int(k[i])
        if nprobes[i]:
            bm = None if f is None else np.ascontiguousarray(f[0], np.uint64)
            wi, wd, wc = _single(ix, qi, ki, int(nprobes[i]), int(rf[i]), vec, bm, None, h,
                                 int(ef[i]) if ef[i] else None)
            wn = min(int(nprobes[i]), K)
        else:
            ff = None if f is None else (np.ascontiguousarray(f[0], np.uint64), f[1], f[2])
            wi, wd, wc, wn = _single_probed(ix, qi, ki, int(mins[i]), int(maxs[i]), int(rf[i]), vec, ff, None, h,
                                            int(ef[i]) if ef[i] else None, 2)
        assert np.array_equal(gi[i, :ki], wi), i
        assert np.array_equal(gd[i, :ki].view(np.uint32), wd.view(np.uint32)), i
        assert gc[i] == wc and gn[i] == wn, (i, gc[i], wc, gn[i], wn)


@pytest.mark.parametrize("metric", ["l2", "cosine", "dot"])
@pytest.mark.parametrize("mix", ["fast", "mixed"])
def test_fast_routes_with_mixed_k_and_filters(metric, mix):
    """IVF_PQ 8-bit: a whole batch on the fast routes (k' + 1 <= 16), or fast and radix queries in one batch, with
    mixed k', filters, ranges and duplicate rows, under the classic and the skewed kernel"""
    data = _data(6000, 128, 17, dup=0.1)
    ix = _build("pq8", data, 16, metric)
    e = ix.export()
    rng = np.random.default_rng(23)
    nq = 300
    q = _data(nq, 128, 18)
    filters = _filters(ix, e, rng)
    k = rng.integers(1, 16, nq)
    rf = np.where((rng.random(nq) < 0.3) & (k <= 7), 2, 0)
    if mix == "mixed":
        big = rng.random(nq) < 0.3
        k[big], rf[big] = rng.integers(16, 80, big.sum()), 0
    nprobes = rng.integers(1, 19, nq)
    fof = rng.integers(-1, 4, nq)
    pl = ix.search_ex(q[:16], k=10, nprobes=4)[1]
    pl = pl[np.isfinite(pl)]
    lo = np.where(rng.random(nq) < 0.15, np.float32(np.quantile(pl, 0.05)), np.nan).astype(np.float32)
    hi = np.where(rng.random(nq) < 0.15, np.float32(np.quantile(pl, 0.7)), np.nan).astype(np.float32)
    params = (k, nprobes, rf, fof, lo, hi, np.zeros(nq, np.int64))
    old = os.environ.get("LB2_SCAN")
    try:
        for scan in ("classic", "skew"):
            os.environ["LB2_SCAN"] = scan
            got = ix.search_batch(q, k, nprobes=nprobes, refine_factor=rf, vectors=data, filters=filters,
                                  filter_of=fof, lower_bound=lo, upper_bound=hi)
            _check_rows(ix, q, data, filters, got, params, int(k.max()))
    finally:
        if old is None:
            os.environ.pop("LB2_SCAN", None)
        else:
            os.environ["LB2_SCAN"] = old


def test_mixed_routes_launch_once_per_route():
    """fast and radix queries in one batch: the scan launches once per route present, whatever the parameter sets"""
    data = _data(6000, 128, 5)
    ix = _build("pq8", data, 32, "l2")
    rng = np.random.default_rng(3)
    nq = 400
    q = _data(nq, 128, 6)
    k = np.where(np.arange(nq) % 2 == 0, rng.integers(1, 16, nq), rng.integers(16, 100, nq))
    lb.profile.enable(True)
    try:
        lb.profile.reset()
        ix.search_batch(q, k, nprobes=rng.integers(1, 11, nq))
        names = lb.profile.dump()
    finally:
        lb.profile.enable(False)
    scans = {n: v for n, v in names.items() if "pq_scan" in n and "tie_replay" not in n}
    assert sum(v[0] if isinstance(v, (tuple, list)) else v["launches"] for v in scans.values()) == 2, names
