"""Mixed query batches and the probe rule past every memory-bounded piece of the query path, bit for bit against
one-query calls and the restatements (ids, distance bits, counts, nprobes_out).

A batch holds its work in pieces, and every piece after the first finds its own queries' entries through an offset:
  1. the fixed-nprobes skeleton's candidate sub-slabs (ivf_search.cu: merge with qp_at(a));
  2. the probe rule's ranking slabs (qpr + q0, nprobes_out + q0) and its sub-slabs, with ranges scanned first
     (qpr + a, nprobes_out + a, the shortcut's slots, qp_at(q0 + a));
  3. IVF_PQ 8-bit route groups per 32 768-query scan slab (qp_host[sl.q0 + q] and the reused glist);
  4. IVF_RQ rotation groups in a batch (qp_at(sl.q0 + a));
  5. knn_combined's batch merge with rows of k_stride > 1024 (merge_kernel, where every single query takes the rank
     kernel), and search_batch's padding past the largest k.
Each case restates its loop's size rule, asserts that it crosses at least two boundaries, confirms the number of
pieces from launch counts, and gives neighbouring pieces different per-query parameters: a wrong offset makes a
query read another query's k', filter, range or probe bounds."""
import numpy as np
import pytest

import flat_reference as fr
import lance_b200 as lb
from test_combined_batch import _bits, _opt, _same_row
from test_combined_batch import _build as _combined_build
from test_probed_search import _expected
from test_rq_sq_routes import _group_size, _launches, _profiled, _rq_index
from test_search_batch import _build, _check_rows, _data, _filters, _single, _single_probed

pytestmark = pytest.mark.gpu

U64MAX = np.uint64(0xFFFFFFFFFFFFFFFF)
PIECE_BYTES = 256 << 20   # candidate sub-slabs, ranking slabs and rotation groups: about 256 MB each
SLAB = 32768              # SEARCH_SLAB: queries per scan launch (the grid.y limit), and the ranking slab's cap
RANK_TILE = 8192          # partitions one block ranks in shared memory (probe.cuh)
MERGE_RANK_MAX = 2048     # candidates merge_lists merges by rank counting; more take merge_kernel
SCAN_KFAST = 16           # IVF_PQ 8-bit: k' + 1 <= SCAN_KFAST takes the fast kernels


# ---- the restated size rules --------------------------------------------------------------------------------------
def _candidate_sub(nq, np_, kc):
    """queries per candidate sub-slab: np_ lists of kc (distance, id) pairs, their count, and a probe id per slot"""
    return max(1, min(nq, PIECE_BYTES // (np_ * kc * 12 + 4 * np_)))


def _ranking_slab(K, L):
    """queries per ranking slab of the probe rule: the distances, two runs of packed words above one tile, L probes"""
    return max(1, min(SLAB, PIECE_BYTES // (K * (20 if K > RANK_TILE else 4) + 8 * L)))


def _pieces(a, b, size):
    return [(s, min(b, s + size)) for s in range(a, b, size)]


def _near(bounds, nq, width, rng, extra):
    """every query within `width` of a boundary, plus `extra` more drawn at random"""
    near = [i for b in bounds for i in range(b - width, b + width) if 0 <= i < nq]
    return np.unique(np.concatenate([near, rng.choice(nq, extra, replace=False)]).astype(np.int64))


def _profiled_call(fn):
    box = []
    prof = _profiled(lambda: box.append(fn()))
    return box[0], prof


def _with_scan(monkeypatch, scan):
    if scan is None:
        monkeypatch.delenv("LB2_SCAN", raising=False)
    else:
        monkeypatch.setenv("LB2_SCAN", scan)


# ---- 1. fixed-nprobes candidate sub-slabs, every kind ------------------------------------------------------------
K1, NQ1 = 1024, 150
HEAVY = 4           # partitions of 700 rows: the k' = 512 lists fill and are cut
KINDS1 = ["flat", "flat_f16", "sq", "pq8-classic", "pq8-skew", "pq4", "rq", "hnsw_sq", "hnsw_pq", "hnsw_flat"]


def _slab_data(d, seed):
    """K1 well-separated centres: 4 with 700 rows each, the others with 15; the centres seed a single Lloyd step,
    so every build keeps those partitions"""
    rng = np.random.default_rng(seed)
    cent = (rng.standard_normal((K1, d)) * 6).astype(np.float32)
    sizes = np.full(K1, 15)
    sizes[rng.choice(K1, HEAVY, replace=False)] = 700
    part = np.repeat(np.arange(K1), sizes)
    x = (cent[part] + 0.5 * rng.standard_normal((len(part), d))).astype(np.float32)
    perm = rng.permutation(len(part))
    return cent, part[perm].astype(np.uint32), x[perm]


def _slab_index(kind):
    d = 128 if kind == "pq8" else 16
    cent, part, x = _slab_data(d, 3)
    hp = lb.HnswBuildParams(m=8, ef_construction=40)
    if kind == "flat_f16":   # the build takes f32 initial centroids: open the 16-bit index from its parts instead
        col = x.astype(np.float16)
        return lb.IvfFlatIndex.from_parts(cent.astype(np.float16), part, col), col, cent
    if kind in ("pq8", "pq4", "hnsw_pq"):
        p = lb.IvfBuildParams(num_partitions=K1, num_sub_vectors=16 if d == 128 else 8,
                              num_bits=4 if kind == "pq4" else 8, max_iters=1, pq_max_iters=2, seed=1, centroids=cent)
        if kind == "hnsw_pq":
            return lb.IvfHnswPqIndex.build(x, "l2", p, hp), x, cent
        return lb.IvfPqIndex.build(x, "l2", p), x, cent
    b = {"flat": lb.IvfFlatIndex, "sq": lb.IvfSqIndex, "rq": lb.IvfRqIndex, "hnsw_sq": lb.IvfHnswSqIndex,
         "hnsw_flat": lb.IvfHnswFlatIndex}[kind]
    kw = {"hnsw_params": hp} if kind.startswith("hnsw") else {}
    return b.build(x, "l2", num_partitions=K1, max_iters=1, seed=1, centroids=cent, **kw), x, cent


@pytest.fixture(scope="module")
def slab_indexes():
    return {}


def _slab_params(ix, cent, col, rng, hnsw):
    """per-query k, refine factor, filter, range, nprobes (up to 2K) and ef; the queries that set the batch's largest
    k' = 512 and np = K sit in the second, third and fourth sub-slab"""
    nq = NQ1
    near = rng.integers(0, K1, nq)
    q = (cent[near] + 0.7 * rng.standard_normal(cent[near].shape)).astype(np.float32)
    k = rng.integers(1, 101, nq)
    rf = np.where(rng.random(nq) < 0.4, rng.integers(1, 6, nq), 0)
    nprobes = rng.integers(1, 40, nq)
    for i, kk, r in ((60, 512, 0), (100, 64, 8), (130, 128, 4)):   # k' = 512
        k[i], rf[i], nprobes[i] = kk, r, K1 + 1
    nprobes[[50, 95, 140]] = (K1 + 7, K1, 2 * K1)
    fof = rng.integers(-1, 4, nq)
    pl = ix.search_ex(q[:16].astype(col.dtype), k=10, nprobes=4)[1]
    pl = pl[np.isfinite(pl)]
    lo = np.where(rng.random(nq) < 0.15, np.float32(np.quantile(pl, 0.02)), np.nan).astype(np.float32)
    hi = np.where(rng.random(nq) < 0.15, np.float32(np.quantile(pl, 0.6)), np.nan).astype(np.float32)
    ef = np.zeros(nq, np.int64)
    if hnsw:
        kc = k * np.maximum(rf, 1)
        ef = np.where(rng.random(nq) < 0.5, kc + rng.integers(0, 40, nq), 0)
    return q, (k, nprobes, rf, fof, lo, hi, ef)


@pytest.mark.parametrize("case", KINDS1)
def test_fixed_nprobes_sub_slabs(case, slab_indexes, monkeypatch):
    kind, _, scan = case.partition("-")
    _with_scan(monkeypatch, scan or None)
    if kind not in slab_indexes:
        slab_indexes[kind] = _slab_index(kind)
    ix, col, cent = slab_indexes[kind]
    e = ix.export()
    sizes = np.diff(e["part_offsets"].astype(np.int64))
    assert (sizes >= 600).sum() >= 2, sorted(sizes)[-8:]
    rng = np.random.default_rng(7 + KINDS1.index(case))
    hnsw = kind.startswith("hnsw")
    q, params = _slab_params(ix, cent, col, rng, hnsw)
    k, nprobes, rf, fof, lo, hi, ef = params
    q = q.astype(col.dtype)
    filters = _filters(ix, e, rng)
    kc = k * np.maximum(rf, 1)
    np_, kcmax = int(np.minimum(nprobes, K1).max()), int(kc.max())
    assert (np_, kcmax) == (K1, 512)
    sub = _candidate_sub(NQ1, np_, kcmax)
    assert sub == 42
    pieces = _pieces(0, NQ1, sub)
    assert len(pieces) >= 3
    anchors = {i // sub for i in range(NQ1) if kc[i] == kcmax or nprobes[i] >= K1}
    assert len(anchors) >= 3 and 0 not in anchors
    got, prof = _profiled_call(lambda: ix.search_batch(q, k, nprobes=nprobes, refine_factor=rf, vectors=col,
                                                       filters=filters, filter_of=fof, lower_bound=lo,
                                                       upper_bound=hi, ef=ef if hnsw else None))
    assert _launches(prof, "merge_topk") == len(pieces), prof
    _check_rows(ix, q, col, filters, got, params, int(k.max()))


# ---- 2. probe-rule ranking slabs and ranged sub-slabs ------------------------------------------------------------
K2, N2, D2, NQ2 = 9000, 30000, 8, 2300
LATE = 2


@pytest.fixture(scope="module", params=["flat", "sq"])
def wide_model(request):
    """K = 9000 partitions (above RANK_TILE: tiled ranking and its merge) of about 3 rows over d = 8"""
    rng = np.random.default_rng(90)
    cent = rng.standard_normal((K2, D2)).astype(np.float32)
    part = rng.integers(0, K2, N2).astype(np.uint32)
    x = (cent[part] + 0.05 * rng.standard_normal((N2, D2))).astype(np.float32)
    if request.param == "flat":
        ix = lb.IvfFlatIndex.from_parts(cent, part, x)
    else:
        codes = np.clip(np.rint((x + 4.0) * (255.0 / 8.0)), 0, 255).astype(np.uint8)
        ix = lb.IvfSqIndex.from_parts(cent, (-4.0, 4.0), part, codes)
    e = ix.export()
    rid = e["row_ids"]
    half = np.sort(rng.choice(rid, len(rid) // 2, replace=False))
    sel = np.sort(rng.choice(rid, 30, replace=False))
    blocked = rng.choice(rid, len(rid) // 3, replace=False)
    # (bitmap, max_len, mask_ids) as search_batch takes it, and the allowed row ids the restatement takes
    specs = [((ix.row_mask(None, blocked), None, None), np.setdiff1d(rid, blocked)),
             ((ix.row_mask(half, None), len(half), half), half),
             ((ix.row_mask(sel, None), len(sel), sel), sel),
             ((ix.row_mask(sel, None), len(sel), None), sel),
             ((ix.row_mask(np.zeros(0, np.uint64), None), 0, np.zeros(0, np.uint64)), np.zeros(0, np.uint64))]
    q = (cent[rng.integers(0, K2, NQ2)] + 0.3 * rng.standard_normal((NQ2, D2))).astype(np.float32)
    return request.param, ix, e, x, q, specs


def _wide_params(nq, rng, ranged, pl):
    """per ranking slab s, the probe bounds stay below caps[s] and one fixed query sits at it, so each slab reads back
    its own largest count; the largest k' = 100 sits in the second and third slab"""
    qs = _ranking_slab(K2, K2)
    caps = (K2, 200, 40)
    k = rng.integers(1, 61, nq)
    rf = np.where(rng.random(nq) < 0.3, rng.integers(1, 6, nq), 0)
    rf = np.where(k * np.maximum(rf, 1) > 100, 0, rf)
    mins = rng.integers(1, 6, nq)
    nprobes = np.where(rng.random(nq) < 0.7, 0, rng.integers(1, 61, nq))
    maxs = mins + rng.integers(0, 60, nq)
    slab = np.arange(nq) // qs
    cap = np.array(caps)[np.minimum(slab, 2)]
    maxs = np.where((slab == 0) & (rng.random(nq) < 0.3), 0, np.minimum(maxs, cap))   # 0: up to every partition
    nprobes = np.minimum(nprobes, cap)
    for s, at in ((0, 700), (1, qs + 300), (2, 2 * qs + 100)):
        nprobes[at] = K2 + 5 if s == 0 else caps[s]
    k[qs + 500], rf[qs + 500] = 100, 0
    k[2 * qs + 60], rf[2 * qs + 60] = 20, 5
    fof = rng.integers(-1, 5, nq)
    hi = lo = np.full(nq, np.nan, np.float32)
    if ranged:
        hi = np.where(rng.random(nq) < 0.3, np.float32(np.quantile(pl, 0.5)), np.nan).astype(np.float32)
        lo = np.where(rng.random(nq) < 0.1, np.float32(np.quantile(pl, 0.05)), np.nan).astype(np.float32)
    return k, rf, nprobes, mins, maxs, fof, lo, hi


@pytest.mark.parametrize("ranged", [False, True], ids=["cutoff_from_counts", "ranged_by_scan"])
def test_probe_rule_slabs(wide_model, ranged):
    kind, ix, e, x, q, specs = wide_model
    rng = np.random.default_rng(91 + ranged)
    pl = ix.search_ex(q[:16], k=10, nprobes=20)[1]
    k, rf, nprobes, mins, maxs, fof, lo, hi = _wide_params(NQ2, rng, ranged, pl[np.isfinite(pl)])
    filters = [s[0] for s in specs]
    kc = k * np.maximum(rf, 1)
    kcmax = int(kc.max())
    L = K2   # some query has maximum None or nprobes >= K
    qs = _ranking_slab(K2, L)
    assert qs == 1065
    assert kcmax == 100 and {i // qs for i in np.nonzero(kc == kcmax)[0]} >= {1, 2}
    slabs = _pieces(0, NQ2, qs)
    assert len(slabs) == 3
    got, prof = _profiled_call(lambda: ix.search_batch(q, k, nprobes=nprobes, minimum_nprobes=mins,
                                                       maximum_nprobes=maxs, refine_factor=rf, vectors=x,
                                                       filters=filters, filter_of=fof, lower_bound=lo, upper_bound=hi,
                                                       late_width=LATE))
    gi, gd, gc, gn = got
    extra = 1   # some probe-rule query has an iterable allow list: every query gets a shortcut slot
    if ranged:  # every query scans its L partitions first
        nls = [L + extra] * len(slabs)
    else:       # the slab's largest count, read back: different in every slab
        nls = [int(gn[a:b].max()) + extra for a, b in slabs]
        assert nls == [K2 + 1, 201, 41], nls
    subs = [_pieces(a, b, _candidate_sub(b - a, nl, kcmax)) for (a, b), nl in zip(slabs, nls)]
    assert sum(len(s) for s in subs) >= 3
    if ranged:
        assert [_candidate_sub(b - a, nl, kcmax) for (a, b), nl in zip(slabs, nls)] == [24, 24, 24]
    assert _launches(prof, "rank_probes") == len(slabs) and _launches(prof, "rank_probes_merge") == len(slabs), prof
    assert _launches(prof, "merge_topk") == sum(len(s) for s in subs), prof
    assert _launches(prof, "probe_cutoff") == (sum(len(s) for s in subs) if ranged else len(slabs)), prof
    bounds = [a for a, _ in slabs[1:]] + [a for s in subs for a, _ in s[1:]]
    sel = _near(bounds, NQ2, 16, rng, 100)
    for i in sel:
        ki = int(k[i])
        f = None if fof[i] < 0 else filters[fof[i]]
        if nprobes[i]:
            bm = None if f is None else np.ascontiguousarray(f[0], np.uint64)
            wi, wd, wc = _single(ix, q[i:i + 1], ki, int(nprobes[i]), int(rf[i]), x, bm, _opt(lo[i]), _opt(hi[i]),
                                 None)
            wn = min(int(nprobes[i]), K2)
        else:
            ff = None if f is None else (np.ascontiguousarray(f[0], np.uint64), f[1], f[2])
            wi, wd, wc, wn = _single_probed(ix, q[i:i + 1], ki, int(mins[i]), int(maxs[i]), int(rf[i]), x, ff,
                                            _opt(lo[i]), _opt(hi[i]), None, LATE)
        assert np.array_equal(gi[i, :ki], wi), i
        assert np.array_equal(gd[i, :ki].view(np.uint32), wd.view(np.uint32)), i
        assert (gc[i], gn[i]) == (wc, wn), (i, gc[i], wc, gn[i], wn)
    # the restated rule followed by the reference search, for the unrefined queries without a range at the slab edges
    ref = [i for i in _near([a for a, _ in slabs[1:]], NQ2, 16, rng, 0) if rf[i] == 0 and np.isnan(lo[i])
           and np.isnan(hi[i])]
    assert len(ref) >= 24
    for i in ref:
        ki = int(k[i])
        (_, max_len, mask_ids), allow = specs[fof[i]] if fof[i] >= 0 else ((None, None, None), None)
        if nprobes[i]:
            mn, mx, max_len, mask_ids = int(nprobes[i]), int(nprobes[i]), None, None
        else:
            mn, mx = int(mins[i]), int(maxs[i]) or None
        wi, wd, wc, wn = _expected(kind, e, "l2", q[i:i + 1], ki, mn, mx, LATE, allow=allow, max_len=max_len,
                                   mask_ids=mask_ids)
        assert (gc[i], gn[i]) == (wc[0], wn[0]), (i, gc[i], wc[0], gn[i], wn[0])
        assert np.array_equal(gi[i, :gc[i]], wi[0, :gc[i]]), i
        assert np.array_equal(gd[i, :gc[i]].view(np.uint32), wd[0, :gc[i]].view(np.uint32)), i


def test_search_probed_ranged_sub_slabs(wide_model):
    """lb2_index_search_probed shares the loops: uniform parameters with a range scan every query's K partitions
    first, and the iterable allow list adds the shortcut slot"""
    kind, ix, e, x, q, specs = wide_model
    rng = np.random.default_rng(93)
    (bm, max_len, mask_ids), _ = specs[1]
    pl = ix.search_ex(q[:16], k=10, nprobes=20)[1]
    hi = float(np.quantile(pl[np.isfinite(pl)], 0.5))
    k, rf = 10, 3
    kw = dict(minimum_nprobes=2, maximum_nprobes=None, late_width=LATE, allow_bitmap=bm, mask_ids=mask_ids,
              mask_max_len=max_len, refine_factor=rf, vectors=x, upper_bound=hi)
    slabs = _pieces(0, NQ2, _ranking_slab(K2, K2))
    subs = [_pieces(a, b, _candidate_sub(b - a, K2 + 1, k * rf)) for a, b in slabs]
    assert len(slabs) == 3 and [len(s) for s in subs] == [14, 14, 3]
    got, prof = _profiled_call(lambda: ix.search_probed(q, k, **kw))
    assert _launches(prof, "rank_probes") == len(slabs), prof
    assert _launches(prof, "merge_topk") == _launches(prof, "probe_cutoff") == sum(len(s) for s in subs), prof
    bounds = [a for a, _ in slabs[1:]] + [a for s in subs for a, _ in s[1:]]
    for i in _near(bounds, NQ2, 16, rng, 100):
        want = ix.search_probed(q[i:i + 1], k, **kw)
        for g, w in zip(got, want):   # ids, distance bits, counts, nprobes
            assert np.array_equal(np.ascontiguousarray(g[i:i + 1]).view(np.uint8), w.view(np.uint8)), i


# ---- 3. IVF_PQ route groups past one query slab ------------------------------------------------------------------
# (k, refine factor, nprobes, filter, lower, upper): fast unfiltered; fast filtered; fast ranged; k' = 15 (the last
# k' of the fast kernels); radix; radix with refine
PQ_SETS = [(10, 0, 4, -1, None, None), (8, 0, 6, 1, None, None), (12, 0, 8, -1, None, 0.6), (5, 3, 5, 0, None, None),
           (40, 0, 7, 1, 0.02, None), (15, 4, 3, -1, None, None)]


def _pq_route(s):
    k, rf, _, f, lo, hi = PQ_SETS[s]
    if k * max(rf, 1) + 1 > SCAN_KFAST:
        return 2
    return 1 if (f >= 0 or lo is not None or hi is not None) else 0


@pytest.fixture(scope="module")
def pq_route_index():
    data = _data(6000, 128, 5)
    ix = _build("pq8", data, 32, "l2")
    return ix, ix.export(), data


@pytest.mark.parametrize("scan", ["classic", "skew"])
def test_pq_route_groups_past_one_slab(pq_route_index, scan, monkeypatch):
    _with_scan(monkeypatch, scan)
    ix, e, data = pq_route_index
    rng = np.random.default_rng(31)
    nq = SLAB + 3000
    q = _data(nq, 128, 6)
    filters = _filters(ix, e, rng)
    pl = ix.search_ex(q[:16], k=10, nprobes=4)[1]
    pl = pl[np.isfinite(pl)]
    # every set in the first slab; the second has no fast unfiltered query, so its glist offsets shift
    sets = np.concatenate([rng.integers(0, len(PQ_SETS), SLAB),
                           rng.choice([s for s in range(len(PQ_SETS)) if _pq_route(s) != 0], nq - SLAB)])
    k, rf, nprobes, fof = (np.array([PQ_SETS[s][j] for s in sets]) for j in range(4))
    lo = np.array([np.nan if PQ_SETS[s][4] is None else np.quantile(pl, PQ_SETS[s][4]) for s in sets], np.float32)
    hi = np.array([np.nan if PQ_SETS[s][5] is None else np.quantile(pl, PQ_SETS[s][5]) for s in sets], np.float32)
    kc = k * np.maximum(rf, 1)
    sub = _candidate_sub(nq, int(nprobes.max()), int(kc.max()))
    slabs = [p for a, b in _pieces(0, nq, sub) for p in _pieces(a, b, SLAB)]
    assert len(slabs) == 2
    routes = [sorted({_pq_route(s) for s in sets[a:b]}) for a, b in slabs]
    assert routes == [[0, 1, 2], [1, 2]], routes
    got, prof = _profiled_call(lambda: ix.search_batch(q, k, nprobes=nprobes, refine_factor=rf, vectors=data,
                                                       filters=filters, filter_of=fof, lower_bound=lo,
                                                       upper_bound=hi))
    scans = sum(v[0] for n, v in prof.items() if "pq_scan" in n and "tie_replay" not in n)
    assert scans == sum(len(r) for r in routes) == 5, prof
    gi, gd, gc, gn = got
    assert (gn == nprobes).all()
    for s, (ks, r, p, f, _, _) in enumerate(PQ_SETS):
        sel = np.nonzero(sets == s)[0]
        wi, wd = ix.search_ex(q[sel], k=ks, nprobes=p, allow_bitmap=None if f < 0 else filters[f], refine_factor=r,
                              vectors=data, lower_bound=_opt(lo[sel[0]]), upper_bound=_opt(hi[sel[0]]))
        assert np.array_equal(gi[sel, :ks], wi), s
        assert np.array_equal(gd[sel, :ks].view(np.uint32), wd.view(np.uint32)), s
        assert np.array_equal(gc[sel], (wi != U64MAX).sum(1)), s
        assert (gi[sel, ks:] == U64MAX).all() and np.isposinf(gd[sel, ks:]).all(), s


# ---- 4. IVF_RQ rotation groups in a batch ------------------------------------------------------------------------
RQ_SIZES = (0, 31, 32, 33, 40, 64, 65, 100, 1, 96, 97, 0, 31, 128, 200, 33)


@pytest.fixture(scope="module")
def wide_rq():
    return _rq_index(16, 512, "l2", sizes=RQ_SIZES, seed=56)


@pytest.mark.parametrize("rule", [False, True], ids=["fixed", "probe_rule"])
def test_rq_rotation_groups_in_a_batch(wide_rq, rule):
    """d = 16, code_dim 8192, 8 of 16 partitions: groups of 1022 queries, three in 2100"""
    d, nb, nq = 16, 512, 2100
    ix, m = wide_rq
    K, n = len(RQ_SIZES), int(sum(RQ_SIZES))
    rng = np.random.default_rng(57 + rule)
    vec = rng.standard_normal((n, d)).astype(np.float32)   # the refine column (row ids are 0 .. n - 1)
    q = rng.standard_normal((nq, d)).astype(np.float32)
    filters = _filters(ix, {"row_ids": m[6]}, rng)
    pl = ix.search_ex(q[:16], k=10, nprobes=4)[1]
    pl = pl[np.isfinite(pl)]
    k = rng.integers(1, 60, nq)
    rf = np.where(rng.random(nq) < 0.4, rng.integers(1, 5, nq), 0)
    fof = rng.integers(-1, 4, nq)
    lo = np.where(rng.random(nq) < 0.15, np.float32(np.quantile(pl, 0.05)), np.nan).astype(np.float32)
    hi = np.where(rng.random(nq) < 0.2, np.float32(np.quantile(pl, 0.6)), np.nan).astype(np.float32)
    nprobes = rng.integers(1, 9, nq)
    mins = rng.integers(1, 5, nq)
    maxs = np.minimum(8, mins + rng.integers(0, 6, nq))
    if rule:   # every query's bounds at most 8; a range scans each query's L = 8 partitions first
        nprobes = np.where(rng.random(nq) < 0.7, 0, nprobes)
        maxs[[40, 1100, 2080]] = 8
        hi[1100] = np.quantile(pl, 0.6)
    nprobes[[30, 1500, 2090]] = 8
    np_ = 8
    qc = _group_size(np_, d, d * nb, min(nq, SLAB))
    groups = _pieces(0, nq, qc)
    assert qc == 1022 and len(groups) == 3
    got, prof = _profiled_call(lambda: ix.search_batch(q, k, nprobes=nprobes, minimum_nprobes=mins,
                                                       maximum_nprobes=maxs, refine_factor=rf, vectors=vec,
                                                       filters=filters, filter_of=fof, lower_bound=lo,
                                                       upper_bound=hi))
    assert _launches(prof, "rq_query_residual") == _launches(prof, "rq_scan") == len(groups), prof
    gi, gd, gc, gn = got
    for i in _near([a for a, _ in groups[1:]], nq, 16, rng, 150):
        ki = int(k[i])
        bm = None if fof[i] < 0 else np.ascontiguousarray(filters[fof[i]], np.uint64)
        if nprobes[i]:
            wi, wd, wc = _single(ix, q[i:i + 1], ki, int(nprobes[i]), int(rf[i]), vec, bm, _opt(lo[i]), _opt(hi[i]),
                                 None)
            wn = min(int(nprobes[i]), K)
        else:
            wi, wd, wc, wn = _single_probed(ix, q[i:i + 1], ki, int(mins[i]), int(maxs[i]), int(rf[i]), vec,
                                            None if bm is None else (bm, None, None), _opt(lo[i]), _opt(hi[i]), None,
                                            1)
        assert np.array_equal(gi[i, :ki], wi), i
        assert np.array_equal(gd[i, :ki].view(np.uint32), wd.view(np.uint32)), i
        assert (gc[i], gn[i]) == (wc, wn), (i, gc[i], wc, gn[i], wn)


# ---- 5. knn_combined rows past the rank merge, and against flat KNN ----------------------------------------------
KS5 = 1031   # output row length: 2 * KS5 candidates per query leave the rank-counting merge


@pytest.mark.parametrize("kind,metric", [("flat", "l2"), ("flat", "dot"), ("sq", "l2")])
def test_combined_rows_past_rank_merge(kind, metric):
    n1, n2, K, nq, d = 3000, 700, 16, 48, 32
    x = _data(n1 + n2, d, 71)
    col, ucol = x[:n1], x[n1:]
    ix = _combined_build(kind, col, metric, "f32", K)
    rng = np.random.default_rng(72)
    q = _data(nq, d, 73)
    urid = np.arange(n1, n1 + n2, dtype=np.uint64)
    k = rng.integers(1, 1025, nq)
    k[[5, 30, 47]] = 1024
    rf = np.where((rng.random(nq) < 0.5) & (k <= 256), rng.integers(1, 5, nq), 0)
    rf[30] = 1
    nprobes = np.where(rng.random(nq) < 0.5, K, K + 3)
    # filters as row-id masks: the index's over its rows, the unindexed half's over the others
    masks = [rng.random(n1) < 0.6, rng.random(n1) < 0.1, np.zeros(n1, bool)]
    umasks = [rng.random(n2) < 0.7, rng.random(n2) < 0.5, np.zeros(n2, bool)]
    uvalid = rng.random(n2) < 0.9
    filters = [ix.row_mask(np.nonzero(mk)[0].astype(np.uint64), None) for mk in masks]
    fof = rng.integers(-1, len(masks), nq)
    dist = fr.distances(q, x, metric, "f32")
    lo = np.where(rng.random(nq) < 0.2, np.float32(np.quantile(dist, 0.01)), np.nan).astype(np.float32)
    hi = np.where(rng.random(nq) < 0.2, np.float32(np.quantile(dist, 0.4)), np.nan).astype(np.float32)
    assert 2 * KS5 > MERGE_RANK_MAX >= 2 * int(k.max())   # the batch merges by merge_kernel, one query by rank
    out = (np.full((nq, KS5), 7, np.uint64), np.full((nq, KS5), 7, np.float32))
    got, prof = _profiled_call(lambda: ix.search_combined_batch(
        q, k, vectors=col, unindexed_vectors=ucol, unindexed_row_ids=urid, nprobes=nprobes, refine_factor=rf,
        filters=filters, filter_of=fof, unindexed_allow_bitmap=_bits(uvalid),
        unindexed_filters=[_bits(u) for u in umasks], lower_bound=lo, upper_bound=hi, out=out))
    assert _launches(prof, "merge_combined") == 1, prof
    gi, gd, gc, gn = got
    assert gi is out[0] and (gn == np.minimum(nprobes, K)).all()
    for i in range(nq):
        f, ki = int(fof[i]), int(k[i])
        want = ix.search_combined(q[i:i + 1], ki, col, ucol, urid, nprobes=int(nprobes[i]), refine_factor=int(rf[i]),
                                  allow_bitmap=filters[f] if f >= 0 else None,
                                  unindexed_allow_bitmap=_bits(umasks[f] if f >= 0 else uvalid),
                                  lower_bound=_opt(lo[i]), upper_bound=_opt(hi[i]))
        _same_row((gi, gd, gc), i, want[:3], (kind, metric))
        if kind != "flat":
            continue
        # every partition probed: exact flat KNN over the whole column under the combined allow bitmap
        allow = np.concatenate([masks[f] if f >= 0 else np.ones(n1, bool), umasks[f] if f >= 0 else uvalid])
        wi, wd, wc = fr.flat_search(x, q[i:i + 1], ki, metric, allow=_bits(allow), lower=_opt(lo[i]),
                                    upper=_opt(hi[i]))
        _same_row((gi, gd, gc), i, (wi, wd, wc), ("flat_search", metric))
    # search_batch with rows longer than its largest k: the tail is padded
    out = (np.full((nq, KS5), 7, np.uint64), np.full((nq, KS5), 7, np.float32))
    params = (k, nprobes, rf, fof, lo, hi, np.zeros(nq, np.int64))
    got = ix.search_batch(q, k, nprobes=nprobes, refine_factor=rf, vectors=col, filters=filters, filter_of=fof,
                          lower_bound=lo, upper_bound=hi, out=out)
    assert got[0] is out[0]
    _check_rows(ix, q, col, filters, got, params, KS5)
