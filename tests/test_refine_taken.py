"""lb2_index_search_candidates + lb2_index_refine_taken: a refined batch over rows the caller takes.  Candidates, a
take of the distinct row ids and the exact re-rank of the taken rows must equal lb2_index_search_batch with the dense
column bit for bit (ids, distance bits, counts, nprobes), on every index kind, element type and metric; and they must
work where the dense column cannot, with sparse 64-bit Lance row ids."""
import ctypes as C

import numpy as np
import pytest

import lance_b200 as lb
from lance_b200 import _lib

pytestmark = pytest.mark.gpu

U64MAX = np.uint64(0xFFFFFFFFFFFFFFFF)
D = 32


def _data(n, d, seed, clusters=12, dup=0.05):
    rng = np.random.default_rng(seed)
    base = rng.standard_normal((clusters, d)).astype(np.float32) * 4
    x = (base[rng.integers(0, clusters, n)] + rng.standard_normal((n, d)).astype(np.float32)).astype(np.float32)
    nd = int(n * dup)  # duplicate rows: ties at the k-th distance
    x[rng.choice(n, nd, replace=False)] = x[rng.choice(n, nd, replace=False)]
    return x


def _typed(x, dt):
    """x in element type dt (bf16: uint16 bit patterns; u8: integer levels)"""
    if dt == "f16":
        return x.astype(np.float16)
    if dt == "bf16":
        return np.ascontiguousarray((x.view(np.uint32) >> 16).astype(np.uint16))
    if dt == "u8":
        return np.clip(np.rint(x * 8 + 128), 0, 255).astype(np.uint8)
    return np.ascontiguousarray(x, np.float32)


def _build(kind, col, metric, dt, K=16, row_ids=None):
    bf16 = dt == "bf16"
    hp = lb.HnswBuildParams(m=8, ef_construction=40) if kind.startswith("hnsw") else None
    if kind in ("pq8", "pq4", "hnsw_pq"):
        p = lb.IvfBuildParams(num_partitions=K, num_sub_vectors=8, num_bits=4 if kind == "pq4" else 8, max_iters=4,
                              pq_max_iters=4, seed=1)
        if kind == "hnsw_pq":
            return lb.IvfHnswPqIndex.build(col, metric, p, hp, row_ids=row_ids, bf16=bf16)
        return lb.IvfPqIndex.build(col, metric, p, row_ids=row_ids, bf16=bf16)
    b = {"flat": lb.IvfFlatIndex, "sq": lb.IvfSqIndex, "rq": lb.IvfRqIndex, "hnsw_sq": lb.IvfHnswSqIndex,
         "hnsw_flat": lb.IvfHnswFlatIndex}[kind]
    kw = {"hnsw_params": hp} if hp is not None else {}
    if kind != "rq":
        kw["bf16"] = bf16
    return b.build(col, metric, num_partitions=K, max_iters=4, seed=1, row_ids=row_ids, **kw)


def _mixed(ix, nq, K, rng, hnsw, rid):
    """a mixed batch: fixed and minimum / maximum nprobes, filters (one with a max_len + mask_ids shortcut), ranges,
    refine factor 0 and > 0, ef on the HNSW kinds"""
    k = rng.integers(1, 31, nq)
    rf = np.where(rng.random(nq) < 0.5, rng.integers(1, 9, nq), 0)
    nprobes = np.where(rng.random(nq) < 0.5, rng.integers(1, K + 3, nq), 0)
    mins = rng.integers(1, 4, nq)
    maxs = np.where(rng.random(nq) < 0.5, 0, mins + rng.integers(0, K, nq))
    few = rng.choice(rid, 6, replace=False)
    filters = [ix.row_mask(None, rng.choice(rid, len(rid) // 3, replace=False)),       # a block list
               ix.row_mask(rng.choice(rid, len(rid) // 2, replace=False), None),       # an allow list, ~50 %
               (ix.row_mask(few, None), len(few), few),                                  # the shortcut: max_len <= k
               ix.row_mask(np.zeros(0, np.uint64), None)]                                # an empty allow list
    fof = rng.integers(-1, len(filters), nq)
    fof[:8] = 2  # selective probe-rule queries that reach the shortcut
    nprobes[:8], k[:8] = 0, rng.integers(6, 20, 8)
    lo = np.where(rng.random(nq) < 0.15, np.float32(0.5), np.nan).astype(np.float32)
    hi = np.where(rng.random(nq) < 0.15, np.float32(1e4), np.nan).astype(np.float32)
    ef = np.zeros(nq, np.int64)
    if hnsw:
        kc = k * np.maximum(rf, 1)
        ef = np.where(rng.random(nq) < 0.5, kc + rng.integers(0, 40, nq), 0)
    return dict(k=k, nprobes=nprobes, minimum_nprobes=mins, maximum_nprobes=maxs, refine_factor=rf, filters=filters,
                filter_of=fof, lower_bound=lo, upper_bound=hi, ef=ef)


def _same(got, want):
    gi, gd, gc = got[:3]
    wi, wd, wc = want[:3]
    assert np.array_equal(gi, wi)
    assert np.array_equal(gd.view(np.uint32), wd.view(np.uint32))
    assert np.array_equal(gc, wc)


def _refine_kw(p):
    return {n: p[n] for n in ("k", "refine_factor", "lower_bound", "upper_bound")}


def _check_distinct(ci, cc, uniq, pos):
    valid = np.arange(ci.shape[1])[None, :] < cc[:, None]
    assert (ci[~valid] == U64MAX).all()
    assert np.array_equal(uniq, np.unique(ci[valid]))
    assert np.array_equal(uniq[pos[valid].astype(np.int64)], ci[valid])
    assert (pos[~valid] == U64MAX).all()


KINDS = ("pq8", "pq4", "flat", "sq", "rq", "hnsw_sq", "hnsw_pq", "hnsw_flat")
CASES = [(kind, dt, m) for kind in KINDS for dt in (("f32",) if kind == "rq" else ("f32", "f16", "bf16", "u8"))
         for m in ("l2", "cosine", "dot")]


@pytest.mark.parametrize("kind,dt,metric", CASES, ids=lambda c: str(c))
def test_candidates_take_refine_equals_search_batch(kind, dt, metric):
    x = _data(3000, D, 7)
    col = _typed(x, dt)
    K = 16
    ix = _build(kind, col, metric, dt, K)
    rid = ix.export()["row_ids"]
    rng = np.random.default_rng(3)
    nq = 120
    q = _typed(_data(nq, D, 8), dt)
    p = _mixed(ix, nq, K, rng, kind.startswith("hnsw"), rid)
    ci, cd, cc, cn, uniq, pos = ix.search_candidates(q, **p, distinct=True)
    _check_distinct(ci, cc, uniq, pos)
    got = ix.refine_taken(q, (ci, cd, cc), col[uniq.astype(np.int64)], pos, **_refine_kw(p))
    want = ix.search_batch(q, **p, vectors=col)
    _same(got, want)
    assert np.array_equal(cn, want[3])
    kc = p["k"] * np.maximum(p["refine_factor"], 1)
    assert (cc <= kc).all()
    # without distinct: the same lists
    ci2, cd2, cc2, cn2 = ix.search_candidates(q, **p)
    assert np.array_equal(ci2, ci) and np.array_equal(cd2.view(np.uint32), cd.view(np.uint32))
    assert np.array_equal(cc2, cc) and np.array_equal(cn2, cn)
    # fixed nprobes: only k' reaches the scan, so the list is search_batch's with k' and refine factor 0
    fx = np.nonzero(p["nprobes"] > 0)[0]
    pf = {n: (v[fx] if isinstance(v, np.ndarray) else v) for n, v in p.items()}
    pf["k"], pf["refine_factor"] = kc[fx], 0
    wi, wd, wc, _ = ix.search_batch(np.ascontiguousarray(q[fx]), **pf)
    kmax = int(kc[fx].max())
    assert np.array_equal(ci[fx, :kmax], wi) and np.array_equal(cd[fx, :kmax].view(np.uint32), wd.view(np.uint32))
    assert np.array_equal(cc[fx], wc)


def _sparse_ids(n, rng):
    """Lance row ids: fragment << 32 | offset over several fragments, with gaps (deleted rows), ids above 2^32"""
    frags, ids, f = [], [], 0
    while sum(len(a) for a in ids) < n:
        f += int(rng.integers(1, 4))
        size = int(rng.integers(300, 900))
        off = np.sort(rng.choice(size + 200, size, replace=False)).astype(np.uint64)
        ids.append((np.uint64(f) << np.uint64(32)) | off)
        frags.append(f)
    return np.concatenate(ids)[:n]


@pytest.mark.parametrize("kind", ["pq8", "flat", "hnsw_sq"])
def test_sparse_row_ids(kind):
    n = 3000
    x = _data(n, D, 5)
    rng = np.random.default_rng(9)
    sid = _sparse_ids(n, rng)
    assert sid.max() > np.uint64(1 << 32) and np.all(np.diff(sid.astype(np.float64)) > 0)
    ix_d = _build(kind, x, "l2", "f32")
    ix_s = _build(kind, x, "l2", "f32", row_ids=sid)
    # the column as Lance stores it: one array per fragment, addressed by offset
    frag = {}
    for i, r in enumerate(sid):
        frag.setdefault(int(r >> np.uint64(32)), {})[int(r & np.uint64(0xFFFFFFFF))] = i
    nq = 100
    q = _data(nq, D, 6)
    p = dict(k=rng.integers(1, 21, nq), nprobes=np.where(rng.random(nq) < 0.5, 4, 0),
             refine_factor=np.where(rng.random(nq) < 0.7, 5, 0), ef=np.zeros(nq, np.int64))
    ci, cd, cc, cn, uniq, pos = ix_s.search_candidates(q, **p, distinct=True)
    taken = np.stack([x[frag[int(r >> np.uint64(32))][int(r & np.uint64(0xFFFFFFFF))]] for r in uniq])
    gi, gd, gc = ix_s.refine_taken(q, (ci, cd, cc), taken, pos, p["k"], p["refine_factor"])
    wi, wd, wc, wn = ix_d.search_batch(q, **p, vectors=x)
    valid = wi != U64MAX
    mapped = np.where(valid, sid[np.where(valid, wi, 0).astype(np.int64)], U64MAX)
    assert np.array_equal(gi, mapped)
    assert np.array_equal(gd.view(np.uint32), wd.view(np.uint32))
    assert np.array_equal(gc, wc) and np.array_equal(cn, wn)
    # the dense refine path reads row id r as row r of the column: with these ids it has no row, and scores NaN
    _, bd, _, _ = ix_s.search_batch(q, **p, vectors=x)
    assert np.isnan(bd[p["refine_factor"] > 0]).any()


def test_taken_memory_kinds():
    x = _data(4000, D, 2)
    ix = _build("flat", x, "cosine", "f32")
    rng = np.random.default_rng(4)
    nq = 200
    q = _data(nq, D, 3)
    p = dict(k=rng.integers(1, 40, nq), nprobes=6, refine_factor=rng.integers(0, 6, nq))
    ci, cd, cc, cn, uniq, pos = ix.search_candidates(q, **p, distinct=True)
    taken = x[uniq.astype(np.int64)]
    want = ix.search_batch(q, **p, vectors=x)
    pinned = lb.PinnedArray(taken.shape, np.float32)
    pinned.array[:] = taken
    dev = lb.DeviceArray.from_numpy(taken)
    dev_pos = lb.DeviceArray.from_numpy(pos)
    dev_c = tuple(lb.DeviceArray.from_numpy(a) for a in (ci, cd, cc))
    for t, ps, c in ((taken, pos, (ci, cd, cc)), (pinned, pos, (ci, cd, cc)), (dev, pos, (ci, cd, cc)),
                     (dev, dev_pos, dev_c), (pinned, dev_pos, (ci, cd, cc))):
        _same(ix.refine_taken(q, c, t, ps, p["k"], p["refine_factor"]), want)
    pinned.free()


def test_taken_rows_past_one_staging_buffer():
    """host rows past the 512 MB staging buffer go in query slabs; the result is the one-copy result"""
    clusters, size, d = 450, 180, 2048
    rng = np.random.default_rng(1)
    centres = rng.standard_normal((clusters, d)).astype(np.float32) * 10
    x = (np.repeat(centres, size, axis=0) + rng.standard_normal((clusters * size, d)).astype(np.float32) * 0.1)
    ix = lb.IvfFlatIndex.build(x, "l2", num_partitions=16, max_iters=2, seed=1)
    q = centres  # each query's candidates: its own cluster, so the batch shares few rows
    nq = len(q)
    k, rf = np.full(nq, 18), np.where(np.arange(nq) % 7 == 0, 0, 10)
    ci, cd, cc, cn, uniq, pos = ix.search_candidates(q, k, nprobes=16, refine_factor=rf, distinct=True)
    taken = x[uniq.astype(np.int64)]
    assert taken.nbytes > (512 << 20), taken.nbytes
    xd = lb.DeviceArray.from_numpy(x)
    want = ix.search_batch(q, k, nprobes=16, refine_factor=rf, vectors=xd)
    _same(ix.refine_taken(q, (ci, cd, cc), taken, pos, k, rf), want)
    pinned = lb.PinnedArray(taken.shape, np.float32)
    pinned.array[:] = taken
    _same(ix.refine_taken(q, (ci, cd, cc), pinned, pos, k, rf), want)
    _same(ix.refine_taken(q, (ci, cd, cc), lb.DeviceArray.from_numpy(taken), pos, k, rf), want)
    pinned.free()


@pytest.mark.parametrize("probed", [False, True])
def test_combined_plan(probed):
    """knn_combined on the new calls: refine_taken with refine factor max(1, rf), flat_search over the unindexed rows,
    and a host merge by (_distance, _rowid) equal search_combined"""
    x = _data(5000, D, 12)
    n1 = 4000
    rid = np.arange(len(x), dtype=np.uint64) * np.uint64(3) + np.uint64(1 << 33)
    ix = _build("pq8", x[:n1], "l2", "f32", row_ids=rid[:n1])
    nq, k, rf = 80, 10, 4
    q = _data(nq, D, 13)
    pk = dict(nprobes=None, minimum_nprobes=1, maximum_nprobes=None) if probed else dict(nprobes=5)
    # the dense index column for search_combined: row id = row number, so an index over row numbers
    ix_dense = _build("pq8", x[:n1], "l2", "f32")
    wi, wd, wc, wn = ix_dense.search_combined(q, k, x[:n1], x[n1:], np.arange(n1, len(x), dtype=np.uint64),
                                              refine_factor=rf, **pk)
    ci, cd, cc, cn, uniq, pos = ix.search_candidates(q, k, refine_factor=rf, **pk, distinct=True)
    by_id = dict(zip(rid[:n1].tolist(), range(n1)))
    taken = x[[by_id[int(r)] for r in uniq]]
    ai, ad, ac = ix.refine_taken(q, (ci, cd, cc), taken, pos, k, max(1, rf))
    ui, ud, uc = lb.flat_search(x[n1:], q, k, "l2", row_ids=rid[n1:])
    to_dense = dict(zip(rid.tolist(), range(len(x))))
    for i in range(nq):
        ids = np.concatenate([ai[i, :ac[i]], ui[i, :uc[i]]])
        ds = np.concatenate([ad[i, :ac[i]], ud[i, :uc[i]]])
        o = np.lexsort((ids, ds))[:k]
        got_i = np.array([to_dense[int(r)] for r in ids[o]], np.uint64)
        assert wc[i] == len(o), i
        assert np.array_equal(got_i, wi[i, :wc[i]]), i
        assert np.array_equal(ds[o].view(np.uint32), wd[i, :wc[i]].view(np.uint32)), i
    if probed:
        assert np.array_equal(cn, wn)


def _raw_candidates(ix, q, cp, kc_stride, filters=None):
    """lb2_index_search_candidates through ctypes on prefilled outputs: (status, outputs)"""
    nq = q.shape[0]
    outs = [np.full((nq, kc_stride), 7, np.uint64), np.full((nq, kc_stride), 7, np.float32),
            np.full(nq, 7, np.uint32), np.full(nq, 7, np.uint32), np.full(nq * kc_stride, 7, np.uint64),
            np.full(1, 7, np.uint64), np.full((nq, kc_stride), 7, np.uint64)]
    cf = (_lib.QueryFilter * 1)() if filters is None else filters
    st = _lib.lib().lb2_index_search_candidates(ix._h, C.c_void_p(q.ctypes.data), C.c_uint64(nq),
                                                C.c_void_p(cp.ctypes.data), cf, C.c_uint32(0), C.c_uint32(1),
                                                C.c_uint32(kc_stride), *[C.c_void_p(o.ctypes.data) for o in outs])
    return st, outs


def test_refusals_write_nothing():
    x = _data(2000, D, 1)
    ix = _build("flat", x, "l2", "f32")
    q = _data(4, D, 2)
    cases = [(dict(k=10, nprobes=4, refine_factor=3), 29, _lib.INVALID_ARG),       # kc_stride below k'
             (dict(k=200, nprobes=4, refine_factor=6), 1200, _lib.UNSUPPORTED),    # k' > 1024
             (dict(k=10, nprobes=4, filter_of=0, filters=[None]), 10, _lib.INVALID_ARG),  # filter 0 of 0 passed
             (dict(k=10, nprobes=4, ef=20), 10, _lib.INVALID_ARG)]                 # ef without graphs
    for kw, stride, want in cases:
        cp = ix._batch_params("t", q, **kw)[4]
        st, outs = _raw_candidates(ix, q, cp, stride)
        assert st == want, (kw, st)
        for o in outs:
            assert (o == 7).all(), kw
    # refine_taken: k' above kc_stride, positions missing, k' > 1024, k_stride below k
    ci, cd, cc, _, uniq, pos = ix.search_candidates(q, 10, nprobes=4, refine_factor=3, distinct=True)
    taken = x[uniq.astype(np.int64)]
    for kw, bad_pos, k_stride, want in ((dict(k=10, refine_factor=4), False, 10, _lib.INVALID_ARG),
                                        (dict(k=10, refine_factor=3), True, 10, _lib.INVALID_ARG),
                                        (dict(k=300, refine_factor=4), False, 300, _lib.UNSUPPORTED),
                                        (dict(k=10, refine_factor=3), False, 9, _lib.INVALID_ARG)):
        cp = ix._batch_params("t", q, kw["k"], 1, refine_factor=kw["refine_factor"])[4]
        oi, od, oc = np.full((4, k_stride), 7, np.uint64), np.full((4, k_stride), 7, np.float32), np.full(4, 7, np.uint32)
        st = _lib.lib().lb2_index_refine_taken(ix._h, C.c_void_p(q.ctypes.data), C.c_uint64(4), C.c_void_p(cp.ctypes.data),
                                               C.c_uint32(30), C.c_void_p(ci.ctypes.data), C.c_void_p(cd.ctypes.data),
                                               C.c_void_p(cc.ctypes.data), C.c_void_p(taken.ctypes.data),
                                               C.c_uint64(len(taken)), None if bad_pos else C.c_void_p(pos.ctypes.data),
                                               C.c_uint32(k_stride), C.c_void_p(oi.ctypes.data),
                                               C.c_void_p(od.ctypes.data), C.c_void_p(oc.ctypes.data))
        assert st == want, (kw, st)
        assert (oi == 7).all() and (od == 7).all() and (oc == 7).all(), kw


def test_position_past_m_scores_nan_last():
    x = _data(2000, D, 1)
    ix = _build("flat", x, "l2", "f32")
    q = _data(3, D, 2)
    ci, cd, cc, _, uniq, pos = ix.search_candidates(q, 8, nprobes=4, refine_factor=1, distinct=True)
    taken = x[uniq.astype(np.int64)]
    pos = pos.copy()
    pos[1, 2] = np.uint64(len(uniq) + 5)
    gi, gd, gc = ix.refine_taken(q, (ci, cd, cc), taken, pos, 8, 1)
    want = ix.search_batch(q, 8, nprobes=4, refine_factor=1, vectors=x)
    for i in (0, 2):
        assert np.array_equal(gi[i], want[0][i]) and np.array_equal(gd[i].view(np.uint32), want[1][i].view(np.uint32))
    assert gc[1] == 8 and np.isnan(gd[1, 7]) and gi[1, 7] == ci[1, 2] and np.isfinite(gd[1, :7]).all()


def test_empty_batch_and_no_refine():
    x = _data(2000, D, 1)
    ix = _build("sq", x, "dot", "f32")
    q0 = np.zeros((0, D), np.float32)
    ci, cd, cc, cn, uniq, pos = ix.search_candidates(q0, 5, nprobes=3, distinct=True)
    assert ci.shape[0] == 0 and len(uniq) == 0
    gi, gd, gc = ix.refine_taken(q0, (ci, cd, cc), np.zeros((0, D), np.float32), pos, 5)
    assert gi.shape[0] == 0 and gc.shape == (0,)
    q = _data(50, D, 2)
    rng = np.random.default_rng(0)
    p = dict(k=rng.integers(1, 30, 50), nprobes=np.where(rng.random(50) < 0.5, 3, 0))
    ci, cd, cc, cn = ix.search_candidates(q, **p)
    got = ix.refine_taken(q, (ci, cd, cc), np.zeros((0, D), np.float32), None, p["k"])
    want = ix.search_batch(q, **p)
    _same(got, want)
    assert np.array_equal(cn, want[3])
