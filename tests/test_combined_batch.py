"""lb2_flat_search_batch and lb2_index_search_combined_batch: flat KNN and knn_combined for batches whose queries
differ in k, range, probes, refine factor and filter.  Row q of either call must equal the single-parameter call for
query q alone bit for bit (ids, distance bits, counts, nprobes), and the number of kernel launches must not grow with
the number of distinct parameter sets."""
import ctypes as C

import numpy as np
import pytest

import lance_b200 as lb
from lance_b200 import _lib

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


def _bits(mask):
    """bool per row -> uint64 words, bit i = row i"""
    bits = np.zeros((len(mask) + 63) // 64 * 64, np.uint8)
    bits[:len(mask)] = mask
    return np.packbits(bits.reshape(-1, 8)[:, ::-1]).view(np.uint64).copy()


def _sparse_ids(n, rng):
    """Lance row ids: fragment << 32 | offset, with gaps, above 2^32"""
    off = np.sort(rng.choice(3 * n, n, replace=False)).astype(np.uint64)
    return (np.uint64(5) << np.uint64(32)) + off


def _same_row(got, i, want, what):
    gi, gd, gc = got[0][i], got[1][i], got[2][i]
    wi, wd, wc = want[0].reshape(-1), want[1].reshape(-1), int(np.asarray(want[2]).reshape(-1)[0])
    kq = len(wi)
    assert gc == wc, (what, i, gc, wc)
    assert np.array_equal(gi[:kq], wi), (what, i)
    assert np.array_equal(gd[:kq].view(np.uint32), wd.view(np.uint32)), (what, i)
    assert (gi[kq:] == U64MAX).all() and np.isposinf(gd[kq:]).all(), (what, i)


def _flat_params(n, nq, rng, kmax=40):
    """per-query k, filters (a random one, an empty bitmap, an all-clear bitmap, a None entry), ranges"""
    filters = [_bits(rng.random(n) < 0.6), _bits(rng.random(n) < 0.1), _bits(np.zeros(n, bool)), None]
    k = rng.integers(1, kmax + 1, nq)
    fof = rng.integers(-1, len(filters), nq)
    lo = np.where(rng.random(nq) < 0.2, np.float32(2.0), np.nan).astype(np.float32)
    hi = np.where(rng.random(nq) < 0.2, np.float32(1e4), np.nan).astype(np.float32)
    return dict(k=k, filters=filters, filter_of=fof, lower_bound=lo, upper_bound=hi)


def _flat_single(col, q, i, p, metric, row_ids=None, bf16=False):
    f = p["filter_of"][i]
    bm = p["filters"][f] if f >= 0 else None
    lo, hi = p["lower_bound"][i], p["upper_bound"][i]
    return lb.flat_search(col, q[i:i + 1], int(p["k"][i]), metric, row_ids=row_ids, allow_bitmap=bm,
                          lower_bound=None if np.isnan(lo) else float(lo),
                          upper_bound=None if np.isnan(hi) else float(hi), bf16=bf16)


# ---------------------------------------------------------------------------------------------------------------
# flat_search_batch
# ---------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["f32", "f16", "bf16", "u8"])
@pytest.mark.parametrize("metric", ["l2", "cosine", "dot"])
@pytest.mark.parametrize("sparse", [False, True])
def test_flat_batch_equals_single(dt, metric, sparse):
    rng = np.random.default_rng(100 + len(dt) + 7 * ("l2", "cosine", "dot").index(metric) + 50 * sparse)
    n, nq = 3000, 70
    x = _data(n, D, 11)
    if dt in ("f32", "f16"):
        x[[5, 77]] = np.inf  # rows whose distances are NaN (inf - inf), sorted after +inf
    col = _typed(x, dt)
    q = _typed(_data(nq, D, 12), dt)
    rid = _sparse_ids(n, rng) if sparse else None
    p = _flat_params(n, nq, rng)
    got = lb.flat_search_batch(col, q, p["k"], metric, row_ids=rid, filters=p["filters"], filter_of=p["filter_of"],
                               lower_bound=p["lower_bound"], upper_bound=p["upper_bound"], bf16=dt == "bf16")
    for i in range(nq):
        _same_row(got, i, _flat_single(col, q, i, p, metric, rid, dt == "bf16"), (dt, metric, sparse))


def _pinned(a):
    p = lb.PinnedArray(a.shape, a.dtype)
    p.array[...] = a
    return p


@pytest.mark.gpu
def test_flat_batch_memory_kinds_chunks_and_slabs(monkeypatch):
    """LB2_CHUNK_ROWS = 1000: a host column of 20 000 rows is staged in 20 chunks, and with k up to 1024 the 1 500
    queries' candidate lists pass one 256 MB query slab; pageable, pinned and device columns give the same rows"""
    rng = np.random.default_rng(200)
    n, nq = 20000, 1500
    x = _data(n, 16, 21)
    q = _data(nq, 16, 22)
    p = _flat_params(n, nq, rng, kmax=1024)
    p["k"][0] = 1024
    monkeypatch.setenv("LB2_CHUNK_ROWS", "1000")
    kw = dict(filters=p["filters"], filter_of=p["filter_of"], lower_bound=p["lower_bound"],
              upper_bound=p["upper_bound"])
    want = lb.flat_search_batch(x, q, p["k"], "l2", **kw)
    for i in range(0, nq, 7):
        _same_row(want, i, _flat_single(x, q, i, p, "l2"), "chunked")
    pin, dev = _pinned(x), lb.DeviceArray.from_numpy(x)
    try:
        for col in (pin, dev):
            got = lb.flat_search_batch(col, q, p["k"], "l2", **kw)
            assert np.array_equal(got[0], want[0]) and np.array_equal(got[1].view(np.uint32), want[1].view(np.uint32))
            assert np.array_equal(got[2], want[2])
    finally:
        pin.free()


@pytest.mark.gpu
def test_flat_batch_empty():
    x = _data(500, D, 1)
    ids, dists, counts = lb.flat_search_batch(x, np.zeros((0, D), np.float32), 5, "l2")
    assert ids.shape[0] == 0 and counts.shape == (0,)
    q = _data(20, D, 2)
    k = np.arange(1, 21)
    ids, dists, counts = lb.flat_search_batch(np.zeros((0, D), np.float32), q, k, "l2",
                                              filters=[np.zeros(0, np.uint64)], filter_of=np.arange(20) % 2 - 1)
    assert (counts == 0).all() and (ids == U64MAX).all() and np.isposinf(dists).all()
    out = (np.full((20, 30), 7, np.uint64), np.full((20, 30), 7, np.float32))
    ids, dists, counts = lb.flat_search_batch(x, q, k, "dot", out=out)
    assert ids is out[0] and (ids[:, 20:] == U64MAX).all()
    for i in range(20):
        _same_row((ids, dists, counts), i, lb.flat_search(x, q[i:i + 1], int(k[i]), "dot"), "out")


# ---------------------------------------------------------------------------------------------------------------
# search_combined_batch
# ---------------------------------------------------------------------------------------------------------------

def _build(kind, col, metric, dt, K=16):
    bf16 = dt == "bf16"
    hp = lb.HnswBuildParams(m=8, ef_construction=40) if kind.startswith("hnsw") else None
    if kind in ("pq8", "pq4", "hnsw_pq"):
        p = lb.IvfBuildParams(num_partitions=K, num_sub_vectors=8, num_bits=4 if kind == "pq4" else 8, max_iters=4,
                              pq_max_iters=4, seed=1)
        if kind == "hnsw_pq":
            return lb.IvfHnswPqIndex.build(col, metric, p, hp, bf16=bf16)
        return lb.IvfPqIndex.build(col, metric, p, bf16=bf16)
    b = {"flat": lb.IvfFlatIndex, "sq": lb.IvfSqIndex, "rq": lb.IvfRqIndex, "hnsw_sq": lb.IvfHnswSqIndex,
         "hnsw_flat": lb.IvfHnswFlatIndex}[kind]
    kw = {"hnsw_params": hp} if hp is not None else {}
    if kind != "rq":
        kw["bf16"] = bf16
    return b.build(col, metric, num_partitions=K, max_iters=4, seed=1, **kw)


def _mixed(ix, nq, K, n1, n2, rng, hnsw):
    """a mixed batch over an index of n1 rows and n2 unindexed rows: fixed and minimum / maximum nprobes, filters (one
    with the max_len + mask_ids shortcut, one empty, one whose unindexed bits are all clear), ranges, refine factor 0
    and > 0, ef on some HNSW queries"""
    rid = np.arange(n1, dtype=np.uint64)
    k = rng.integers(1, 31, nq)
    rf = np.where(rng.random(nq) < 0.5, rng.integers(1, 9, nq), 0)
    nprobes = np.where(rng.random(nq) < 0.5, rng.integers(1, K + 3, nq), 0)
    mins = rng.integers(1, 4, nq)
    maxs = np.where(rng.random(nq) < 0.5, 0, mins + rng.integers(0, K, nq))
    few = rng.choice(rid, 6, replace=False)
    filters = [ix.row_mask(None, rng.choice(rid, n1 // 3, replace=False)),
               ix.row_mask(rng.choice(rid, n1 // 2, replace=False), None),
               (ix.row_mask(few, None), len(few), few),
               ix.row_mask(np.zeros(0, np.uint64), None)]
    ufilters = [_bits(rng.random(n2) < 0.7), _bits(rng.random(n2) < 0.5), _bits(np.zeros(n2, bool)), None]
    fof = rng.integers(-1, len(filters), nq)
    fof[:8] = 2  # selective probe-rule queries that reach the shortcut
    nprobes[:8], k[:8] = 0, rng.integers(6, 20, 8)
    lo = np.where(rng.random(nq) < 0.15, np.float32(0.5), np.nan).astype(np.float32)
    hi = np.where(rng.random(nq) < 0.15, np.float32(1e4), np.nan).astype(np.float32)
    ef = np.zeros(nq, np.int64)
    if hnsw:
        kc = k * np.maximum(rf, 1)
        ef = np.where(rng.random(nq) < 0.4, kc + rng.integers(0, 40, nq), 0)
    return dict(k=k, nprobes=nprobes, minimum_nprobes=mins, maximum_nprobes=maxs, refine_factor=rf, filters=filters,
                filter_of=fof, lower_bound=lo, upper_bound=hi, ef=ef), ufilters


def _opt(v):
    return None if np.isnan(v) else float(v)


def _combined_single(ix, q, i, p, ufilters, col, ucol, urid, uvalid):
    f = int(p["filter_of"][i])
    flt = p["filters"][f] if f >= 0 else None
    bm, max_len, mask_ids = flt if isinstance(flt, tuple) else (flt, None, None)
    probed = p["nprobes"][i] == 0
    out = ix.search_combined(q[i:i + 1], int(p["k"][i]), col, ucol, urid,
                             nprobes=None if probed else int(p["nprobes"][i]),
                             minimum_nprobes=int(p["minimum_nprobes"][i]),
                             maximum_nprobes=int(p["maximum_nprobes"][i]) or None,
                             refine_factor=int(p["refine_factor"][i]), allow_bitmap=bm,
                             unindexed_allow_bitmap=ufilters[f] if f >= 0 else uvalid,
                             mask_ids=mask_ids if probed else None, mask_max_len=max_len if probed else None,
                             lower_bound=_opt(p["lower_bound"][i]), upper_bound=_opt(p["upper_bound"][i]))
    return out


def _merge_rows(a, b, k):
    """the (distance, row id) merge of two result rows, first k"""
    (ai, ad, ac), (bi, bd, bc) = a, b
    ids = np.concatenate([ai[:ac], bi[:bc]])
    ds = np.concatenate([ad[:ac], bd[:bc]])
    o = np.lexsort((ids, ds.view(np.int32) ^ ((ds.view(np.int32) >> 31) & 0x7FFFFFFF)))[:k]
    return ids[o], ds[o], len(o)


KINDS = ("pq8", "pq4", "flat", "sq", "rq", "hnsw_sq", "hnsw_pq", "hnsw_flat")
CASES = [(kind, dt, m) for kind in KINDS for dt in (("f32",) if kind == "rq" else ("f32", "f16", "bf16", "u8"))
         for m in ("l2", "cosine", "dot")]


@pytest.mark.gpu
@pytest.mark.parametrize("kind,dt,metric", CASES, ids=lambda c: str(c))
def test_combined_batch_equals_single(kind, dt, metric):
    n1, n2, K, nq = 3000, 700, 16, 60
    x = _data(n1 + n2, D, 7)
    col, ucol = _typed(x[:n1], dt), _typed(x[n1:], dt)
    ix = _build(kind, col, metric, dt, K)
    rng = np.random.default_rng(3 + KINDS.index(kind))
    urid = np.arange(n1, n1 + n2, dtype=np.uint64)
    uvalid = _bits(rng.random(n2) < 0.9)
    q = _typed(_data(nq, D, 8), dt)
    p, uf = _mixed(ix, nq, K, n1, n2, rng, kind.startswith("hnsw"))
    gi, gd, gc, gn = ix.search_combined_batch(q, **p, vectors=col, unindexed_vectors=ucol, unindexed_row_ids=urid,
                                              unindexed_allow_bitmap=uvalid, unindexed_filters=uf)
    for i in np.nonzero(p["ef"] == 0)[0]:
        wi, wd, wc, wn = _combined_single(ix, q, i, p, uf, col, ucol, urid, uvalid)
        _same_row((gi, gd, gc), i, (wi, wd, wc), (kind, dt, metric))
        if p["nprobes"][i] == 0:
            assert gn[i] == wn[0], i
        else:
            assert gn[i] == min(p["nprobes"][i], K), i
    ef = np.nonzero(p["ef"] > 0)[0]
    if len(ef):  # search_batch (ef, refine factor max(1, rf)) + flat_search over the unindexed rows, merged
        pe = {n: (v[ef] if isinstance(v, np.ndarray) else v) for n, v in p.items()}
        pe["refine_factor"] = np.maximum(pe["refine_factor"], 1)
        ai, ad, ac, an = ix.search_batch(np.ascontiguousarray(q[ef]), **pe, vectors=col)
        for j, i in enumerate(ef):
            f = int(p["filter_of"][i])
            ui, ud, uc = lb.flat_search(ucol, q[i:i + 1], int(p["k"][i]), metric, row_ids=urid,
                                        allow_bitmap=uf[f] if f >= 0 else uvalid, lower_bound=_opt(p["lower_bound"][i]),
                                        upper_bound=_opt(p["upper_bound"][i]), bf16=dt == "bf16")
            wi, wd, wc = _merge_rows((ai[j], ad[j], ac[j]), (ui[0], ud[0], uc[0]), int(p["k"][i]))
            _same_row((gi, gd, gc), i, (wi, wd, np.array([wc])), (kind, "ef"))
            assert gn[i] == an[j]


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["pq8", "flat"])
def test_combined_batch_without_unindexed_rows(kind):
    """unindexed n = 0, and unindexed rows whose bits are all clear: the index half re-scored, alone"""
    n1, K, nq = 3000, 16, 40
    x = _data(n1 + 300, D, 9)
    ix = _build(kind, x[:n1], "l2", "f32", K)
    rng = np.random.default_rng(10)
    q = _data(nq, D, 11)
    p, _ = _mixed(ix, nq, K, n1, 300, rng, False)
    for ucol, urid, uvalid, uf in ((np.zeros((0, D), np.float32), np.zeros(0, np.uint64), None, [None] * 4),
                                   (x[n1:], np.arange(n1, n1 + 300, dtype=np.uint64), _bits(np.zeros(300, bool)),
                                    [_bits(np.zeros(300, bool))] * 4)):
        got = ix.search_combined_batch(q, **p, vectors=x[:n1], unindexed_vectors=ucol, unindexed_row_ids=urid,
                                       unindexed_allow_bitmap=uvalid, unindexed_filters=uf)
        for i in range(nq):
            want = _combined_single(ix, q, i, p, uf, x[:n1], ucol, urid, uvalid)
            _same_row(got[:3], i, want[:3], len(ucol))


@pytest.mark.gpu
def test_sparse_row_id_plan():
    """candidates (refine factor max(1, rf)), a take of the distinct ids, refine_taken, flat_search_batch over the
    unindexed rows and a host merge by (_distance, _rowid) equal search_combined_batch with the dense column"""
    n1, n2, K, nq = 4000, 900, 16, 80
    x = _data(n1 + n2, D, 12)
    rng = np.random.default_rng(13)
    sid = _sparse_ids(n1 + n2, rng)
    p = lb.IvfBuildParams(num_partitions=K, num_sub_vectors=8, max_iters=4, pq_max_iters=4, seed=1)
    ix_s = lb.IvfPqIndex.build(x[:n1], "l2", p, row_ids=sid[:n1])
    ix_d = lb.IvfPqIndex.build(x[:n1], "l2", p)
    pm, uf = _mixed(ix_d, nq, K, n1, n2, rng, False)
    # the sparse index's filters select the same rows as the dense index's
    e = ix_d.export()
    filters_s = []
    for f in pm["filters"]:
        bm, ml, mids = f if isinstance(f, tuple) else (f, None, None)
        words = np.asarray(bm, np.uint64)
        allowed = np.unpackbits(words.view(np.uint8), bitorder="little")[:n1].astype(bool)
        dense_ids = e["row_ids"][allowed].astype(np.int64)
        m = ix_s.row_mask(sid[dense_ids], None)
        filters_s.append((m, ml, sid[np.asarray(mids, np.int64)]) if mids is not None else m)
    ps = dict(pm, filters=filters_s)
    q = _data(nq, D, 14)
    wi, wd, wc, wn = ix_d.search_combined_batch(q, **pm, vectors=x[:n1], unindexed_vectors=x[n1:],
                                                unindexed_row_ids=np.arange(n1, n1 + n2, dtype=np.uint64),
                                                unindexed_filters=uf)
    rf1 = np.maximum(ps["refine_factor"], 1)
    cand = dict(ps, refine_factor=rf1)
    ci, cd, cc, cn, uniq, pos = ix_s.search_candidates(q, **cand, distinct=True)
    by_id = dict(zip(sid[:n1].tolist(), range(n1)))
    taken = x[[by_id[int(r)] for r in uniq]]
    ai, ad, ac = ix_s.refine_taken(q, (ci, cd, cc), taken, pos, ps["k"], rf1, ps["lower_bound"], ps["upper_bound"])
    ui, ud, uc = lb.flat_search_batch(x[n1:], q, ps["k"], "l2", row_ids=sid[n1:], filters=uf,
                                      filter_of=ps["filter_of"], lower_bound=ps["lower_bound"],
                                      upper_bound=ps["upper_bound"])
    to_dense = dict(zip(sid.tolist(), range(n1 + n2)))
    for i in range(nq):
        mi, md, mc = _merge_rows((ai[i], ad[i], ac[i]), (ui[i], ud[i], uc[i]), int(ps["k"][i]))
        assert wc[i] == mc, i
        assert np.array_equal(np.array([to_dense[int(r)] for r in mi], np.uint64), wi[i, :mc]), i
        assert np.array_equal(md.view(np.uint32), wd[i, :mc].view(np.uint32)), i
    assert np.array_equal(cn, wn)


@pytest.mark.gpu
def test_launches_do_not_grow_with_parameter_sets():
    n1, n2, nq = 6000, 3000, 512
    x = _data(n1 + n2, 64, 5)
    ix = lb.IvfFlatIndex.build(x[:n1], "l2", num_partitions=32, max_iters=4, seed=1)
    e = ix.export()
    rng = np.random.default_rng(2)
    q = _data(nq, 64, 6)
    filters = [ix.row_mask(rng.choice(e["row_ids"], 3000, replace=False), None) for _ in range(nq)]
    ufilters = [_bits(rng.random(n2) < 0.5) for _ in range(nq)]
    k = rng.integers(1, 60, nq)
    k[0] = 59
    lo = np.where(rng.random(nq) < 0.5, rng.random(nq).astype(np.float32), np.nan).astype(np.float32)
    hi = np.where(rng.random(nq) < 0.5, np.float32(1e4) + rng.random(nq).astype(np.float32), np.nan).astype(np.float32)
    lo[0], hi[0] = 0.5, 1e4
    urid = np.arange(n1, n1 + n2, dtype=np.uint64)
    lb.launch_count(reset=True)
    lb.flat_search_batch(x[n1:], q, k, "l2", filters=ufilters, filter_of=np.arange(nq), lower_bound=lo,
                         upper_bound=hi)
    mixed = lb.launch_count(reset=True)
    lb.flat_search_batch(x[n1:], q, 59, "l2", filters=ufilters[:1], filter_of=0, lower_bound=0.5, upper_bound=1e4)
    uniform = lb.launch_count(reset=True)
    assert mixed == uniform, (mixed, uniform)
    kw = dict(vectors=x[:n1], unindexed_vectors=x[n1:], unindexed_row_ids=urid)
    lb.launch_count(reset=True)
    rf = rng.integers(0, 5, nq)
    rf[0] = 4
    ix.search_combined_batch(q, k, nprobes=6, refine_factor=rf, filters=filters,
                             filter_of=np.arange(nq), unindexed_filters=ufilters, lower_bound=lo, upper_bound=hi, **kw)
    mixed = lb.launch_count(reset=True)
    ix.search_combined_batch(q, 59, nprobes=6, refine_factor=4, filters=filters[:1], filter_of=0,
                             unindexed_filters=ufilters[:1], lower_bound=0.5, upper_bound=1e4, **kw)
    uniform = lb.launch_count(reset=True)
    assert mixed == uniform, (mixed, uniform)


def _raw_flat(x, q, cp, filters, k_stride):
    nq = q.shape[0]
    outs = [np.full((nq, k_stride), 7, np.uint64), np.full((nq, k_stride), 7, np.float32), np.full(nq, 7, np.uint32)]
    keep = []
    table = lb._bitmap_table(filters, keep)
    st = _lib.lib().lb2_flat_search_batch(C.c_void_p(x.ctypes.data), x.shape[0], x.shape[1], _lib.F32, _lib.L2, None,
                                          C.c_void_p(q.ctypes.data), nq, C.c_void_p(cp.ctypes.data), table,
                                          len(filters), k_stride, *[C.c_void_p(o.ctypes.data) for o in outs])
    return st, outs


def _flat_cp(nq, k, filt=0xFFFFFFFF):
    cp = np.zeros(nq, np.dtype({"names": [f for f, _ in _lib.FlatQueryParams._fields_],
                                "formats": [np.float32 if t is C.c_float else np.uint32
                                            for _, t in _lib.FlatQueryParams._fields_]}))
    cp["k"], cp["filter"] = k, filt
    return cp


def _last_error():
    buf = C.create_string_buffer(2048)
    _lib.lib().lb2_last_error(buf, 2048)
    return buf.value.decode()


@pytest.mark.gpu
def test_refusals_write_nothing():
    x = _data(2000, D, 1)
    q = _data(4, D, 2)
    for k, filt, stride, nf, want, msg in (
            ([5, 0, 5, 5], 0xFFFFFFFF, 5, 0, _lib.INVALID_ARG, "query 1"),        # k = 0
            ([5, 5, 1025, 5], 0xFFFFFFFF, 1025, 0, _lib.UNSUPPORTED, "query 2"),  # k > 1024
            ([5, 5, 5, 9], 0xFFFFFFFF, 5, 0, _lib.INVALID_ARG, "k_stride"),       # k_stride below the largest k
            ([5, 5, 5, 5], [0, 0, 1, 0], 5, 1, _lib.INVALID_ARG, "query 2")):     # filter 1 of 1
        st, outs = _raw_flat(x, q, _flat_cp(4, k, filt), [None] * nf, stride)
        assert st == want and msg in _last_error(), (k, st, _last_error())
        for o in outs:
            assert (o == 7).all(), k
    ix = _build("flat", x, "l2", "f32")
    ux, urid = _data(300, D, 3), np.arange(2000, 2300, dtype=np.uint64)
    ok_table = (C.c_void_p * 1)()

    def raw(kw, stride, vectors=True, u="ok", nf=0, table=ok_table):
        cp = ix._batch_params("t", q, **kw)[4]
        cf = (_lib.QueryFilter * 1)()
        rows = _lib.UnindexedRows(ux.ctypes.data, 300, urid.ctypes.data if u != "no_ids" else None, None)
        ub = _lib.UnindexedBatch(rows, C.cast(table, C.c_void_p) if table is not None else None)
        outs = [np.full((4, stride), 7, np.uint64), np.full((4, stride), 7, np.float32), np.full(4, 7, np.uint32),
                np.full(4, 7, np.uint32)]
        st = _lib.lib().lb2_index_search_combined_batch(
            ix._h, C.c_void_p(q.ctypes.data), 4, C.c_void_p(cp.ctypes.data), cf, nf,
            C.c_void_p(x.ctypes.data) if vectors else None, 2000, 1, None if u is None else C.byref(ub), stride,
            *[C.c_void_p(o.ctypes.data) for o in outs])
        return st, outs

    for args, want in (((dict(k=10, nprobes=4), 10, False), _lib.INVALID_ARG),                 # no refine vectors
                       ((dict(k=10, nprobes=4), 10, True, None), _lib.INVALID_ARG),            # no unindexed rows
                       ((dict(k=10, nprobes=4), 10, True, "no_ids"), _lib.INVALID_ARG),        # no unindexed row ids
                       ((dict(k=10, nprobes=4), 10, True, "ok", 1, None), _lib.INVALID_ARG),   # no filter bitmaps
                       ((dict(k=10, nprobes=4), 9), _lib.INVALID_ARG),                         # k_stride below k
                       ((dict(k=200, nprobes=4, refine_factor=6), 200), _lib.UNSUPPORTED),     # k' > 1024
                       ((dict(k=10, nprobes=4, filter_of=0, filters=[None]), 10), _lib.INVALID_ARG),  # filter 0 of 0
                       ((dict(k=10, nprobes=4, ef=20), 10), _lib.INVALID_ARG)):                # ef without graphs
        st, outs = raw(*args)
        assert st == want, (args, st)
        for o in outs:
            assert (o == 7).all(), args
    st, _ = raw(dict(k=np.array([10, 10, 10, 300]), nprobes=4, refine_factor=4), 300)
    assert st == _lib.UNSUPPORTED and "query 3" in _last_error()


# ---------------------------------------------------------------------------------------------------------------
# CPU: struct layout and Python argument checks
# ---------------------------------------------------------------------------------------------------------------

def test_struct_layout_matches_header(tmp_path):
    import os
    import shutil
    import subprocess
    if shutil.which("cc") is None:
        pytest.skip("needs a C compiler")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    fields = {"lb2_flat_query_params": (_lib.FlatQueryParams, ["k", "filter", "has_lower_bound", "has_upper_bound",
                                                               "lower_bound", "upper_bound"]),
              "lb2_unindexed_rows": (_lib.UnindexedRows, ["vectors", "n", "row_ids", "allow_bitmap"]),
              "lb2_unindexed_batch": (_lib.UnindexedBatch, ["rows", "filter_bitmaps"])}
    lines = ["#include <stdio.h>", "#include <stddef.h>", '#include "lance_b200.h"', "int main(void) {"]
    for name, (_, fl) in fields.items():
        lines.append(f'  printf("{name} %zu\\n", sizeof({name}));')
        lines += [f'  printf("{name}.{f} %zu\\n", offsetof({name}, {f}));' for f in fl]
    lines += ["  return 0;", "}"]
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text("\n".join(lines) + "\n")
    subprocess.run(["cc", "-I", os.path.join(root, "include"), str(src), "-o", str(exe)], check=True)
    got = dict(line.split() for line in subprocess.run([str(exe)], check=True, capture_output=True,
                                                       text=True).stdout.splitlines())
    for name, (cls, fl) in fields.items():
        assert int(got[name]) == C.sizeof(cls), name
        assert [f for f, _ in cls._fields_] == fl
        for f in fl:
            assert int(got[f"{name}.{f}"]) == getattr(cls, f).offset, (name, f)


class _NoLibrary(lb.IvfPqIndex):
    """an index whose handle must never reach the library"""

    def __init__(self):
        super().__init__(None)


@pytest.mark.parametrize("kw", [
    dict(k=np.array([5, 5, 5])),                                   # k of the wrong length
    dict(k=np.array([5, 0, 5, 5])),                                # k = 0
    dict(filter_of=0),                                             # no filters
    dict(filters=[np.zeros(1, np.uint64)], filter_of=np.array([0, 1, -1, 0])),
    dict(lower_bound=np.zeros(3, np.float32)),
    dict(out=(np.empty((4, 3), np.uint64), np.empty((4, 3), np.float32))),   # rows shorter than the largest k
    dict(out=(np.empty((3, 5), np.uint64), np.empty((3, 5), np.float32))),   # wrong number of rows
])
def test_flat_batch_arguments_are_checked_before_the_library(kw, monkeypatch):
    monkeypatch.setattr(lb, "lib", lambda: pytest.fail("reached the library"))
    args = dict(k=5)
    args.update(kw)
    with pytest.raises(ValueError):
        lb.flat_search_batch(np.zeros((10, 8), np.float32), np.zeros((4, 8), np.float32), **args)


@pytest.mark.parametrize("kw", [
    dict(k=np.array([5, 5, 5])),                                   # k of the wrong length
    dict(nprobes=-1),
    dict(filters=[np.zeros(1, np.uint64)], filter_of=0),           # no unindexed bitmap for the filter
    dict(filters=[np.zeros(1, np.uint64)], filter_of=0, unindexed_filters=[None, None]),
    dict(vectors=None),                                            # the index half is always re-scored
    dict(unindexed_row_ids=None),
    dict(out=(np.empty((4, 3), np.uint64), np.empty((4, 3), np.float32))),
])
def test_combined_batch_arguments_are_checked_before_the_library(kw):
    args = dict(k=5, nprobes=3, vectors=np.zeros((10, 8), np.float32), unindexed_vectors=np.zeros((3, 8), np.float32),
                unindexed_row_ids=np.arange(10, 13, dtype=np.uint64))
    args.update(kw)
    with pytest.raises(ValueError):
        _NoLibrary().search_combined_batch(np.zeros((4, 8), np.float32), **args)
