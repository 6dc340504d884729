"""IVF_HNSW_SQ against the restatement of the reference (tests/hnsw_reference.py): the restatement's own invariants
on the CPU, and on the device the IVF stage and codes equal to IVF_SQ's, the graphs bit for bit (levels, every list's
ids, distances and order) and every search result (ids, distances, counts) bit-identical."""
import numpy as np
import pytest

import lance_b200 as lb
import hnsw_reference as hr
from sq_reference import sq_encode


def _data(n, d, seed, dup=0):
    rng = np.random.default_rng(seed)
    x = (rng.standard_normal((n, d)) + 3 * rng.standard_normal((8, d))[rng.integers(0, 8, n)]).astype(np.float32)
    if dup:
        x[-dup:] = x[:dup]     # duplicated rows: their distances tie
    return x


def _csr(n, K, seed):
    """random partition ids with one empty partition, one single-row partition and one smaller than m"""
    rng = np.random.default_rng(seed)
    p = rng.integers(3, K, n).astype(np.uint32)
    p[:1] = 1
    p[1:4] = 2
    return p


def _assert_graph_equal(got, want):
    assert got["max_level"] == want["max_level"] and got["m"] == want["m"]
    assert np.array_equal(got["levels"], want["levels"])
    assert np.array_equal(got["counts0"], want["counts0"])
    assert np.array_equal(got["counts_up"], want["counts_up"])
    for r, c in enumerate(want["counts0"]):
        assert np.array_equal(got["neighbors0"][r, :c], want["neighbors0"][r, :c]), r
        assert np.array_equal(got["dists0"][r, :c].view(np.uint32), want["dists0"][r, :c].view(np.uint32)), r
    for u, c in enumerate(want["counts_up"]):
        assert np.array_equal(got["neighbors_up"][u, :c], want["neighbors_up"][u, :c]), u
        assert np.array_equal(got["dists_up"][u, :c].view(np.uint32), want["dists_up"][u, :c].view(np.uint32)), u


# ---- CPU: the restatement -----------------------------------------------------------------------------------------
def test_reference_heap_is_rust_binary_heap_order():
    h = hr.RHeap()
    for key, v in [(3, 0), (1, 1), (3, 2), (2, 3), (3, 4), (0, 5)]:
        h.push(key, v)
    assert h.pop() == (3, 0)
    assert [k for k, _ in hr.RHeap.into_sorted(h)] == [0, 1, 2, 3, 3]


@pytest.mark.parametrize("metric", ["l2", "dot"])
@pytest.mark.parametrize("m,efc", [(20, 150), (4, 8)])
def test_reference_graph_invariants(metric, m, efc):
    rng = np.random.default_rng(1)
    codes = rng.integers(0, 256, (300, 16), dtype=np.uint8)
    codes[-20:] = codes[:20]
    offs = np.array([0, 0, 1, 4, 300], np.uint64)
    g = hr.build(codes, offs, (-1.0, 2.0), metric, m=m, max_level=5, efc=efc, seed=3)
    lv = g["levels"].astype(np.int64)
    assert (g["counts0"] <= 2 * m).all() and (g["counts_up"] <= m).all()          # degrees
    assert len(g["counts_up"]) == int((lv - 1).sum())                             # level counts add up
    up = np.concatenate([[0], np.cumsum(lv - 1)])
    for p in range(4):
        a, b = int(offs[p]), int(offs[p + 1])
        if b > a:
            assert lv[a] == 5
        for r in range(a, b):
            assert (g["neighbors0"][r, :g["counts0"][r]] < b - a).all()
            for level in range(1, lv[r]):
                u = up[r] + level - 1
                for nid in g["neighbors_up"][u, :g["counts_up"][u]]:
                    assert lv[a + nid] > level                                   # every neighbour has the level
    assert g["counts0"][4:].min() > 0                                             # a partition > 1 row is connected


def test_reference_levels_follow_the_thresholds():
    lv = np.array(hr.node_levels(0, 0, 20001, 20, 7))
    assert lv[0] == 7 and lv[1:].max() <= 7
    frac = (lv[1:] >= 2).mean()
    assert abs(frac - 1 / 20) < 0.01


def test_reference_search_finds_itself():
    rng = np.random.default_rng(2)
    x = rng.standard_normal((200, 8)).astype(np.float32)
    bounds = (float(x.min()), float(x.max()))
    codes = sq_encode(x, *bounds)
    offs = np.array([0, 200], np.uint64)
    g = hr.build(codes, offs, bounds, "l2", m=8, max_level=4, efc=40, seed=0)
    ids, d, c = hr.search(np.zeros((1, 8), np.float32), bounds, offs, codes, np.arange(200, dtype=np.uint64), g,
                          x[:10], 1, 1)
    assert (d[:, 0] == 0).all() and (c == 1).all()


# ---- GPU: build ---------------------------------------------------------------------------------------------------
def _typed(x, dt):
    if dt == "f32":
        return x, {}
    if dt == "f16":
        return x.astype(np.float16), {}
    if dt == "bf16":
        b = np.ascontiguousarray(x, np.float32).view(np.uint32).astype(np.uint64)
        return ((b + 0x7FFF + ((b >> 16) & 1)) >> 16).astype(np.uint16), {"bf16": True}
    return np.clip(x * 20 + 128, 0, 255).astype(np.uint8), {}


BUILD_CASES = [("l2", "f32", 8, 20, 150), ("cosine", "f32", 36, 20, 150), ("dot", "f32", 128, 20, 150),
               ("l2", "f16", 36, 4, 8), ("dot", "bf16", 8, 4, 8), ("l2", "u8", 128, 4, 8), ("cosine", "f16", 8, 4, 8),
               ("dot", "u8", 36, 20, 150), ("l2", "bf16", 128, 20, 150)]


@pytest.mark.gpu
@pytest.mark.parametrize("metric,dt,d,m,efc", BUILD_CASES)
def test_build_bit_identical(metric, dt, d, m, efc):
    x, kw = _typed(_data(700, d, seed=d + m, dup=40), dt)
    args = dict(num_partitions=6, max_iters=10, seed=5)
    ix = lb.IvfHnswSqIndex.build(x, metric, hnsw_params=lb.HnswBuildParams(max_level=5, m=m, ef_construction=efc),
                                 **args, **kw)
    sq = lb.IvfSqIndex.build(x, metric, **args, **kw).export()
    got = ix.export()
    for key in ("centroids", "part_offsets", "codes", "row_ids"):
        assert np.array_equal(got[key], sq[key]), key
    assert got["bounds"] == sq["bounds"]
    want = hr.build(got["codes"], got["part_offsets"], got["bounds"], "dot" if metric == "dot" else "l2", m=m,
                    max_level=5, efc=efc, seed=5)
    _assert_graph_equal(got["graph"], want)


@pytest.mark.gpu
def test_build_small_partitions_bit_identical():
    """partitions with fewer rows than m, one row or none: a device build over many small partitions, and a graph
    with an empty, a one-row and a three-row partition loaded through from_parts"""
    x = _data(160, 16, seed=9, dup=30)
    ix = lb.IvfHnswSqIndex.build(x, "l2", num_partitions=12, max_iters=10)
    got = ix.export()
    assert np.diff(got["part_offsets"].astype(np.int64)).min() < 20
    _assert_graph_equal(got["graph"], hr.build(got["codes"], got["part_offsets"], got["bounds"], "l2"))
    # a device build with an empty partition (a far centroid) and a one-row partition (a far row with its own
    # centroid), then a search that probes both
    y = x.copy()
    y[7] = 500.0
    cent = np.stack([y[:80].mean(axis=0), y[80:].mean(axis=0), np.full(16, -900.0, np.float32), y[7]])
    ix = lb.IvfHnswSqIndex.build(y, "l2", num_partitions=4, max_iters=1, centroids=cent)
    got = ix.export()
    sizes = np.diff(got["part_offsets"].astype(np.int64))
    assert 0 in sizes.tolist() and 1 in sizes.tolist(), sizes
    _assert_graph_equal(got["graph"], hr.build(got["codes"], got["part_offsets"], got["bounds"], "l2"))
    q = np.concatenate([y[7:8] + 1, np.full((1, 16), -800.0, np.float32), y[:3]])
    ids, d = ix.search(q, k=5, nprobes=4)
    wi, wd, _ = _ref_search(got, "l2", q, 5, 4)
    assert np.array_equal(ids, wi) and np.array_equal(d.view(np.uint32), wd.view(np.uint32))
    bounds = (float(x.min()), float(x.max()))
    codes = sq_encode(x, *bounds)
    part = _csr(160, 6, seed=4)
    sq = lb.IvfSqIndex.from_parts(np.zeros((6, 16), np.float32), bounds, part, codes,
                                  np.arange(160, dtype=np.uint64)).export()
    offs = sq["part_offsets"].astype(np.int64)
    assert offs[1] - offs[0] == 0 and offs[2] - offs[1] == 1 and offs[3] - offs[2] == 3
    g = hr.build(sq["codes"], sq["part_offsets"], bounds, "l2")
    ix = lb.IvfHnswSqIndex.from_parts(np.zeros((6, 16), np.float32), bounds, part, codes,
                                      np.arange(160, dtype=np.uint64), graph=g)
    _assert_graph_equal(ix.export()["graph"], g)


# ---- GPU: search --------------------------------------------------------------------------------------------------
def _index(metric="l2", n=1500, d=16, K=4, m=8, efc=40, seed=0):
    x = _data(n, d, seed=seed, dup=50)
    ix = lb.IvfHnswSqIndex.build(x, metric, num_partitions=K, max_iters=10, seed=seed,
                                 hnsw_params=lb.HnswBuildParams(max_level=4, m=m, ef_construction=efc))
    return x, ix, ix.export()


def _ref_search(parts, metric, q, k, nprobes, **kw):
    return hr.search(parts["centroids"], parts["bounds"], parts["part_offsets"], parts["codes"], parts["row_ids"],
                     parts["graph"], q, k, nprobes, metric=metric, **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("metric", ["l2", "cosine", "dot"])
@pytest.mark.parametrize("k,ef", [(1, None), (10, None), (10, 50), (100, None), (1024, None), (1024, 1100), (7, 7)])
def test_search_bit_identical(metric, k, ef):
    x, ix, parts = _index(metric, n=2600 if k == 1024 else 1500)
    q = _data(12, 16, seed=77)
    ids, d = ix.search(q, k=k, nprobes=2, ef=ef)
    wi, wd, wc = _ref_search(parts, metric, q, k, 2, ef=ef)
    assert np.array_equal(d.view(np.uint32), wd.view(np.uint32))
    assert np.array_equal(ids, wi)


@pytest.mark.gpu
def test_ef_below_k_is_refused():
    _, ix, _ = _index()
    with pytest.raises(lb.LanceB200Error) as e:
        ix.search(_data(2, 16, seed=1), k=10, nprobes=1, ef=9)
    assert e.value.status == lb._lib.INVALID_ARG


@pytest.mark.gpu
@pytest.mark.parametrize("side", [-1, 0, 1])
def test_prefilter_either_side_of_the_switch(side):
    x, ix, parts = _index(K=1)
    n = x.shape[0]
    want = n * 10 // 100 + side        # side -1: flat branch; 0, 1: the graph
    rng = np.random.default_rng(3)
    allowed_pos = np.sort(rng.choice(n, want, replace=False))
    bits = np.zeros(n, bool)
    bits[allowed_pos] = True
    bm = np.packbits(bits, bitorder="little")
    bm = np.concatenate([bm, np.zeros((-bm.size) % 8, np.uint8)]).view(np.uint64)
    q = _data(8, 16, seed=5)
    ids, d = ix.search_ex(q, k=10, nprobes=1, allow_bitmap=bm)
    wi, wd, _ = _ref_search(parts, "l2", q, 10, 1, allow_bits=bits)
    assert np.array_equal(d.view(np.uint32), wd.view(np.uint32))
    assert np.array_equal(ids, wi)


@pytest.mark.gpu
@pytest.mark.parametrize("flat", [False, True])
def test_range_bounds_on_rows(flat):
    x, ix, parts = _index(K=1)
    n = x.shape[0]
    q = _data(4, 16, seed=6)
    ids0, d0 = ix.search(q, k=30, nprobes=1)
    lower, upper = float(d0[0, 3]), float(d0[0, 20])     # rows exactly on both bounds
    bits = np.ones(n, bool)
    if flat:                                             # 5 % of the rows allowed: the flat branch
        bits[:] = False
        bits[:n // 20] = True
    bm = np.packbits(bits, bitorder="little")
    bm = np.concatenate([bm, np.zeros((-bm.size) % 8, np.uint8)]).view(np.uint64)
    ids, d = ix.search_ex(q, k=30, nprobes=1, allow_bitmap=bm, lower_bound=lower, upper_bound=upper)
    wi, wd, _ = _ref_search(parts, "l2", q, 30, 1, allow_bits=bits, lower=lower, upper=upper)
    assert np.array_equal(d.view(np.uint32), wd.view(np.uint32))
    assert np.array_equal(ids, wi)


def _refined(x, q, cand, k):
    """the refine step over one candidate list per query: exact distances (the refine rule of flat_reference), the k
    smallest by (distance, row id)"""
    import flat_reference as fr
    ids, ds = [], []
    for r in range(q.shape[0]):
        c = cand[r][cand[r] != np.iinfo(np.uint64).max]
        d = fr.distances(q[r:r + 1], x[c.astype(np.int64)], "l2", "f32")[0].astype(np.float32)
        o = np.lexsort((c, fr.total_order_key(d)))[:k]
        ids.append(c[o])
        ds.append(d[o])
    return ids, ds


@pytest.mark.gpu
def test_refine_probed_async_sharded_match_search():
    x, ix, parts = _index()
    q = _data(6, 16, seed=8)
    # refine: the graph search's k' = k * refine_factor candidates, then the exact re-rank
    for ef in (None, 40):
        ids, d = ix.search_refine(x, q, k=5, nprobes=2, refine_factor=3, ef=ef)
        ci, _, _ = _ref_search(parts, "l2", q, 15, 2, ef=ef)
        wi, wd = _refined(x, q, ci, 5)
        for r in range(q.shape[0]):
            assert np.array_equal(ids[r], wi[r]) and np.array_equal(d[r].view(np.uint32), wd[r].view(np.uint32))
    with pytest.raises(lb.LanceB200Error) as e:       # ef < k' = k * refine_factor
        ix.search_refine(x, q, k=5, nprobes=2, refine_factor=3, ef=14)
    assert e.value.status == lb._lib.INVALID_ARG
    si, sd = ix.search(q, k=10, nprobes=2)
    pi, pd, pc, _ = ix.search_probed(q, 10, minimum_nprobes=2, maximum_nprobes=2)
    assert np.array_equal(pi, si) and np.array_equal(pd.view(np.uint32), sd.view(np.uint32))
    pi, pd, pc, _ = ix.search_probed(q, 10, minimum_nprobes=2, maximum_nprobes=2, ef=30)
    wi, wd, _ = _ref_search(parts, "l2", q, 10, 2, ef=30)
    assert np.array_equal(pi, wi) and np.array_equal(pd.view(np.uint32), wd.view(np.uint32))
    hi, hd = ix.search_sharded(q, k=10, nprobes=2)
    assert np.array_equal(hi, si) and np.array_equal(hd.view(np.uint32), sd.view(np.uint32))
    # async: the scratch of the pending search is freed in stream order
    qd = lb.DeviceArray.from_numpy(q)
    oi, od = lb.DeviceArray((6, 10), np.uint64), lb.DeviceArray((6, 10), np.float32)
    ix.search_async(qd, (oi, od), k=10, nprobes=2)
    lb.synchronize()
    wi, wd, _ = _ref_search(parts, "l2", q, 10, 2)
    assert np.array_equal(oi.numpy(), wi) and np.array_equal(od.numpy().view(np.uint32), wd.view(np.uint32))


@pytest.mark.gpu
def test_combined_search_bit_identical():
    """knn_combined: the graph search at refine max(1, rf) re-ranked exactly, a flat search over the unindexed rows,
    one merge by (distance, row id)"""
    import flat_reference as fr
    x, ix, parts = _index()
    q = _data(5, 16, seed=13)
    extra = _data(300, 16, seed=14)
    extra_ids = np.arange(5000, 5300, dtype=np.uint64)
    for rf in (0, 2):
        ids, d, c, _ = ix.search_combined(q, 10, x, extra, extra_ids, nprobes=2, refine_factor=rf)
        ci, _, _ = _ref_search(parts, "l2", q, 10 * max(1, rf), 2)
        ai, ad = _refined(x, q, ci, 10)
        fi, fd, fc = fr.flat_search(extra, q, 10, "l2", "f32", row_ids=extra_ids)
        for r in range(q.shape[0]):
            mi = np.concatenate([ai[r], fi[r][:fc[r]]])
            md = np.concatenate([ad[r], fd[r][:fc[r]]])
            o = np.lexsort((mi, fr.total_order_key(md)))[:10]
            assert np.array_equal(ids[r][:c[r]], mi[o]) and np.array_equal(d[r][:c[r]].view(np.uint32),
                                                                           md[o].view(np.uint32))


@pytest.mark.gpu
def test_graph_from_reference_with_other_m_searches_identically():
    x, ix, parts = _index()
    g = hr.build(parts["codes"], parts["part_offsets"], parts["bounds"], "l2", m=5, max_level=3, efc=20, seed=11)
    ix2 = lb.IvfHnswSqIndex.from_parts(parts["centroids"], parts["bounds"],
                                       np.repeat(np.arange(4, dtype=np.uint32),
                                                 np.diff(parts["part_offsets"]).astype(np.int64)),
                                       parts["codes"], parts["row_ids"], graph=g)
    parts2 = dict(parts, graph=g)
    q = _data(10, 16, seed=12)
    for k, ef in ((10, None), (10, 40), (50, None)):
        ids, d = ix2.search(q, k=k, nprobes=3, ef=ef)
        wi, wd, _ = _ref_search(parts2, "l2", q, k, 3, ef=ef)
        assert np.array_equal(d.view(np.uint32), wd.view(np.uint32))
        assert np.array_equal(ids, wi)
    # exported and reloaded: the same results
    e = ix2.export()
    ix3 = lb.IvfHnswSqIndex.from_parts(parts["centroids"], parts["bounds"],
                                       np.repeat(np.arange(4, dtype=np.uint32),
                                                 np.diff(e["part_offsets"]).astype(np.int64)),
                                       e["codes"], e["row_ids"], graph=e["graph"])
    assert np.array_equal(ix3.search(q, k=10, nprobes=3)[0], ix2.search(q, k=10, nprobes=3)[0])


@pytest.mark.gpu
@pytest.mark.parametrize("metric,floor", [("l2", 0.9), ("cosine", 0.9), ("dot", 0.85)])
def test_recall_floor(metric, floor):
    """test_create_ivf_hnsw_sq (rust/lance/src/index/vector/ivf/v2.rs:1470-1496 via test_recall, :1962-2007): 512 x 32
    uniform [0, 1) rows, nlist 4, the query row 0, k = 100, nprobes = nlist, against the exact ground truth"""
    rng = np.random.default_rng(0)
    x = rng.random((512, 32)).astype(np.float32)
    ix = lb.IvfHnswSqIndex.build(x, metric, num_partitions=4)
    q = x[:1]
    ids, _ = ix.search(q, k=100, nprobes=4)
    xs, qs = x.astype(np.float64), q[0].astype(np.float64)
    if metric == "l2":
        dist = ((xs - qs) ** 2).sum(axis=1)
    elif metric == "cosine":
        dist = 1 - xs @ qs / (np.linalg.norm(xs, axis=1) * np.linalg.norm(qs))
    else:
        dist = 1 - xs @ qs
    truth = set(np.argsort(dist, kind="stable")[:100].tolist())
    assert len(set(ids[0].tolist())) == 100
    assert len(truth & set(ids[0].tolist())) / 100 >= floor
