"""IVF_HNSW_PQ against the restatement of the reference (tests/hnsw_pq_reference.py): the restatement's own invariants
and its two distances on the CPU, and on the device the IVF stage, codebook and codes equal to IVF_PQ's, the graphs bit
for bit (levels, every list's ids, distances and order) and every search result (ids, distances, counts)
bit-identical."""
import numpy as np
import pytest

import flat_reference as fr
import hnsw_pq_reference as pr
import lance_b200 as lb
from oracle import binding as ob
from test_ivf_hnsw_sq import _assert_graph_equal, _data, _typed


def _codebook(M, nbits, ds, seed, dt="f32"):
    cb = np.random.default_rng(seed).standard_normal((M, 1 << nbits, ds)).astype(np.float32)
    if dt == "f16":
        cb = cb.astype(np.float16).astype(np.float32)
    elif dt == "bf16":
        cb = (cb.view(np.uint32) & 0xFFFF0000).view(np.float32)
    return cb


def _codes(n, M, nbits, seed):
    c = np.random.default_rng(seed).integers(0, 1 << nbits, (n, M)).astype(np.uint8)
    return c if nbits == 8 else (c[:, 0::2] | (c[:, 1::2] << 4)).astype(np.uint8)


# ---- CPU: the restatement -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("metric", ["l2", "dot"])
@pytest.mark.parametrize("nbits", [8, 4])
@pytest.mark.parametrize("m,efc", [(20, 150), (4, 8)])
def test_reference_graph_invariants(metric, nbits, m, efc):
    M, ds = 8, 4
    codes = _codes(300, M, nbits, 1)
    codes[-20:] = codes[:20]
    offs = np.array([0, 0, 1, 4, 300], np.uint64)
    g = pr.build(codes, offs, _codebook(M, nbits, ds, 2), nbits, metric, m=m, max_level=5, efc=efc, seed=3)
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


@pytest.mark.parametrize("nbits", [8, 4])
@pytest.mark.parametrize("d,M", [(16, 4), (32, 4), (64, 4), (36, 6)])     # sub-vector widths 4, 8, 16 and 6
@pytest.mark.parametrize("metric", ["l2", "dot"])
def test_node_matrix_zero_diagonal_and_symmetric(nbits, d, M, metric):
    codes = _codes(60, M, nbits, 5)
    codes[-5:] = codes[:5]
    D = pr.node_matrix(_codebook(M, nbits, d // M, 6), codes, nbits, metric)
    assert np.array_equal(D.view(np.uint32), D.T.view(np.uint32))               # bit for bit
    if metric == "l2":
        assert (np.diag(D) == 0).all()


@pytest.mark.parametrize("d,M", [(16, 4), (32, 4), (64, 4), (36, 6)])
def test_node_table_sum_is_the_pq_scan_sum(d, M):
    """8-bit: a row of D is the oracle's ADC scan (the IVF_PQ scan's sum) on node i's table"""
    cb = _codebook(M, 8, d // M, 7)
    codes = _codes(40, M, 8, 8)
    D = pr.node_matrix(cb, codes, 8, "l2")
    X = pr.decode(cb, codes, 8)
    for i in (0, 17, 39):
        want = ob.pq_scan(ob.build_lut(cb, X[i]), ob.transpose_codes(codes))
        assert np.array_equal(D[i].view(np.uint32), want.view(np.uint32))


@pytest.mark.parametrize("dt", ["f32", "f16", "bf16"])
@pytest.mark.parametrize("metric", ["l2", "dot"])
@pytest.mark.parametrize("nbits", [8, 4])
def test_between_matrix_is_the_oracle_distance(dt, metric, nbits):
    """H[u][v] = the oracle's distance function of the column type on the decoded rows"""
    M, ds = 6, 7
    cb = _codebook(M, nbits, ds, 9, dt)
    codes = _codes(24, M, nbits, 10)
    H = pr.between_matrix(cb, codes, nbits, metric, dt)
    X = pr.decode(cb, codes, nbits)
    fn = {("f32", "l2"): ob.l2, ("f32", "dot"): ob.dot, ("f16", "l2"): ob.l2_f16, ("f16", "dot"): ob.dot_f16,
          ("bf16", "l2"): ob.l2_bf16, ("bf16", "dot"): ob.dot_bf16}[(dt, metric)]
    conv = {"f32": lambda v: v, "f16": lambda v: v.astype(np.float16),
            "bf16": lambda v: (v.view(np.uint32) >> 16).astype(np.uint16)}[dt]
    for u in range(0, 24, 5):
        for v in range(0, 24, 3):
            want = np.float32(fn(conv(X[u]), conv(X[v])))
            if metric == "dot":                          # the oracle returns the product, the distance is 1 - it
                want = np.float32(1.0) - want
            assert want.view(np.uint32) == H[u, v].view(np.uint32), (u, v)


# ---- GPU: build ---------------------------------------------------------------------------------------------------
BUILD_CASES = [  # metric, dtype, d, M, nbits, m, efc: sub-vector widths 4, 8 and the generic loop (12, 2)
    ("l2", "f32", 16, 4, 8, 20, 150), ("cosine", "f32", 32, 4, 8, 4, 8), ("dot", "f32", 48, 4, 8, 20, 150),
    ("l2", "f32", 32, 16, 8, 4, 8), ("l2", "f16", 32, 4, 8, 4, 8), ("dot", "f16", 16, 4, 8, 4, 8),
    ("dot", "bf16", 32, 4, 4, 20, 150), ("l2", "bf16", 16, 4, 8, 4, 8), ("l2", "u8", 16, 4, 4, 4, 8),
    ("dot", "u8", 32, 4, 8, 4, 8), ("cosine", "f16", 48, 4, 4, 4, 8), ("l2", "f32", 32, 16, 4, 20, 150),
    ("dot", "f32", 16, 4, 4, 4, 8), ("dot", "bf16", 32, 16, 8, 4, 8)]


def _params(M, nbits, K=6, seed=5):
    return lb.IvfBuildParams(num_partitions=K, num_sub_vectors=M, num_bits=nbits, max_iters=10, pq_max_iters=10,
                             seed=seed)


def _ref_build(parts, nbits, metric, dt, **kw):
    return pr.build(parts["codes"], parts["part_offsets"], parts["codebook"], nbits, metric, dt, **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("metric,dt,d,M,nbits,m,efc", BUILD_CASES)
def test_build_bit_identical(metric, dt, d, M, nbits, m, efc):
    x, kw = _typed(_data(700, d, seed=d + m + nbits, dup=40), dt)
    hp = lb.HnswBuildParams(max_level=5, m=m, ef_construction=efc)
    ix = lb.IvfHnswPqIndex.build(x, metric, _params(M, nbits), hp, **kw)
    pq = lb.IvfPqIndex.build(x, metric, _params(M, nbits), **kw).export()
    got = ix.export()
    for key in ("centroids", "codebook", "part_offsets", "codes", "row_ids"):
        assert np.array_equal(got[key], pq[key]), key
    _assert_graph_equal(got["graph"], _ref_build(got, nbits, metric, dt, m=m, max_level=5, efc=efc, seed=5))


def _part_ids(offs):
    return np.repeat(np.arange(len(offs) - 1, dtype=np.uint32), np.diff(np.asarray(offs, np.int64)))


@pytest.mark.gpu
@pytest.mark.parametrize("nbits", [8, 4])
def test_build_small_partitions_bit_identical(nbits):
    """a device build over many small partitions (fewer rows than m, duplicated rows), and a graph with an empty, a
    one-row and a three-row partition loaded through from_parts and searched"""
    x = _data(400, 16, seed=9, dup=60)
    ix = lb.IvfHnswPqIndex.build(x, "l2", _params(4, nbits, K=30))
    got = ix.export()
    assert np.diff(got["part_offsets"].astype(np.int64)).min() < 20
    _assert_graph_equal(got["graph"], _ref_build(got, nbits, "l2", "f32", seed=5))
    cb = got["codebook"]
    codes = _codes(160, 4, nbits, 4)
    codes[-30:] = codes[:30]
    part = np.random.default_rng(4).integers(3, 6, 160).astype(np.uint32)
    part[:1], part[1:4] = 1, 2
    cent = _data(6, 16, seed=3)
    base = lb.IvfPqIndex.from_parts(cent, cb, part, codes, np.arange(160, dtype=np.uint64), num_bits=nbits).export()
    offs = base["part_offsets"].astype(np.int64)
    assert offs[1] - offs[0] == 0 and offs[2] - offs[1] == 1 and offs[3] - offs[2] == 3
    g = pr.build(base["codes"], base["part_offsets"], cb, nbits, "l2")
    ix2 = lb.IvfHnswPqIndex.from_parts(cent, cb, part, codes, np.arange(160, dtype=np.uint64), num_bits=nbits, graph=g)
    _assert_graph_equal(ix2.export()["graph"], g)
    q = _data(5, 16, seed=2)
    ids, d = ix2.search(q, k=5, nprobes=6)
    wi, wd, _ = pr.search(cent, cb, nbits, base["part_offsets"], base["codes"], base["row_ids"], g, q, 5, 6)
    assert np.array_equal(ids, wi) and np.array_equal(d.view(np.uint32), wd.view(np.uint32))


# ---- GPU: search --------------------------------------------------------------------------------------------------
def _index(metric="l2", n=1500, d=16, M=4, nbits=8, K=4, m=8, efc=40, seed=0):
    x = _data(n, d, seed=seed, dup=50)
    ix = lb.IvfHnswPqIndex.build(x, metric, _params(M, nbits, K=K, seed=seed),
                                 lb.HnswBuildParams(max_level=4, m=m, ef_construction=efc))
    return x, ix, ix.export()


def _ref_search(parts, metric, q, k, nprobes, nbits=8, **kw):
    return pr.search(parts["centroids"], parts["codebook"], nbits, parts["part_offsets"], parts["codes"],
                     parts["row_ids"], parts["graph"], q, k, nprobes, metric=metric, **kw)


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
@pytest.mark.parametrize("metric", ["l2", "dot"])
@pytest.mark.parametrize("d,M", [(16, 4), (32, 4), (64, 4), (36, 6)])     # sub-vector widths 4, 8, 16 and 6
def test_search_4bit_and_every_width_bit_identical(metric, d, M):
    """every width the IVF_PQ kind searches, 8-bit and 4-bit: an index opened from parts with the restatement's graph"""
    n, K = 600, 3
    x = _data(n, d, seed=d + M)
    cent = _data(K, d, seed=1)
    part = np.random.default_rng(2).integers(0, K, n).astype(np.uint32)
    q = _data(8, d, seed=78)
    for nbits in (8, 4):
        cb = _codebook(M, nbits, d // M, d)
        codes = _codes(n, M, nbits, d + 1)
        base = lb.IvfPqIndex.from_parts(cent, cb, part, codes, np.arange(n, dtype=np.uint64), metric,
                                        num_bits=nbits).export()
        g = pr.build(base["codes"], base["part_offsets"], cb, nbits, metric, m=6, max_level=3, efc=24, seed=1)
        ix = lb.IvfHnswPqIndex.from_parts(cent, cb, part, codes, np.arange(n, dtype=np.uint64), metric,
                                          num_bits=nbits, graph=g)
        parts = dict(base, graph=g)
        for k, ef in ((10, None), (30, 60)):
            ids, dist = ix.search(q, k=k, nprobes=2, ef=ef)
            wi, wd, _ = _ref_search(parts, metric, q, k, 2, nbits=nbits, ef=ef)
            assert np.array_equal(dist.view(np.uint32), wd.view(np.uint32)), (nbits, k)
            assert np.array_equal(ids, wi), (nbits, k)


@pytest.mark.gpu
def test_ef_below_k_is_refused():
    _, ix, _ = _index()
    with pytest.raises(lb.LanceB200Error) as e:
        ix.search(_data(2, 16, seed=1), k=10, nprobes=1, ef=9)
    assert e.value.status == lb._lib.INVALID_ARG


def _bitmap(bits):
    bm = np.packbits(bits, bitorder="little")
    return np.concatenate([bm, np.zeros((-bm.size) % 8, np.uint8)]).view(np.uint64)


@pytest.mark.gpu
@pytest.mark.parametrize("nbits", [8, 4])
@pytest.mark.parametrize("side", [-1, 0, 1])
def test_prefilter_either_side_of_the_switch(nbits, side):
    x, ix, parts = _index(K=1, nbits=nbits)
    n = x.shape[0]
    want = n * 10 // 100 + side        # side -1: flat branch; 0, 1: the graph
    rng = np.random.default_rng(3)
    bits = np.zeros(n, bool)
    bits[np.sort(rng.choice(n, want, replace=False))] = True
    q = _data(8, 16, seed=5)
    ids, d = ix.search_ex(q, k=10, nprobes=1, allow_bitmap=_bitmap(bits))
    wi, wd, _ = _ref_search(parts, "l2", q, 10, 1, nbits=nbits, allow_bits=bits)
    assert np.array_equal(d.view(np.uint32), wd.view(np.uint32))
    assert np.array_equal(ids, wi)
    if side == -1 and nbits == 8:
        # the flat branch scores every allowed row from the IVF_PQ scan's table: IVF_PQ's prefiltered search returns
        # the same distances.  (4-bit: HNSW sums pair sums, the IVF_PQ scan adds the two entries one at a time, so
        # their last bits may differ.)
        pq = lb.IvfPqIndex.from_parts(parts["centroids"], parts["codebook"], np.zeros(n, np.uint32), parts["codes"],
                                      parts["row_ids"])
        pi, pd = pq.search_ex(q, k=10, nprobes=1, allow_bitmap=_bitmap(bits))
        assert np.array_equal(pd.view(np.uint32), d.view(np.uint32))


@pytest.mark.gpu
@pytest.mark.parametrize("flat", [False, True])
def test_range_bounds_on_rows(flat):
    x, ix, parts = _index(K=1)
    n = x.shape[0]
    q = _data(4, 16, seed=6)
    _, d0 = ix.search(q, k=30, nprobes=1)
    lower, upper = float(d0[0, 3]), float(d0[0, 20])     # rows exactly on both bounds
    bits = np.ones(n, bool)
    if flat:                                             # 5 % of the rows allowed: the flat branch
        bits[:] = False
        bits[:n // 20] = True
    ids, d = ix.search_ex(q, k=30, nprobes=1, allow_bitmap=_bitmap(bits), lower_bound=lower, upper_bound=upper)
    wi, wd, _ = _ref_search(parts, "l2", q, 30, 1, allow_bits=bits, lower=lower, upper=upper)
    assert np.array_equal(d.view(np.uint32), wd.view(np.uint32))
    assert np.array_equal(ids, wi)


def _refined(x, q, cand, k):
    """the refine step over one candidate list per query: exact distances, the k smallest by (distance, row id)"""
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
    qd = lb.DeviceArray.from_numpy(q)
    oi, od = lb.DeviceArray((6, 10), np.uint64), lb.DeviceArray((6, 10), np.float32)
    ix.search_async(qd, (oi, od), k=10, nprobes=2)
    lb.synchronize()
    wi, wd, _ = _ref_search(parts, "l2", q, 10, 2)
    assert np.array_equal(oi.numpy(), wi) and np.array_equal(od.numpy().view(np.uint32), wd.view(np.uint32))


@pytest.mark.gpu
def test_combined_search_bit_identical():
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
@pytest.mark.parametrize("dt", ["f32", "bf16"])
def test_graph_from_reference_with_other_m_searches_identically(dt):
    x, kw = _typed(_data(1500, 16, seed=0, dup=50), dt)
    ix = lb.IvfHnswPqIndex.build(x, "dot", _params(4, 8, K=4), lb.HnswBuildParams(max_level=4, m=8, ef_construction=40),
                                 **kw)
    parts = ix.export()
    g = _ref_build(parts, 8, "dot", dt, m=5, max_level=3, efc=20, seed=11)
    opts = dict(distance_type="dot", bf16=dt == "bf16")
    ix2 = lb.IvfHnswPqIndex.from_parts(parts["centroids"], parts["codebook"], _part_ids(parts["part_offsets"]),
                                       parts["codes"], parts["row_ids"], graph=g, **opts)
    parts2 = dict(parts, graph=g)
    q, _ = _typed(_data(10, 16, seed=12), dt)
    qf = q if dt != "bf16" else (q.astype(np.uint32) << 16).view(np.float32)
    for k, ef in ((10, None), (10, 40), (50, None)):
        ids, d = ix2.search(q, k=k, nprobes=3, ef=ef)
        wi, wd, _ = _ref_search(parts2, "dot", qf, k, 3, ef=ef)
        assert np.array_equal(d.view(np.uint32), wd.view(np.uint32))
        assert np.array_equal(ids, wi)
    e = ix2.export()
    ix3 = lb.IvfHnswPqIndex.from_parts(parts["centroids"], parts["codebook"], _part_ids(e["part_offsets"]), e["codes"],
                                       e["row_ids"], graph=e["graph"], **opts)
    _assert_graph_equal(ix3.export()["graph"], g)
    assert np.array_equal(ix3.search(q, k=10, nprobes=3)[0], ix2.search(q, k=10, nprobes=3)[0])
    # a device build and a load of its own export search alike
    ix4 = lb.IvfHnswPqIndex.from_parts(parts["centroids"], parts["codebook"], _part_ids(parts["part_offsets"]),
                                       parts["codes"], parts["row_ids"], graph=parts["graph"], **opts)
    for a, b in zip(ix4.search(q, k=10, nprobes=3, ef=30), ix.search(q, k=10, nprobes=3, ef=30)):
        assert np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8))


@pytest.mark.gpu
def test_graph_index_refusals():
    x, ix, parts = _index()
    with pytest.raises(lb.LanceB200Error) as e:
        ix.update(add_part_ids=np.zeros(1, np.uint32), add_codes=parts["codes"][:1],
                  add_row_ids=np.array([9999], np.uint64))
    assert e.value.status == lb._lib.UNSUPPORTED and "IVF_HNSW_PQ" in str(e.value)
    with pytest.raises(lb.LanceB200Error) as e:
        ix.repartition()
    assert e.value.status == lb._lib.UNSUPPORTED and "IVF_HNSW_PQ" in str(e.value)
    with pytest.raises(lb.LanceB200Error) as e:
        lb._lib.check(lb._lib.lib().lb2_index_load(ix._h, None, None, None, lb._lib.C.c_uint64(0)))
    assert "already has an HNSW graph" in str(e.value)
    with pytest.raises(lb.LanceB200Error):      # an IVF_HNSW_PQ graph is not an IVF_HNSW_SQ one
        lb._lib.check(lb._lib.lib().lb2_index_hnsw_sq_info(ix._h, None, None, None, None))
    bad = dict(parts["graph"])
    bad["neighbors0"] = bad["neighbors0"].copy()
    bad["neighbors0"][5, 0] = 10 ** 6                  # a neighbour outside its partition
    with pytest.raises(lb.LanceB200Error) as e:
        lb.IvfHnswPqIndex.from_parts(parts["centroids"], parts["codebook"], _part_ids(parts["part_offsets"]),
                                     parts["codes"], parts["row_ids"], graph=bad)
    assert e.value.status == lb._lib.INVALID_ARG and "IVF_HNSW_PQ" in str(e.value)


@pytest.mark.gpu
@pytest.mark.parametrize("metric,floor", [("l2", 0.9), ("cosine", 0.9), ("dot", 0.85)])
def test_recall_floor(metric, floor):
    """test_create_ivf_hnsw_pq (rust/lance/src/index/vector/ivf/v2.rs:1497-1524 via test_recall): 512 x 32 uniform
    [0, 1) rows, nlist 4, PQ 16 x 8-bit, the query row 0, k = 100, nprobes = nlist, against the exact ground truth"""
    rng = np.random.default_rng(0)
    x = rng.random((512, 32)).astype(np.float32)
    ix = lb.IvfHnswPqIndex.build(x, metric, lb.IvfBuildParams(num_partitions=4, num_sub_vectors=16))
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
