"""The HNSW graph engine (lance_b200/csrc/hnsw.cu) of IVF_HNSW_SQ, IVF_HNSW_PQ and IVF_HNSW_FLAT at the shapes where its
launch loops turn over and at its table, tail and parameter limits, against the three restatements of the reference
(tests/hnsw_reference.py, hnsw_pq_reference.py, hnsw_flat_reference.py), bit for bit: graphs (levels, every list's ids,
distances and order), search ids, distance bits and counts.

  1. build grid turnover: more partitions with >= 2 rows than build warps, so every warp builds several partitions,
     largest first, on the scratch a larger one left behind (PQ: 8-bit M = 256 tables, where the scratch cap binds);
  2. search grid turnover: more (query, probe) slots than search warps, with a prefilter that sends some partitions to
     the flat branch and others to the graph, so one warp takes both across its loop;
  3. past one query slab (SEARCH_SLAB queries), and past one candidate sub-slab of the probed search;
  4. PQ tables of 8-bit M = 128 and 256 and 4-bit M = 256;
  5. the flat rule's d % 16 tail groups (d = 4, 12, 44, 140) for every metric and column type;
  6. the parameter limits: max_level 1 and 64, m 1, 2 and 64, ef_construction 1.

Every regime test asserts that it reached its regime: the warp counts are computed with hnsw.cu's scratch formula and
launch counts come from lb.profile, so a later change to a cap cannot void a test without failing it."""
import numpy as np
import pytest

import flat_reference as fr
import hnsw_flat_reference as hf
import hnsw_pq_reference as pr
import hnsw_reference as hr
import lance_b200 as lb
from oracle import binding as ob
from test_ivf_hnsw_sq import _assert_graph_equal, _data, _typed

SEARCH_SLAB = 32768        # ivf_search.cuh
KINDS = ["sq", "pq", "flat"]


# ---- the engine's grid sizes, restated from hnsw.cu ----------------------------------------------------------------
def _num_sms():
    import torch  # device properties only
    return torch.cuda.get_device_properties(0).multi_processor_count


def _scratch_words(nmax, E, B, LB, TW=0, QW=0):
    """hnsw.cu scratch_words: the u32 words of one warp's scratch"""
    w = TW + QW + (nmax + 31) // 32 + 2 * (nmax + 1) + 2 * (E + 1) + 4 * B + 3 * LB
    return (w + 3) & ~3 if TW or QW else w


def _policy_words(kind, d, M=0, nbits=8):
    """hnsw.cu pq_table_words / query_words: (TW, QW) of a kind's warp"""
    return (M << nbits if kind == "pq" else 0), ((d + 3) & ~3 if kind in ("pq", "flat") else 0)


def _build_grid(nparts2, nmax, m, efc, TW, QW):
    """hnsw.cu build_graphs: (warps, fit) for nparts2 partitions of >= 2 rows, the largest of nmax rows"""
    E, B = efc, 2 * m + 1
    words = _scratch_words(nmax, E, B, max(E, B), TW, QW)
    fit = max(1, (512 << 20) // (words * 4))
    return min(nparts2, 32 * _num_sms(), fit), fit


def _search_grid(nmax, k, ef, m, TW, QW):
    """hnsw.cu search_graphs: cap, the most warps of one search launch"""
    ef = k + k // 2 if ef is None else ef
    E, B = max(ef, k), max(2 * m, 32)
    words = _scratch_words(max(nmax, 1), E, B, 0, TW, QW)
    return max(1, min(32 * _num_sms(), (256 << 20) // (words * 4)))


def _probed_sub(nl, k):
    """ivf_search.cu ivf_search_probed: the queries of one candidate sub-slab"""
    return max(1, (256 << 20) // (nl * k * 12 + 4 * nl))


def _launches(fn, name):
    """fn()'s result and the launches of kernel family `name` under any tag"""
    lb.profile.reset()
    lb.profile.enable(True)
    try:
        out = fn()
    finally:
        lb.profile.enable(False)
    return out, sum(v[0] for key, v in lb.profile.dump().items() if key.split(":")[-1] == name)


# ---- building and restating each kind ------------------------------------------------------------------------------
def _build(kind, x, metric, K, hp, kw=None, centroids=None, M=4, nbits=8, seed=5):
    """a device build; given centroids: one Lloyd iteration from them"""
    kw = kw or {}
    iters = 1 if centroids is not None else 10
    if kind == "pq":
        params = lb.IvfBuildParams(num_partitions=K, num_sub_vectors=M, num_bits=nbits, max_iters=iters, pq_max_iters=4,
                                   seed=seed, centroids=centroids)
        return lb.IvfHnswPqIndex.build(x, metric, params, hp, **kw)
    cls = lb.IvfHnswSqIndex if kind == "sq" else lb.IvfHnswFlatIndex
    return cls.build(x, metric, num_partitions=K, max_iters=iters, seed=seed, centroids=centroids, hnsw_params=hp, **kw)


def _ref_build(kind, parts, metric, hp, dt="f32", nbits=8, seed=5):
    g = dict(m=hp.m, max_level=hp.max_level, efc=hp.ef_construction, seed=seed)
    if kind == "sq":
        return hr.build(parts["codes"], parts["part_offsets"], parts["bounds"], "dot" if metric == "dot" else "l2", **g)
    if kind == "pq":
        return pr.build(parts["codes"], parts["part_offsets"], parts["codebook"], nbits, metric, dt, **g)
    return hf.build(parts["vectors"], parts["part_offsets"], metric, dt, **g)


def _ref_search(kind, parts, metric, q, k, nprobes, dt="f32", nbits=8, **kw):
    """the restatement's search; q as f32 values"""
    if kind == "sq":
        return hr.search(parts["centroids"], parts["bounds"], parts["part_offsets"], parts["codes"], parts["row_ids"],
                         parts["graph"], q, k, nprobes, metric=metric, **kw)
    if kind == "pq":
        return pr.search(parts["centroids"], parts["codebook"], nbits, parts["part_offsets"], parts["codes"],
                         parts["row_ids"], parts["graph"], q, k, nprobes, metric=metric, **kw)
    return hf.search(parts["centroids"], parts["part_offsets"], parts["vectors"], parts["row_ids"], parts["graph"], q, k,
                     nprobes, metric=metric, dt=dt, **kw)


def _tw_qw(kind, parts, nbits=8):
    d = parts["centroids"].shape[1]
    return _policy_words(kind, d, parts["codebook"].shape[0] if kind == "pq" else 0, nbits)


def _nmax(parts):
    return int(np.diff(parts["part_offsets"].astype(np.int64)).max())


def _bitmap(bits):
    bm = np.packbits(bits, bitorder="little")
    return np.concatenate([bm, np.zeros((-bm.size) % 8, np.uint8)]).view(np.uint64)


def _assert_unused_slots_zero(g):
    """build_graphs zeroes every list slot past its count: ids and distance bits"""
    for c, ids, dist in ((g["counts0"], g["neighbors0"], g["dists0"]), (g["counts_up"], g["neighbors_up"], g["dists_up"])):
        unused = np.arange(ids.shape[1])[None, :] >= np.asarray(c, np.int64)[:, None]
        assert not ids[unused].any() and not dist.view(np.uint32)[unused].any()


def _assert_same(got, want, what=""):
    """(ids, dists[, counts]) bit for bit"""
    assert np.array_equal(got[0], want[0]), what
    assert np.array_equal(np.asarray(got[1], np.float32).view(np.uint32),
                          np.asarray(want[1], np.float32).view(np.uint32)), what
    if len(got) > 2 and len(want) > 2:
        assert np.array_equal(got[2], want[2]), what


# ---- CPU: the restatement at the parameter limits -----------------------------------------------------------------
LIMITS = [(1, 4, 8), (64, 1, 4), (64, 2, 16), (4, 64, 300), (4, 8, 1)]   # (max_level, m, ef_construction)


def test_reference_levels_at_the_limits():
    assert hr.node_levels(3, 1, 500, 1, 64) == [64] * 500                    # m = 1: every node on every level
    assert hr.node_levels(3, 1, 500, 4, 1) == [1] * 500                      # max_level = 1: level 0 only
    thr = hr.thresholds(2, 64)                                              # m = 2: the thresholds reach 0 at 2^33
    assert thr[32] == 1 and thr[33:] == [0] * 31
    lv = np.array(hr.node_levels(3, 1, 20000, 2, 64))
    assert lv[0] == 64 and lv[1:].max() < 34


@pytest.mark.parametrize("max_level,m,efc", LIMITS)
def test_reference_graph_at_the_limits(max_level, m, efc):
    rng = np.random.default_rng(m + efc)
    codes = rng.integers(0, 256, (260, 8), dtype=np.uint8)
    codes[-10:] = codes[:10]
    offs = np.array([0, 1, 260], np.uint64)
    g = hr.build(codes, offs, (-1.0, 2.0), "l2", m=m, max_level=max_level, efc=efc, seed=3)
    lv = g["levels"].astype(np.int64)
    c0, cu = g["counts0"].astype(np.int64), g["counts_up"].astype(np.int64)
    assert (c0 <= 2 * m).all() and (cu <= m).all()                           # degrees
    assert len(cu) == int((lv - 1).sum()) and lv[0] == lv[1] == max_level
    if max_level == 1:
        assert len(cu) == 0 and g["neighbors_up"].shape == (0, m)            # no upper-level rows
    if m == 1:
        assert (lv == max_level).all() and len(cu) == 260 * (max_level - 1)
    if m == 64:
        assert c0.max() > 96                                                 # lists past three warp widths
    up = np.concatenate([[0], np.cumsum(lv - 1)])
    for r in range(1, 260):
        nb = g["neighbors0"][r, :c0[r]].astype(np.int64)
        assert (nb < 259).all() and len(set(nb.tolist())) == len(nb)
        for level in range(1, lv[r]):
            u = up[r] + level - 1
            nb = g["neighbors_up"][u, :cu[u]].astype(np.int64)
            assert (lv[1 + nb] > level).all() and len(set(nb.tolist())) == len(nb)
    assert c0[1:].min() > 0                                                  # the 259-row partition is connected


# ---- GPU 1, 2: build and search grid turnover ----------------------------------------------------------------------
def _cluster_sizes(nparts, seed):
    """mostly 2 to 5 rows, every twelfth partition 17 or 40 rows"""
    sizes = np.random.default_rng(seed).integers(2, 6, nparts)
    big = np.arange(0, nparts, 12)
    sizes[big] = np.where(np.arange(big.size) % 2 == 0, 17, 40)
    return sizes


def _clusters(sizes, d, seed, spread=2.0):
    """tight clusters around distinct points of the lattice {-100, 0, 100}^8 (the first 8 dimensions), far apart
    against their spread; rows in partition order, and the centres"""
    rng = np.random.default_rng(seed)
    idx = rng.choice(3 ** 8, sizes.size, replace=False)
    digits = (idx[:, None] // 3 ** np.arange(8)[None, :]) % 3
    cent = np.zeros((sizes.size, d), np.float32)
    cent[:, :8] = (digits - 1) * 100.0
    x = (np.repeat(cent, sizes, axis=0) + spread * rng.standard_normal((int(sizes.sum()), d))).astype(np.float32)
    return x, cent


TURNOVER = [("sq", 8, 0, 4500), ("flat", 8, 0, 4500), ("pq", 1024, 256, 2150), ("pq", 512, 256, 2150)]
TURNOVER_HP = lb.HnswBuildParams(max_level=3, m=4, ef_construction=12)


@pytest.fixture(scope="module", params=TURNOVER, ids=lambda c: f"{c[0]}-d{c[1]}")
def turnover(request):
    kind, d, M, nparts = request.param
    sizes = _cluster_sizes(nparts, seed=d)
    x, cent = _clusters(sizes, d, seed=d + 1)
    start = np.stack([x[a:b].mean(axis=0) for a, b in zip(np.cumsum(sizes) - sizes, np.cumsum(sizes))])
    ix = _build(kind, x, "l2", nparts, TURNOVER_HP, centroids=start, M=M)
    parts = ix.export()
    assert np.array_equal(np.diff(parts["part_offsets"].astype(np.int64)), sizes)   # one partition per cluster
    return kind, ix, parts, sizes, cent


@pytest.mark.gpu
def test_build_grid_turnover(turnover):
    kind, ix, parts, sizes, _ = turnover
    TW, QW = _tw_qw(kind, parts)
    nparts2 = int((sizes >= 2).sum())
    warps, fit = _build_grid(nparts2, int(sizes.max()), TURNOVER_HP.m, TURNOVER_HP.ef_construction, TW, QW)
    assert nparts2 > warps                                    # every warp builds more than one partition
    if kind == "pq":
        assert fit < 32 * _num_sms() and warps == fit         # the 256 KB tables make the scratch cap bind
    g = parts["graph"]
    _assert_unused_slots_zero(g)
    _assert_graph_equal(g, _ref_build(kind, parts, "l2", TURNOVER_HP))


@pytest.mark.gpu
def test_search_grid_turnover(turnover):
    """more (query, probe) slots than warps, every warp at least two; partitions of 40 rows alternate between 2 allowed
    rows (the flat branch) and all rows (the graph), the small ones allow three rows in four (the graph)"""
    kind, ix, parts, sizes, cent = turnover
    k, nprobes = 10, 4
    TW, QW = _tw_qw(kind, parts)
    cap = _search_grid(int(sizes.max()), k, None, TURNOVER_HP.m, TW, QW)
    nq = 2 * cap // nprobes + 97
    rng = np.random.default_rng(7)
    bits = rng.random(int(sizes.sum())) < 0.75
    offs = parts["part_offsets"].astype(np.int64)
    forty = np.flatnonzero(sizes == 40)
    for j, p in enumerate(forty):
        bits[offs[p]:offs[p + 1]] = j % 2 == 1
        if j % 2 == 0:
            bits[offs[p] + 3] = bits[offs[p] + 29] = True
    pick = np.where(rng.random(nq) < 0.5, rng.choice(forty[::2], nq), rng.integers(0, sizes.size, nq))
    q = (cent[pick] + 2.0 * rng.standard_normal((nq, cent.shape[1]))).astype(np.float32)
    # the regime: each warp's slots (slot = query * nprobes + probe, warp = slot % cap) take both branches
    acnt = np.add.reduceat(bits.astype(np.int64), offs[:-1])
    flat = acnt < sizes * 10 // 100
    assert flat.any() and not flat.all()
    slots = np.concatenate([ob.find_partitions(parts["centroids"], q[i], nprobes)[0] for i in range(nq)])
    assert slots.size > 2 * cap
    per_warp = np.zeros((cap, 2), bool)
    per_warp[np.arange(slots.size) % cap, flat[slots].astype(np.int64)] = True
    assert per_warp.all(axis=1).sum() > cap // 20, per_warp.all(axis=1).sum()
    (ids, dist), launches = _launches(lambda: ix.search_ex(q, k=k, nprobes=nprobes, allow_bitmap=_bitmap(bits)),
                                      "hnsw_search")
    assert launches == 1
    _assert_same((ids, dist), _ref_search(kind, parts, "l2", q, k, nprobes, allow_bits=bits))


# ---- GPU 3: past one query slab and one candidate sub-slab ---------------------------------------------------------
SLAB_HP = lb.HnswBuildParams(max_level=4, m=8, ef_construction=40)


def _small_index(kind, seed=0):
    x = _data(1500, 16, seed=seed, dup=50)
    ix = _build(kind, x, "l2", 4, SLAB_HP, seed=seed)
    return ix, ix.export()


def _chunked(fn, nq, chunk):
    parts = [fn(a, min(nq, a + chunk)) for a in range(0, nq, chunk)]
    return tuple(np.concatenate([p[i] for p in parts]) for i in range(len(parts[0])))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_search_past_one_slab(kind):
    ix, parts = _small_index(kind)
    k, nprobes = 10, 2
    nq = SEARCH_SLAB + 77
    q = _data(nq, 16, seed=31)
    cap = _search_grid(_nmax(parts), k, None, SLAB_HP.m, *_tw_qw(kind, parts))
    got, launches = _launches(lambda: ix.search(q, k=k, nprobes=nprobes), "hnsw_search")
    assert launches == 2                                     # two slabs
    # the same queries in chunks of one grid pass each
    want = _chunked(lambda a, b: ix.search(q[a:b], k=k, nprobes=nprobes), nq, cap // nprobes)
    _assert_same(got, want)
    sample = np.r_[0:3, SEARCH_SLAB - 20:SEARCH_SLAB + 21, nq - 3:nq]
    wi, wd, _ = _ref_search(kind, parts, "l2", q[sample], k, nprobes)
    _assert_same((got[0][sample], got[1][sample]), (wi, wd))
    # search_probed at minimum = maximum nprobes: its own slabs, the same results
    (pi, pd, pc, pn), launches = _launches(
        lambda: ix.search_probed(q, k, minimum_nprobes=nprobes, maximum_nprobes=nprobes, ef=k + k // 2), "hnsw_search")
    assert launches == 2 and (pn == nprobes).all()
    _assert_same((pi, pd), got)
    # a range bound: every probe is scanned and the cutoff reads the lists (by_scan), over two slabs as well
    lower, upper = float(np.median(got[1][:, 0])), float(np.median(got[1][:, -1]))
    (ri, rd, rc, _), launches = _launches(
        lambda: ix.search_probed(q, k, minimum_nprobes=nprobes, maximum_nprobes=nprobes, lower_bound=lower,
                                 upper_bound=upper, ef=k + k // 2), "hnsw_search")
    assert launches == 2
    want = _chunked(lambda a, b: ix.search_ex(q[a:b], k=k, nprobes=nprobes, lower_bound=lower, upper_bound=upper),
                    nq, cap // nprobes)
    _assert_same((ri, rd), want)
    assert 0 < rc[sample].sum() < k * sample.size
    wi, wd, wc = _ref_search(kind, parts, "l2", q[sample], k, nprobes, lower=lower, upper=upper)
    _assert_same((ri[sample], rd[sample], rc[sample]), (wi, wd, wc))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_search_probed_past_one_sub_slab(kind):
    """k = 1024 at 4 probes: the probed search's candidate lists split the queries into sub-slabs"""
    ix, parts = _small_index(kind, seed=1)
    k, nprobes = 1024, 4
    sub = _probed_sub(nprobes, k)
    nq = sub + 500
    assert nq < SEARCH_SLAB
    q = _data(nq, 16, seed=32)
    (pi, pd, pc, _), launches = _launches(
        lambda: ix.search_probed(q, k, minimum_nprobes=nprobes, maximum_nprobes=nprobes), "hnsw_search")
    assert launches == 2                                     # two sub-slabs
    ids, dist = ix.search(q, k=k, nprobes=nprobes)
    _assert_same((pi, pd), (ids, dist))
    sample = np.r_[0:2, sub - 3:sub + 3, nq - 2:nq]
    wi, wd, wc = _ref_search(kind, parts, "l2", q[sample], k, nprobes)
    _assert_same((pi[sample], pd[sample], pc[sample]), (wi, wd, wc))


# ---- GPU 4: PQ at large M ------------------------------------------------------------------------------------------
LARGE_M = [(128, 8, 512), (256, 8, 256), (256, 4, 512)]   # (M, nbits, d): sub-vector widths 4, 1 and 2


@pytest.mark.gpu
@pytest.mark.parametrize("M,nbits,d", LARGE_M)
def test_pq_large_tables(M, nbits, d):
    hp = lb.HnswBuildParams(max_level=4, m=6, ef_construction=24)
    x = _data(700, d, seed=M + nbits, dup=30)
    ix = _build("pq", x, "l2", 2, hp, M=M, nbits=nbits)
    parts = ix.export()
    assert parts["codebook"].shape[:2] == (M, 1 << nbits)
    _assert_graph_equal(parts["graph"], _ref_build("pq", parts, "l2", hp, nbits=nbits))
    q = _data(10, d, seed=9)
    for k, ef in ((10, None), (20, 60)):
        got = ix.search(q, k=k, nprobes=2, ef=ef)
        wi, wd, _ = _ref_search("pq", parts, "l2", q, k, 2, nbits=nbits, ef=ef)
        _assert_same(got, (wi, wd), (k, ef))
    # 5 % of the rows allowed: the flat branch in both partitions
    n = x.shape[0]
    bits = np.zeros(n, bool)
    bits[np.random.default_rng(2).choice(n, n // 20, replace=False)] = True
    got = ix.search_ex(q, k=10, nprobes=2, allow_bitmap=_bitmap(bits))
    wi, wd, _ = _ref_search("pq", parts, "l2", q, 10, 2, nbits=nbits, allow_bits=bits)
    _assert_same(got, (wi, wd))
    if M == 128 and nbits == 8:
        # the table still fits shared memory: IVF_PQ's prefiltered search gives the flat branch's distances
        pq = lb.IvfPqIndex.from_parts(parts["centroids"], parts["codebook"], np.repeat(
            np.arange(2, dtype=np.uint32), np.diff(parts["part_offsets"].astype(np.int64))), parts["codes"],
            parts["row_ids"])
        _, pd = pq.search_ex(q, k=10, nprobes=2, allow_bitmap=_bitmap(bits))
        assert np.array_equal(pd.view(np.uint32), got[1].view(np.uint32))


# ---- GPU 5: the flat rule's tail groups ----------------------------------------------------------------------------
TAIL_D = [4, 12, 44, 140]     # d % 16 = 4, 12, 12, 12; 16-bit rows of 44 and 140 elements alternate 16-byte alignment


def _f32(x, dt):
    return hf.stored_f32(x, dt)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["f32", "f16", "bf16"])
@pytest.mark.parametrize("d", TAIL_D)
def test_cosine_rule_is_the_ivf_flat_scan_at_tails(dt, d):
    n = 300
    x, kw = _typed(_data(n, d, seed=d), dt)
    q, _ = _typed(_data(6, d, seed=d + 50), dt)
    ix = lb.IvfFlatIndex.from_parts(np.zeros((1, d), np.float32), np.zeros(n, np.uint32), x,
                                    np.arange(n, dtype=np.uint64), "cosine", **kw)
    ids, dist = ix.search(q, k=n, nprobes=1)
    D = hf.distances(ob.normalize_rows(_f32(q, dt)), _f32(x, dt), "cosine")
    for r in range(q.shape[0]):
        o = np.lexsort((np.arange(n), fr.total_order_key(D[r])))
        assert np.array_equal(ids[r], o.astype(np.uint64))
        assert np.array_equal(dist[r].view(np.uint32), D[r, o].view(np.uint32))


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["f32", "f16", "bf16", "u8"])
@pytest.mark.parametrize("metric", ["l2", "cosine", "dot"])
@pytest.mark.parametrize("d", TAIL_D)
def test_flat_tails_build_and_search(d, metric, dt):
    hp = lb.HnswBuildParams(max_level=4, m=6, ef_construction=24)
    x, kw = _typed(_data(400, d, seed=d + 3, dup=20), dt)
    ix = _build("flat", x, metric, 2, hp, kw)
    parts = ix.export()
    _assert_graph_equal(parts["graph"], _ref_build("flat", parts, metric, hp, dt=dt))
    q, _ = _typed(_data(8, d, seed=d + 4), dt)
    got = ix.search(q, k=10, nprobes=2)
    wi, wd, _ = _ref_search("flat", parts, metric, _f32(q, dt), 10, 2, dt=dt)
    _assert_same(got, (wi, wd))


# ---- GPU 6: the parameter limits -----------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("max_level,m,efc", LIMITS)
@pytest.mark.parametrize("kind", KINDS)
def test_parameter_limits(kind, max_level, m, efc):
    hp = lb.HnswBuildParams(max_level=max_level, m=m, ef_construction=efc)
    x = _data(400, 16, seed=m + efc, dup=20)
    ix = _build(kind, x, "l2", 2, hp)
    parts = ix.export()
    g = parts["graph"]
    assert g["max_level"] == max_level and g["m"] == m
    _assert_unused_slots_zero(g)
    _assert_graph_equal(g, _ref_build(kind, parts, "l2", hp))
    if m == 64:
        assert g["counts0"].max() > 96                         # lists past three warp widths
    q = _data(8, 16, seed=11)
    for k, ef in ((10, None), (10, _nmax(parts) + 20)):      # ef above the partition size
        got = ix.search(q, k=k, nprobes=2, ef=ef)
        wi, wd, _ = _ref_search(kind, parts, "l2", q, k, 2, ef=ef)
        _assert_same(got, (wi, wd), ef)
