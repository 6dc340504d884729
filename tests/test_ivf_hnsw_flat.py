"""IVF_HNSW_FLAT against the restatement of the reference (tests/hnsw_flat_reference.py): the exact FMA emulation, the
restatement's invariants and its distance matrix on the CPU, and on the device the restated cosine rule equal to
IVF_FLAT's scan, the IVF stage, vectors and row ids equal to IVF_FLAT's, the graphs bit for bit (levels, every list's
ids, distances and order) and every search result (ids, distances, counts) bit-identical."""
from fractions import Fraction

import numpy as np
import pytest

import flat_reference as fr
import hnsw_flat_reference as hf
import lance_b200 as lb
from oracle import binding as ob
from test_ivf_hnsw_sq import _assert_graph_equal, _data, _typed


def _f32(x, dt):
    """typed values (as _typed returns them) as f32"""
    return fr._f32(x, "bf16" if dt == "bf16" else "f32")


# ---- CPU: the FMA emulation ---------------------------------------------------------------------------------------
def _exact_fma(a, b, c):
    """fmaf by rational arithmetic: the exact a * b + c rounded to the nearest f32, ties to even"""
    a, b, c = np.float32(a), np.float32(b), np.float32(c)
    x = Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c))
    guess = np.float32(float(x))
    cands = [np.nextafter(guess, np.float32(-np.inf)), guess, np.nextafter(guess, np.float32(np.inf))]
    cands = [v for v in cands if np.isfinite(v)]
    err = [abs(Fraction(float(v)) - x) for v in cands]
    best = min(err)
    ties = [v for v, e in zip(cands, err) if e == best]
    return min(ties, key=lambda v: int(np.float32(v).view(np.uint32)) & 1)   # ties: the even mantissa


def _adversarial(rng, count):
    """ties at the f32 half-ulp, ties missed by less than an f64 ulp, exponent gaps and cancellations"""
    out = []
    for _ in range(count):
        c = np.float32(rng.uniform(1, 2) * 2.0 ** rng.integers(-20, 20))
        half = np.float64(np.spacing(c)) / 2                           # the half-ulp of c
        a = np.float32(rng.uniform(1, 2) * 2.0 ** rng.integers(-10, 10))
        b = np.float32(half / np.float64(a))                          # a * b lands on or next to the tie
        out.append((a, b, c))
        out.append((a, b, -c))
        out.append((a, np.nextafter(b, np.float32(np.inf)), c))
        out.append((np.float32(2.0 ** rng.integers(-60, -30)), a, c))   # a product far below c
        out.append((a, np.float32(2.0 ** rng.integers(30, 60)), c))      # c far below the product
        p = np.float32(np.float64(a) * np.float64(b))
        out.append((a, b, -p))                                         # cancellation: the product's rounding error
    return out


def test_fma_emulation_equals_exact_rounding():
    rng = np.random.default_rng(0)
    rand = [tuple(np.float32(v) for v in rng.standard_normal(3) * 2.0 ** rng.integers(-30, 30, 3)) for _ in range(3000)]
    cases = rand + _adversarial(rng, 400)
    a, b, c = (np.array(v, np.float32) for v in zip(*cases))
    got = hf.fma32(a, b, c)
    want = np.array([_exact_fma(*t) for t in cases], np.float32)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    # the adversarial set has teeth: rounding the f64 sum twice (to nearest) gets some of them wrong
    naive = (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(np.float32)
    assert (naive.view(np.uint32) != want.view(np.uint32)).sum() > 0


def test_fma_emulation_on_constructed_double_rounding():
    """a * b = 2^-24 + j 2^-70 with 0 < j < 2^17: 1 + a * b lies above the f32 tie 1 + 2^-24 by less than half an f64
    ulp, so the f64 sum rounds onto the tie and a second rounding to nearest-even gives 1; the exact result is
    1 + 2^-23.  a = a_m 2^-23 and b = b_m 2^-47 with 24-bit integers a_m b_m = 2^46 + j."""
    for t in range(1, 1 << 20):
        a_m = (1 << 23) + t
        b_m = -(-(1 << 46) // a_m)
        j = a_m * b_m - (1 << 46)
        if 0 < j < (1 << 17):
            break
    a, b, c = np.float32(a_m * 2.0 ** -23), np.float32(b_m * 2.0 ** -47), np.float32(1.0)
    assert Fraction(float(a)) * Fraction(float(b)) == Fraction(1, 1 << 24) + Fraction(j, 1 << 70)
    naive = np.float32(float(a) * float(b) + 1.0)
    assert naive == np.float32(1.0)
    assert hf.fma32(a, b, c) == np.float32(1 + 2.0 ** -23) == _exact_fma(a, b, c)
    assert hf.fma32(a, -b, -c) == np.float32(-(1 + 2.0 ** -23))


# ---- CPU: the restatement -----------------------------------------------------------------------------------------
def _cosine_scalar(q, y):
    """the COSINE rule of one pair, one element at a time through the exact rational fma"""
    xy, yy, qq = [np.float32(0)] * 16, [np.float32(0)] * 16, [np.float32(0)] * 16
    for e in range(len(q)):
        l = e % 16
        xy[l] = _exact_fma(q[e], y[e], xy[l])
        yy[l] = _exact_fma(y[e], y[e], yy[l])
        qq[l] = _exact_fma(q[e], q[e], qq[l])
    t = hf.tree16
    return np.float32(np.float32(1.0) - t(xy) / np.sqrt(t(qq)) / np.sqrt(t(yy)))


@pytest.mark.parametrize("d", [4, 20, 36])
def test_cosine_rule_equals_the_scalar_rule(d):
    x = _data(7, d, seed=d)
    P = hf.pair_matrix(x, "cosine")
    for u in range(7):
        for v in range(7):
            assert P[u, v].view(np.uint32) == _cosine_scalar(x[u], x[v]).view(np.uint32), (u, v)


def test_cosine_matrix_is_not_symmetric():
    """the two norms round separately, so dist_between(u, v) and dist_between(v, u) differ in the last bits for some
    pairs; the restatement's P[u][v] puts u in the query role.  (Rows of norm far from 1 show it most often; the
    stored rows are normalised, where it is rarer but still possible.)"""
    x = _data(200, 36, seed=3)
    P = hf.pair_matrix(x, "cosine")
    assert (P.view(np.uint32) != P.T.view(np.uint32)).any()
    for u, v in [(0, 1), (5, 190), (77, 3)]:
        assert P[u, v].view(np.uint32) == hf.cosine_rule(x[u:u + 1], x[v:v + 1])[0, 0].view(np.uint32)


@pytest.mark.parametrize("metric", ["l2", "dot"])
@pytest.mark.parametrize("d", [4, 20, 128])
def test_pair_matrix_is_the_flat_rule(metric, d):
    """L2 / dot: the 16-lane rule, pinned to the oracle's per-row functions; the two are symmetric bit for bit"""
    x = _data(24, d, seed=d + 1)
    P = hf.pair_matrix(x, metric)
    fn = ob.l2 if metric == "l2" else ob.dot
    for u in range(0, 24, 5):
        for v in range(0, 24, 3):
            want = np.float32(fn(x[u], x[v]))
            if metric == "dot":
                want = np.float32(1.0) - want
            assert want.view(np.uint32) == P[u, v].view(np.uint32), (u, v)
    assert np.array_equal(P.view(np.uint32), P.T.view(np.uint32))


@pytest.mark.parametrize("metric", ["l2", "cosine", "dot"])
@pytest.mark.parametrize("m,efc", [(20, 150), (4, 8)])
def test_reference_graph_invariants(metric, m, efc):
    x = _data(300, 12, seed=1, dup=20)
    if metric == "cosine":
        x = ob.normalize_rows(x)
    offs = np.array([0, 0, 1, 4, 300], np.uint64)
    g = hf.build(x, offs, metric, m=m, max_level=5, efc=efc, seed=3)
    lv = g["levels"].astype(np.int64)
    assert (g["counts0"] <= 2 * m).all() and (g["counts_up"] <= m).all()          # degrees
    assert len(g["counts_up"]) == int((lv - 1).sum())                             # level counts add up
    up = np.concatenate([[0], np.cumsum(lv - 1)])
    for p in range(4):
        a, b = int(offs[p]), int(offs[p + 1])
        if b > a:
            assert lv[a] == 5
        P = hf.pair_matrix(x[a:b], metric)
        K = fr.total_order_key(P)
        lists = []
        for r in range(a, b):
            c = int(g["counts0"][r])
            lists.append((r, 0, g["neighbors0"][r, :c].astype(np.int64), g["dists0"][r, :c]))
            for level in range(1, lv[r]):
                u = up[r] + level - 1
                cu = int(g["counts_up"][u])
                lists.append((r, level, g["neighbors_up"][u, :cu].astype(np.int64), g["dists_up"][u, :cu]))
        for r, level, nb, dist in lists:
            i = r - a
            assert (nb < b - a).all() and len(set(nb.tolist())) == len(nb)
            assert (lv[a + nb] > level).all()                                     # every neighbour has the level
            # a list entry carries the distance of the insertion that made it: the inserting node in the query role,
            # so P[i][v] for i's own list and P[j][i] for a back-link of a later node j
            own, back = P[i, nb].view(np.uint32), P[nb, i].view(np.uint32)
            assert ((dist.view(np.uint32) == own) | (dist.view(np.uint32) == back)).all()
            if i == b - a - 1:   # the last node's lists never took a back-link: ranked, ascending by total order
                assert (np.diff(K[i, nb]) >= 0).all()
    assert g["counts0"][4:].min() > 0                                             # a partition > 1 row is connected


# ---- GPU: the restated cosine rule is the IVF_FLAT scan's ----------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["f32", "f16", "bf16"])
@pytest.mark.parametrize("d", [8, 20, 36, 128])
def test_cosine_rule_is_the_ivf_flat_scan(dt, d):
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


# ---- GPU: build ---------------------------------------------------------------------------------------------------
BUILD_CASES = [  # metric, dtype, d, m, efc
    ("l2", "f32", 8, 20, 150), ("cosine", "f32", 36, 4, 8), ("dot", "f32", 128, 20, 150),
    ("l2", "f16", 36, 4, 8), ("cosine", "f16", 128, 20, 150), ("dot", "f16", 8, 4, 8),
    ("l2", "bf16", 128, 4, 8), ("cosine", "bf16", 8, 20, 150), ("dot", "bf16", 36, 20, 150),
    ("l2", "u8", 36, 20, 150), ("cosine", "u8", 8, 4, 8), ("dot", "u8", 128, 4, 8),
    ("cosine", "f32", 768, 20, 150), ("l2", "f16", 768, 4, 8)]


def _args(K=6, seed=5):
    return dict(num_partitions=K, max_iters=10, seed=seed)


@pytest.mark.gpu
@pytest.mark.parametrize("metric,dt,d,m,efc", BUILD_CASES)
def test_build_bit_identical(metric, dt, d, m, efc):
    x, kw = _typed(_data(700, d, seed=d + m, dup=40), dt)
    hp = lb.HnswBuildParams(max_level=5, m=m, ef_construction=efc)
    ix = lb.IvfHnswFlatIndex.build(x, metric, hnsw_params=hp, **_args(), **kw)
    flat = lb.IvfFlatIndex.build(x, metric, **_args(), **kw).export()
    got = ix.export()
    for key in ("centroids", "part_offsets", "vectors", "row_ids"):
        assert np.array_equal(got[key].view(np.uint8), flat[key].view(np.uint8)), key
    want = hf.build(got["vectors"], got["part_offsets"], metric, dt, m=m, max_level=5, efc=efc, seed=5)
    _assert_graph_equal(got["graph"], want)


def _part_ids(offs):
    return np.repeat(np.arange(len(offs) - 1, dtype=np.uint32), np.diff(np.asarray(offs, np.int64)))


@pytest.mark.gpu
def test_build_partitions_of_0_1_2_and_m_plus_1_rows():
    """a device build whose partitions hold 1, 2 and m + 1 rows (far groups with their own centroids), searched over
    every partition; and a restated graph over partitions of 0, 1, 2 and m + 1 rows loaded through from_parts and
    searched.  (The IVF stage's k-means splits a cluster into an empty one, so a device build keeps no empty
    partition.)"""
    m = 4
    x = _data(200, 16, seed=9, dup=30)
    far = np.random.default_rng(1).standard_normal((8, 16)).astype(np.float32)
    x[0] = 900 + far[0]                                  # 1 row
    x[1:3] = 500 + far[1:3]                              # 2 rows
    x[3:3 + m + 1] = -300 + far[3:3 + m + 1]             # m + 1 rows
    cent = np.stack([x[10:100].mean(axis=0), x[100:].mean(axis=0), x[0], x[1:3].mean(axis=0),
                     x[3:3 + m + 1].mean(axis=0)])
    ix = lb.IvfHnswFlatIndex.build(x, "l2", num_partitions=5, max_iters=1, centroids=cent,
                                   hnsw_params=lb.HnswBuildParams(max_level=3, m=m, ef_construction=8))
    got = ix.export()
    sizes = sorted(np.diff(got["part_offsets"].astype(np.int64)).tolist())
    assert sizes[:3] == [1, 2, m + 1], sizes
    _assert_graph_equal(got["graph"], hf.build(got["vectors"], got["part_offsets"], "l2", m=m, max_level=3, efc=8))
    q = np.concatenate([x[0:1] + 1, x[1:2] - 1, x[4:5], np.full((1, 16), -800.0, np.float32), x[50:53]])
    ids, d = ix.search(q, k=5, nprobes=5)
    wi, wd, _ = hf.search(got["centroids"], got["part_offsets"], got["vectors"], got["row_ids"], got["graph"], q, 5, 5)
    assert np.array_equal(ids, wi) and np.array_equal(d.view(np.uint32), wd.view(np.uint32))
    part = np.random.default_rng(4).integers(4, 6, 160).astype(np.uint32)
    part[:1], part[1:3], part[3:3 + m + 1] = 1, 2, 3     # partition 0 empty
    y = _data(160, 16, seed=3)
    base = lb.IvfFlatIndex.from_parts(_data(6, 16, seed=2), part, y, np.arange(160, dtype=np.uint64)).export()
    assert np.diff(base["part_offsets"].astype(np.int64))[:4].tolist() == [0, 1, 2, m + 1]
    g = hf.build(base["vectors"], base["part_offsets"], "l2", m=m, max_level=3, efc=8)
    ix2 = lb.IvfHnswFlatIndex.from_parts(_data(6, 16, seed=2), part, y, np.arange(160, dtype=np.uint64), graph=g)
    _assert_graph_equal(ix2.export()["graph"], g)
    ids, d = ix2.search(y[:5], k=5, nprobes=6)
    wi, wd, _ = hf.search(base["centroids"], base["part_offsets"], base["vectors"], base["row_ids"], g, y[:5], 5, 6)
    assert np.array_equal(ids, wi) and np.array_equal(d.view(np.uint32), wd.view(np.uint32))


# ---- GPU: search --------------------------------------------------------------------------------------------------
def _index(metric="l2", n=1500, d=16, K=4, m=8, efc=40, seed=0):
    x = _data(n, d, seed=seed, dup=50)
    ix = lb.IvfHnswFlatIndex.build(x, metric, num_partitions=K, max_iters=10, seed=seed,
                                   hnsw_params=lb.HnswBuildParams(max_level=4, m=m, ef_construction=efc))
    return x, ix, ix.export()


def _ref_search(parts, metric, q, k, nprobes, dt="f32", **kw):
    return hf.search(parts["centroids"], parts["part_offsets"], parts["vectors"], parts["row_ids"], parts["graph"], q,
                     k, nprobes, metric=metric, dt=dt, **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("metric", ["l2", "cosine", "dot"])
@pytest.mark.parametrize("k,ef", [(1, None), (10, None), (10, 50), (100, None), (100, 150), (1024, None),
                                  (1024, 1100), (7, 7)])
def test_search_bit_identical(metric, k, ef):
    x, ix, parts = _index(metric, n=2600 if k == 1024 else 1500)
    q = _data(12, 16, seed=77)
    ids, d = ix.search(q, k=k, nprobes=2, ef=ef)
    wi, wd, wc = _ref_search(parts, metric, q, k, 2, ef=ef)
    assert np.array_equal(d.view(np.uint32), wd.view(np.uint32))
    assert np.array_equal(ids, wi)


@pytest.mark.gpu
@pytest.mark.parametrize("metric", ["l2", "cosine", "dot"])
@pytest.mark.parametrize("dt", ["f16", "bf16", "u8"])
def test_search_typed_columns_bit_identical(metric, dt):
    x, kw = _typed(_data(1200, 36, seed=4, dup=30), dt)
    ix = lb.IvfHnswFlatIndex.build(x, metric, num_partitions=3, max_iters=10,
                                   hnsw_params=lb.HnswBuildParams(max_level=4, m=6, ef_construction=30), **kw)
    parts = ix.export()
    q, _ = _typed(_data(8, 36, seed=5), dt)
    for k, ef in ((10, None), (20, 60)):
        ids, d = ix.search(q, k=k, nprobes=2, ef=ef)
        wi, wd, _ = _ref_search(parts, metric, _f32(q, dt), k, 2, dt=dt, ef=ef)
        assert np.array_equal(d.view(np.uint32), wd.view(np.uint32)), k
        assert np.array_equal(ids, wi), k


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
@pytest.mark.parametrize("metric", ["l2", "cosine"])
@pytest.mark.parametrize("side", [-1, 0, 1])
def test_prefilter_either_side_of_the_switch(metric, side):
    x = _data(1500, 16, seed=0)                          # no duplicated rows: no ties between the two kinds' orders
    ix = lb.IvfHnswFlatIndex.build(x, metric, num_partitions=1, max_iters=10,
                                   hnsw_params=lb.HnswBuildParams(max_level=4, m=8, ef_construction=40))
    parts = ix.export()
    n = x.shape[0]
    want = n * 10 // 100 + side        # side -1: flat branch; 0, 1: the graph
    rng = np.random.default_rng(3)
    bits = np.zeros(n, bool)
    bits[np.sort(rng.choice(n, want, replace=False))] = True
    q = _data(8, 16, seed=5)
    ids, d = ix.search_ex(q, k=10, nprobes=1, allow_bitmap=_bitmap(bits))
    wi, wd, _ = _ref_search(parts, metric, q, 10, 1, allow_bits=bits)
    assert np.array_equal(d.view(np.uint32), wd.view(np.uint32))
    assert np.array_equal(ids, wi)
    if side == -1:
        # the flat branch scores every allowed row with the IVF_FLAT scan's rule: IVF_FLAT's prefiltered search
        # returns the same rows and distances
        flat = lb.IvfFlatIndex.from_parts(parts["centroids"], np.zeros(n, np.uint32), parts["vectors"],
                                          parts["row_ids"], metric)
        fi, fd = flat.search_ex(q, k=10, nprobes=1, allow_bitmap=_bitmap(bits))
        assert np.array_equal(fd.view(np.uint32), d.view(np.uint32)) and np.array_equal(fi, ids)


@pytest.mark.gpu
@pytest.mark.parametrize("flat", [False, True])
def test_range_bounds_on_rows(flat):
    x, ix, parts = _index("cosine", K=1)
    n = x.shape[0]
    q = _data(4, 16, seed=6)
    _, d0 = ix.search(q, k=30, nprobes=1)
    lower, upper = float(d0[0, 3]), float(d0[0, 20])     # rows exactly on both bounds
    bits = np.ones(n, bool)
    if flat:                                             # 5 % of the rows allowed: the flat branch
        bits[:] = False
        bits[:n // 20] = True
    ids, d = ix.search_ex(q, k=30, nprobes=1, allow_bitmap=_bitmap(bits), lower_bound=lower, upper_bound=upper)
    wi, wd, _ = _ref_search(parts, "cosine", q, 30, 1, allow_bits=bits, lower=lower, upper=upper)
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
@pytest.mark.parametrize("metric,dt", [("cosine", "f32"), ("dot", "bf16")])
def test_graph_from_reference_with_other_m_searches_identically(metric, dt):
    x, kw = _typed(_data(1500, 16, seed=0, dup=50), dt)
    ix = lb.IvfHnswFlatIndex.build(x, metric, num_partitions=4, max_iters=10,
                                   hnsw_params=lb.HnswBuildParams(max_level=4, m=8, ef_construction=40), **kw)
    parts = ix.export()
    g = hf.build(parts["vectors"], parts["part_offsets"], metric, dt, m=5, max_level=3, efc=20, seed=11)
    opts = dict(distance_type=metric, bf16=dt == "bf16")
    ix2 = lb.IvfHnswFlatIndex.from_parts(parts["centroids"], _part_ids(parts["part_offsets"]), parts["vectors"],
                                         parts["row_ids"], graph=g, **opts)
    parts2 = dict(parts, graph=g)
    q, _ = _typed(_data(10, 16, seed=12), dt)
    for k, ef in ((10, None), (10, 40), (50, None)):
        ids, d = ix2.search(q, k=k, nprobes=3, ef=ef)
        wi, wd, _ = _ref_search(parts2, metric, _f32(q, dt), k, 3, dt=dt, ef=ef)
        assert np.array_equal(d.view(np.uint32), wd.view(np.uint32))
        assert np.array_equal(ids, wi)
    e = ix2.export()
    ix3 = lb.IvfHnswFlatIndex.from_parts(parts["centroids"], _part_ids(e["part_offsets"]), e["vectors"], e["row_ids"],
                                         graph=e["graph"], **opts)
    _assert_graph_equal(ix3.export()["graph"], g)
    assert np.array_equal(ix3.search(q, k=10, nprobes=3)[0], ix2.search(q, k=10, nprobes=3)[0])
    # a device build and a load of its own export search alike
    ix4 = lb.IvfHnswFlatIndex.from_parts(parts["centroids"], _part_ids(parts["part_offsets"]), parts["vectors"],
                                         parts["row_ids"], graph=parts["graph"], **opts)
    for a, b in zip(ix4.search(q, k=10, nprobes=3, ef=30), ix.search(q, k=10, nprobes=3, ef=30)):
        assert np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8))


@pytest.mark.gpu
def test_graph_index_refusals():
    x, ix, parts = _index()
    L, C = lb._lib.lib(), lb._lib.C
    with pytest.raises(lb.LanceB200Error) as e:
        lb._lib.check(L.lb2_index_load_flat(ix._h, None, None, None, C.c_uint64(0)))
    assert e.value.status == lb._lib.INVALID_ARG and "IVF_HNSW_FLAT" in str(e.value)
    with pytest.raises(lb.LanceB200Error) as e:
        ix.update(add_part_ids=np.zeros(1, np.uint32), add_codes=np.zeros((1, 64), np.uint8),
                  add_row_ids=np.array([9999], np.uint64))
    assert e.value.status == lb._lib.UNSUPPORTED and "IVF_HNSW_FLAT" in str(e.value)
    with pytest.raises(lb.LanceB200Error) as e:
        ix.repartition()
    assert e.value.status == lb._lib.UNSUPPORTED and "IVF_HNSW_FLAT" in str(e.value)
    with pytest.raises(lb.LanceB200Error):      # an IVF_HNSW_FLAT graph is not an IVF_HNSW_SQ or _PQ one
        lb._lib.check(L.lb2_index_hnsw_sq_info(ix._h, None, None, None, None))
    with pytest.raises(lb.LanceB200Error):
        lb._lib.check(L.lb2_index_export_hnsw_pq(ix._h, None, None, None, None, None, None, None))
    g = parts["graph"]
    ptr = {k: lb._lib.as_ptr(np.ascontiguousarray(g[k]))[0] for k in
           ("levels", "counts0", "neighbors0", "dists0", "counts_up", "neighbors_up", "dists_up")}
    sq = lb.IvfSqIndex.build(x, "l2", num_partitions=4, max_iters=10)
    with pytest.raises(lb.LanceB200Error) as e:      # a flat graph on an IVF_SQ index
        lb._lib.check(L.lb2_index_load_hnsw_flat(sq._h, C.c_uint32(g["max_level"]), C.c_uint32(g["m"]), C.c_uint32(0),
                                                 ptr["levels"], ptr["counts0"], ptr["neighbors0"], ptr["dists0"],
                                                 ptr["counts_up"], ptr["neighbors_up"], ptr["dists_up"]))
    assert e.value.status == lb._lib.INVALID_ARG and "not an IVF_FLAT index" in str(e.value)
    bad = dict(g)
    bad["neighbors0"] = bad["neighbors0"].copy()
    bad["neighbors0"][5, 0] = 10 ** 6                  # a neighbour outside its partition
    with pytest.raises(lb.LanceB200Error) as e:
        lb.IvfHnswFlatIndex.from_parts(parts["centroids"], _part_ids(parts["part_offsets"]), parts["vectors"],
                                       parts["row_ids"], graph=bad)
    assert e.value.status == lb._lib.INVALID_ARG and "IVF_HNSW_FLAT" in str(e.value)
    with pytest.raises(ValueError):
        lb.IvfHnswFlatIndex.from_parts(parts["centroids"], _part_ids(parts["part_offsets"]), parts["vectors"])


@pytest.mark.gpu
@pytest.mark.parametrize("metric,floor", [("l2", 0.9), ("cosine", 0.9), ("dot", 0.85)])
def test_recall_floor(metric, floor):
    """test_create_ivf_hnsw_flat (rust/lance/src/index/vector/ivf/v2.rs:1450-1467 via test_recall): 512 x 32 uniform
    [0, 1) rows, nlist 4, the default HNSW parameters, the query row 0, k = 100, nprobes = nlist, against the exact
    ground truth"""
    rng = np.random.default_rng(0)
    x = rng.random((512, 32)).astype(np.float32)
    ix = lb.IvfHnswFlatIndex.build(x, metric, num_partitions=4)
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
