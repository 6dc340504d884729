"""The batched HNSW build (insert_batch B) of IVF_HNSW_SQ, IVF_HNSW_PQ and IVF_HNSW_FLAT against its restatement
(tests/hnsw_batch_reference.py): on the CPU the restatement's rounds, its B = 1 identity with the serial restatements
and its invariants; on the device the graphs byte for byte (levels, counts, neighbours, distances, zeroed slots), the
searches over them, optimize's rebuilt partitions, the refusals and the recall against the serial build."""
import numpy as np
import pytest

import hnsw_batch_reference as hb
import hnsw_flat_reference as hf
import hnsw_pq_reference as hp
import hnsw_reference as hr
import lance_b200 as lb


def _data(n, d, seed, dup=0):
    rng = np.random.default_rng(seed)
    x = (rng.standard_normal((n, d)) + 3 * rng.standard_normal((8, d))[rng.integers(0, 8, n)]).astype(np.float32)
    if dup:
        x[-dup:] = x[:dup]     # duplicated rows: their distances tie
    return x


def _typed(x, dt):
    if dt == "f16":
        return x.astype(np.float16), {}
    if dt == "bf16":
        b = np.ascontiguousarray(x, np.float32).view(np.uint32).astype(np.uint64)
        return ((b + 0x7FFF + ((b >> 16) & 1)) >> 16).astype(np.uint16), {"bf16": True}
    return x, {}


def _assert_graph_bytes(got, want):
    """every array of the layout byte for byte, unused slots included"""
    assert got["max_level"] == want["max_level"] and got["m"] == want["m"]
    for key in ("levels", "counts0", "neighbors0", "dists0", "counts_up", "neighbors_up", "dists_up"):
        a, b = np.asarray(got[key]), np.asarray(want[key])
        assert a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8)), key


# ---- CPU: the restatement -----------------------------------------------------------------------------------------
def test_round_boundaries():
    assert hb.rounds(2, 64) == [(1, 2)]
    assert hb.rounds(1, 8) == [] and hb.rounds(0, 8) == []
    assert hb.rounds(40, 8) == [(1, 2), (2, 4), (4, 8), (8, 16), (16, 24), (24, 32), (32, 40)]
    assert hb.rounds(11, 3) == [(1, 2), (2, 4), (4, 7), (7, 10), (10, 11)]
    assert hb.rounds(6, 1) == [(i, i + 1) for i in range(1, 6)]
    for n, b in [(1000, 64), (999, 100), (5, 65536)]:
        r = hb.rounds(n, b)
        assert r[0][0] == 1 and r[-1][1] == n and all(r[t][1] == r[t + 1][0] for t in range(len(r) - 1))
        assert all(e - s == min(b, s) for s, e in r[:-1])


@pytest.mark.parametrize("seed,sizes", [(0, [0, 1, 2, 37]), (3, [5, 120]), (7, [64, 65, 200])])
def test_batch_1_is_the_serial_restatement_sq(seed, sizes):
    rng = np.random.default_rng(seed)
    offs = np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint64)
    codes = rng.integers(0, 256, (int(offs[-1]), 8), dtype=np.uint8)
    codes[-10:] = codes[:10]
    for metric in ("l2", "dot"):
        want = hr.build(codes, offs, (-1.0, 2.0), metric, m=4, max_level=4, efc=10, seed=seed)
        _assert_graph_bytes(hb.build_sq(codes, offs, (-1.0, 2.0), metric, m=4, max_level=4, efc=10, seed=seed,
                                        batch=1), want)


@pytest.mark.parametrize("seed,nbits,metric", [(1, 8, "l2"), (2, 4, "dot"), (5, 8, "cosine")])
def test_batch_1_is_the_serial_restatement_pq(seed, nbits, metric):
    rng = np.random.default_rng(seed)
    M, ds = 4, 2
    cb = rng.standard_normal((M, 1 << nbits, ds)).astype(np.float32)
    offs = np.array([0, 1, 3, 90], np.uint64)
    codes = rng.integers(0, 1 << nbits, (90, M), dtype=np.uint8)
    if nbits == 4:
        codes = (codes[:, 0::2] | (codes[:, 1::2] << 4)).astype(np.uint8)
    want = hp.build(codes, offs, cb, nbits, metric, m=4, max_level=3, efc=12, seed=seed)
    _assert_graph_bytes(hb.build_pq(codes, offs, cb, nbits, metric, m=4, max_level=3, efc=12, seed=seed, batch=1),
                        want)


@pytest.mark.parametrize("seed,metric", [(1, "l2"), (2, "cosine"), (4, "dot")])
def test_batch_1_is_the_serial_restatement_flat(seed, metric):
    x = _data(110, 8, seed, dup=8)
    offs = np.array([0, 2, 30, 110], np.uint64)
    want = hf.build(x, offs, metric, m=4, max_level=3, efc=12, seed=seed)
    _assert_graph_bytes(hb.build_flat(x, offs, metric, m=4, max_level=3, efc=12, seed=seed, batch=1), want)


@pytest.mark.parametrize("batch", [2, 3, 16, 1000])
def test_batched_restatement_invariants(batch):
    rng = np.random.default_rng(batch)
    m = 4
    codes = rng.integers(0, 256, (300, 16), dtype=np.uint8)
    codes[-20:] = codes[:20]
    offs = np.array([0, 0, 1, 4, 300], np.uint64)
    g = hb.build_sq(codes, offs, (-1.0, 2.0), "l2", m=m, max_level=4, efc=12, seed=3, batch=batch)
    lv = g["levels"].astype(np.int64)
    assert (g["counts0"] <= 2 * m).all() and (g["counts_up"] <= m).all()
    up = np.concatenate([[0], np.cumsum(lv - 1)])
    for p in range(4):
        a, b = int(offs[p]), int(offs[p + 1])
        for r in range(a, b):
            ids = g["neighbors0"][r, :g["counts0"][r]]
            assert (ids < b - a).all() and len(set(ids.tolist())) == ids.size and r - a not in ids.tolist()
            assert not g["neighbors0"][r, g["counts0"][r]:].any() and not g["dists0"][r, g["counts0"][r]:].any()
            for level in range(1, lv[r]):
                u = up[r] + level - 1
                ids = g["neighbors_up"][u, :g["counts_up"][u]]
                assert len(set(ids.tolist())) == ids.size and all(lv[a + i] > level for i in ids)
    assert g["counts0"][4:].min() > 0
    serial = hr.build(codes, offs, (-1.0, 2.0), "l2", m=m, max_level=4, efc=12, seed=3)
    assert np.array_equal(g["levels"], serial["levels"])          # levels do not depend on B


# ---- GPU: build byte for byte ---------------------------------------------------------------------------------------
BATCHES = [1, 2, 3, 64]
HP = dict(max_level=4, m=6, ef_construction=16)


def _hp(batch):
    return lb.HnswBuildParams(insert_batch=batch, **HP)


def _ref_kw(batch, seed=5):
    return dict(m=HP["m"], max_level=HP["max_level"], efc=HP["ef_construction"], seed=seed, batch=batch)


def _pq_params(M, nbits, K=4, seed=5):
    return lb.IvfBuildParams(num_partitions=K, num_sub_vectors=M, num_bits=nbits, max_iters=10, pq_max_iters=10,
                             seed=seed)


def _build(kind, x, metric, batch, kw=None, K=4, nbits=8, seed=5):
    kw = kw or {}
    if kind == "sq":
        return lb.IvfHnswSqIndex.build(x, metric, num_partitions=K, max_iters=10, seed=seed, hnsw_params=_hp(batch),
                                       **kw)
    if kind == "pq":
        return lb.IvfHnswPqIndex.build(x, metric, _pq_params(4, nbits, K, seed), _hp(batch), **kw)
    return lb.IvfHnswFlatIndex.build(x, metric, num_partitions=K, max_iters=10, seed=seed, hnsw_params=_hp(batch),
                                     **kw)


def _ref(kind, e, metric, batch, nbits=8, dt="f32", seed=5):
    if kind == "sq":
        return hb.build_sq(e["codes"], e["part_offsets"], e["bounds"], "dot" if metric == "dot" else "l2",
                           **_ref_kw(batch, seed))
    if kind == "pq":
        return hb.build_pq(e["codes"], e["part_offsets"], e["codebook"], nbits, metric, dt, **_ref_kw(batch, seed))
    return hb.build_flat(e["vectors"], e["part_offsets"], metric, dt, **_ref_kw(batch, seed))


@pytest.mark.gpu
@pytest.mark.parametrize("batch", BATCHES)
@pytest.mark.parametrize("metric", ["l2", "cosine", "dot"])
def test_sq_build_equals_restatement(metric, batch):
    x = _data(500, 16, seed=11, dup=30)
    e = _build("sq", x, metric, batch).export()
    _assert_graph_bytes(e["graph"], _ref("sq", e, metric, batch))


@pytest.mark.gpu
@pytest.mark.parametrize("batch", BATCHES)
@pytest.mark.parametrize("metric,nbits,dt", [("l2", 8, "f32"), ("cosine", 8, "f32"), ("dot", 8, "f32"),
                                             ("l2", 4, "f32"), ("cosine", 4, "f32"), ("dot", 4, "f32"),
                                             ("dot", 8, "f16"), ("dot", 4, "bf16")])
def test_pq_build_equals_restatement(metric, nbits, dt, batch):
    x, kw = _typed(_data(400, 16, seed=12 + nbits, dup=30), dt)
    e = _build("pq", x, metric, batch, kw, nbits=nbits).export()
    _assert_graph_bytes(e["graph"], _ref("pq", e, metric, batch, nbits, dt))


@pytest.mark.gpu
@pytest.mark.parametrize("batch", BATCHES)
@pytest.mark.parametrize("metric", ["l2", "cosine", "dot"])
@pytest.mark.parametrize("dt", ["f32", "f16", "bf16"])
def test_flat_build_equals_restatement(dt, metric, batch):
    x, kw = _typed(_data(400, 16, seed=13, dup=30), dt)
    e = _build("flat", x, metric, batch, kw).export()
    _assert_graph_bytes(e["graph"], _ref("flat", e, metric, batch, dt=dt))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["sq", "pq", "flat"])
def test_batch_1_equals_the_default_build(kind, monkeypatch):
    """insert_batch 1 and 0 are the serial build, and the round driver at B = 1 (LB2_HNSW_ROUNDS=1) gives the same
    bytes as the serial kernel"""
    x = _data(900, 16, seed=14, dup=30)
    metric = "cosine" if kind == "flat" else "l2"
    if kind == "sq":
        default = lb.IvfHnswSqIndex.build(x, metric, num_partitions=4, max_iters=10, seed=5,
                                          hnsw_params=lb.HnswBuildParams(**HP))
    elif kind == "pq":
        default = lb.IvfHnswPqIndex.build(x, metric, _pq_params(4, 8), lb.HnswBuildParams(**HP))
    else:
        default = lb.IvfHnswFlatIndex.build(x, metric, num_partitions=4, max_iters=10, seed=5,
                                            hnsw_params=lb.HnswBuildParams(**HP))
    want = default.export()["graph"]
    for batch in (1, 0):
        _assert_graph_bytes(_build(kind, x, metric, batch).export()["graph"], want)
    monkeypatch.setenv("LB2_HNSW_ROUNDS", "1")
    _assert_graph_bytes(_build(kind, x, metric, 1).export()["graph"], want)


# ---- GPU: shapes -----------------------------------------------------------------------------------------------------
def _sq_from_parts(x, part, K, seed=5):
    """an IVF_HNSW_SQ index over chosen partitions: the restated serial graph loaded through from_parts"""
    bounds = (float(x.min()), float(x.max()))
    from sq_reference import sq_encode
    codes = sq_encode(x, *bounds)
    cent = np.zeros((K, x.shape[1]), np.float32)
    base = lb.IvfSqIndex.from_parts(cent, bounds, part, codes, np.arange(x.shape[0], dtype=np.uint64)).export()
    g = hr.build(base["codes"], base["part_offsets"], bounds, "l2", m=HP["m"], max_level=HP["max_level"],
                 efc=HP["ef_construction"], seed=seed)
    return lb.IvfHnswSqIndex.from_parts(cent, bounds, part, codes, np.arange(x.shape[0], dtype=np.uint64), graph=g)


@pytest.mark.gpu
def test_shapes_0_1_2_rows_smaller_than_b_and_on_a_round_boundary():
    """B = 3: rounds [1, 2), [2, 4), [4, 7), [7, 10), ..  Partitions of 0, 1, 2 rows, 3 rows (< B), 7 and 10 rows (a
    round boundary) and 11 rows (one past it), rebuilt through an optimize that removes one row of each"""
    sizes = [0, 1, 2, 3, 7, 10, 11, 40]
    K = len(sizes)
    part = np.repeat(np.arange(K, dtype=np.uint32), [s + 1 if s else 0 for s in sizes])
    x = _data(part.size, 16, seed=15, dup=10)
    ix = _sq_from_parts(x, part, K)
    old = ix.export()
    offs = old["part_offsets"].astype(np.int64)
    gone = old["row_ids"][offs[1:][np.diff(offs) > 0] - 1]          # the last row of every non-empty partition
    new = ix.optimize(remove_row_ids=gone, seed=5, insert_batch=3).export()
    assert np.diff(new["part_offsets"].astype(np.int64)).tolist() == sizes
    _assert_graph_bytes(new["graph"], _ref("sq", new, "l2", 3))


@pytest.mark.gpu
def test_one_round_with_more_items_than_resident_warps():
    """64 partitions x B = 128: the round at s = 128 holds 8192 (partition, node) items, more than 132 SMs x 32
    one-warp CTAs"""
    K, per = 64, 260
    part = np.repeat(np.arange(K, dtype=np.uint32), per)
    x = _data(part.size, 8, seed=16)
    x += np.repeat(np.random.default_rng(1).standard_normal((K, 8)).astype(np.float32) * 50, per, axis=0)
    ix = _sq_from_parts(x, part, K)
    old = ix.export()
    new = ix.optimize(remove_row_ids=old["row_ids"][old["part_offsets"][1:].astype(np.int64) - 1], seed=5,
                      insert_batch=128).export()
    _assert_graph_bytes(new["graph"], _ref("sq", new, "l2", 128))


# ---- GPU: searches over a batched graph ------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["sq", "pq", "flat"])
def test_search_of_a_batched_index_equals_the_restatement(kind):
    metric = "l2" if kind != "flat" else "cosine"
    x = _data(600, 16, seed=17, dup=20)
    ix = _build(kind, x, metric, 16)
    e = ix.export()
    _assert_graph_bytes(e["graph"], _ref(kind, e, metric, 16))
    q = _data(10, 16, seed=18)
    ids, d = ix.search(q, k=10, nprobes=2, ef=30)
    if kind == "sq":
        wi, wd, _ = hr.search(e["centroids"], e["bounds"], e["part_offsets"], e["codes"], e["row_ids"], e["graph"], q,
                              10, 2, metric=metric, ef=30)
    elif kind == "pq":
        wi, wd, _ = hp.search(e["centroids"], e["codebook"], 8, e["part_offsets"], e["codes"], e["row_ids"],
                              e["graph"], q, 10, 2, metric=metric, ef=30)
    else:
        wi, wd, _ = hf.search(e["centroids"], e["part_offsets"], e["vectors"], e["row_ids"], e["graph"], q, 10, 2,
                              metric=metric, ef=30)
    assert np.array_equal(d.view(np.uint32), wd.view(np.uint32)) and np.array_equal(ids, wi)


# ---- GPU: optimize ---------------------------------------------------------------------------------------------------
def _add_to(ix, x_add, ids):
    t = ix.transform(x_add)
    ok = t["valid"]
    return dict(add_part_ids=t["part_ids"][ok], add_payload=t["payload"][ok], add_row_ids=ids[ok]), t["part_ids"][ok]


@pytest.mark.gpu
def test_optimize_rebuilds_changed_partitions_with_the_index_b():
    x = _data(1100, 16, seed=19)
    ix = _build("sq", x[:900], "l2", 64)
    old = ix.export()
    _assert_graph_bytes(old["graph"], _ref("sq", old, "l2", 64))
    add, parts = _add_to(ix, x[900:], np.arange(900, 1100, dtype=np.uint64))
    keep_p = int(np.setdiff1d(np.arange(4), parts)[0]) if np.setdiff1d(np.arange(4), parts).size else None
    new = ix.optimize(seed=5, **add).export()       # insert_batch None: the index's B = 64, the build's seed
    _assert_graph_bytes(new["graph"], _ref("sq", new, "l2", 64))
    over = ix.optimize(seed=5, insert_batch=2, **add).export()
    _assert_graph_bytes(over["graph"], _ref("sq", over, "l2", 2))
    assert not np.array_equal(over["graph"]["neighbors0"], new["graph"]["neighbors0"])
    if keep_p is not None:                           # a partition that received nothing keeps its graph verbatim
        a, b = (int(v) for v in old["part_offsets"][keep_p:keep_p + 2])
        c, d = (int(v) for v in new["part_offsets"][keep_p:keep_p + 2])
        assert np.array_equal(new["graph"]["neighbors0"][c:d], old["graph"]["neighbors0"][a:b])


@pytest.mark.gpu
def test_optimize_of_a_loaded_graph_is_serial_by_default():
    part = np.repeat(np.arange(3, dtype=np.uint32), [60, 80, 100])
    x = _data(part.size, 16, seed=20)
    ix = _sq_from_parts(x, part, 3)
    old = ix.export()
    gone = old["row_ids"][old["part_offsets"][1:].astype(np.int64) - 1]
    new = ix.optimize(remove_row_ids=gone, seed=5).export()
    _assert_graph_bytes(new["graph"], _ref("sq", new, "l2", 1))
    b8 = ix.optimize(remove_row_ids=gone, seed=5, insert_batch=8).export()
    _assert_graph_bytes(b8["graph"], _ref("sq", b8, "l2", 8))


# ---- GPU: refusals ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["sq", "pq", "flat"])
def test_insert_batch_above_65536_is_refused(kind):
    x = _data(400, 16, seed=21)
    with pytest.raises(lb.LanceB200Error) as e:
        _build(kind, x, "l2", 65537)
    assert e.value.status == lb._lib.INVALID_ARG
    ix = _build(kind, x[:300], "l2", 65536)
    add, _ = _add_to(ix, x[300:], np.arange(300, 400, dtype=np.uint64))
    with pytest.raises(lb.LanceB200Error) as e:
        ix.optimize(insert_batch=65537, **add)
    assert e.value.status == lb._lib.INVALID_ARG


# ---- GPU: quality ----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_batched_recall_within_0_02_of_serial():
    """20 000 x 32 f32, K = 4, m 16, ef_construction 100: recall@10 at nprobes 4, ef 50 against brute force"""
    rng = np.random.default_rng(22)
    n, d = 20000, 32
    x = (rng.standard_normal((n, d)) + 2 * rng.standard_normal((64, d))[rng.integers(0, 64, n)]).astype(np.float32)
    q = x[rng.choice(n, 200, replace=False)] + 0.1 * rng.standard_normal((200, d)).astype(np.float32)
    d2 = (q * q).sum(1)[:, None] - 2 * q @ x.T + (x * x).sum(1)[None, :]
    truth = np.argsort(d2, axis=1)[:, :10]
    recall = {}
    for batch in (1, 64):
        ix = lb.IvfHnswFlatIndex.build(x, "l2", num_partitions=4, max_iters=10, seed=1,
                                       hnsw_params=lb.HnswBuildParams(m=16, ef_construction=100, insert_batch=batch))
        ids, _ = ix.search(q, k=10, nprobes=4, ef=50)
        recall[batch] = np.mean([len(set(ids[i].tolist()) & set(truth[i].tolist())) / 10 for i in range(len(q))])
    assert recall[64] >= recall[1] - 0.02, recall
