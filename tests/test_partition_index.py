"""The partition index (an HNSW graph over the IVF centroids, lance-index/src/vector/utils.rs:26-108) against its
restatement (tests/centroid_graph_reference.py).  On the CPU: may_train_index's mode rule, and the restated search
returning, for every row, a node at exactly the 16-lane distance the oracle computes.  On the device: the graph bit for
bit (levels, lists, distances; serial and batched), and every row's (part, dist, valid) bit for bit, across
non-finite and overflowing rows, rows equal to a centroid, tied centroids, normalised cosine columns, u8 columns,
chunked and streamed inputs; the exact modes and 16-bit models equal to compute_partitions; the refusals."""
import numpy as np
import pytest

import centroid_graph_reference as cg
import lance_b200 as lb
from lance_b200 import _lib
from oracle import binding as ob


def _centroids(k, d, seed, dup=True):
    """normal centroids; with dup, a few exact duplicates (exact-distance ties)"""
    rng = np.random.default_rng(seed)
    c = rng.standard_normal((k, d)).astype(np.float32)
    if dup and k >= 8:
        for a, b in ((1, k - 1), (2, k // 2), (3, k // 3 + 1)):
            if a != b:
                c[b] = c[a]
    return c


def _rows(cent, n, seed, special=True):
    """rows near random centroids, plus rows equal to a centroid, non-finite rows and rows whose distances overflow"""
    rng = np.random.default_rng(seed)
    k, d = cent.shape
    x = (cent[rng.integers(0, k, n)] + rng.standard_normal((n, d)).astype(np.float32) * np.float32(0.3))
    x = x.astype(np.float32)
    if special and n >= 16:
        x[0] = cent[0]
        x[1] = cent[k - 1]
        x[2, d // 2] = np.nan
        x[3, 0] = np.inf
        x[4, d - 1] = -np.inf
        x[5] = np.float32(3e30)               # finite; every L2 distance overflows
        x[6] = 0.0
        x[7, :] = cent[min(2, k - 1)] * np.float32(1e18)   # finite; large products
    return x


def _assert_assign_equal(got, want):
    gp, gd, gv = got
    wp, wd, wv = want
    assert np.array_equal(gv, wv), np.flatnonzero(gv != wv)[:10]
    assert np.array_equal(gp, wp), np.flatnonzero(gp != wp)[:10]
    assert np.array_equal(gd[wv].view(np.uint32), wd[wv].view(np.uint32)), np.flatnonzero(gd[wv] != wd[wv])[:10]
    assert np.isnan(gd[~wv]).all() and (gp[~wv] == 0).all()


# ---- CPU: the mode rule and the restatement -------------------------------------------------------------------------
MODE_CASES = [(999, 1000), (1000, 1000), (1, 999_999), (1, 1_000_000), (4096, 768), (65536, 128), (256, 128),
              (244, 4096), (245, 4096), (2, 4)]


@pytest.mark.parametrize("mode", ["exact", "auto", "hnsw"])
@pytest.mark.parametrize("dtype", ["f32", "f16", "bf16", "u8"])
def test_mode_rule_matches_reference(mode, dtype):
    np_dt = {"f32": np.float32, "f16": np.float16, "bf16": np.uint16, "u8": np.uint8}[dtype]
    for k, d in MODE_CASES:
        got = lb.PartitionIndex.uses_graph(k, d, mode, np_dt, bf16=dtype == "bf16")
        assert got == cg.uses_graph(k, d, dtype, mode), (k, d)
    assert lb.PartitionIndex.uses_graph(999, 1000, "auto") is False
    assert lb.PartitionIndex.uses_graph(1000, 1000, "auto") is True


def test_unknown_mode_is_refused():
    with pytest.raises(ValueError):
        lb.PartitionIndex.uses_graph(4, 4, "sometimes")
    import ctypes as C
    out = C.c_int()
    st = _lib.lib().lb2_partition_index_uses_graph(C.c_uint64(4), C.c_uint32(4), C.c_int(0), C.c_int(3), C.byref(out))
    assert st == _lib.INVALID_ARG


@pytest.mark.parametrize("metric", ["l2", "dot"])
def test_restated_search_returns_a_node_at_its_exact_distance(metric):
    cent = _centroids(96, 20, 1)
    rows = _rows(cent, 200, 2)
    g = cg.build(cent, metric, seed=5)
    part, dist, valid = cg.assign(g, cent, rows, metric)
    fin = np.isfinite(rows).all(axis=1)
    assert not valid[~fin].any()
    f = ob.l2 if metric == "l2" else ob.dot
    for i in np.flatnonzero(valid):
        want = np.float32(f(rows[i], cent[part[i]]))
        want = want if metric == "l2" else np.float32(1.0) - want
        assert np.float32(dist[i]).view(np.uint32) == want.view(np.uint32) or (np.isnan(want) and np.isnan(dist[i])), i
    # the graph never beats the exact scan, and on these rows it mostly agrees with it
    exact = cg.distances(rows[valid], cent, metric).min(axis=1)
    assert (dist[valid] >= exact).all()
    assert (dist[valid] == exact).mean() > 0.8


# ---- GPU: the graph -----------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("metric", ["l2", "dot"])
@pytest.mark.parametrize("k", [1, 2, 13, 4096])
@pytest.mark.parametrize("batch", [1, 16])
def test_graph_and_assignment_equal_restatement(metric, k, batch):
    d = 8 if k >= 1024 else 16
    cent = _centroids(k, d, 10 + k)
    pi = lb.PartitionIndex.build(cent, metric, mode="hnsw", seed=77, insert_batch=batch)
    assert pi.has_graph
    got = pi.export()
    want = cg.build(cent, metric, seed=77, batch=batch)
    assert (got["max_level"], got["m"], got["ef_construction"]) == (7, 12, 15)
    from test_ivf_hnsw_sq import _assert_graph_equal
    _assert_graph_equal(got, want)
    rows = _rows(cent, 300 if k >= 1024 else 120, 3 + k)
    _assert_assign_equal(pi.assign(rows), cg.assign(want, cent, rows, metric))


# ---- GPU: the assignment ------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("metric", ["l2", "dot"])
@pytest.mark.parametrize("d", [12, 64, 100])
def test_assignment_equals_restatement(metric, d):
    cent = _centroids(300, d, 20 + d)
    rows = _rows(cent, 1200, 21 + d)
    pi = lb.PartitionIndex.build(cent, metric, mode="hnsw", seed=3)
    got = pi.assign(rows)
    want = cg.assign(pi.export(), cent, rows, metric)
    _assert_assign_equal(got, want)
    assert not want[2][2:5].any()          # non-finite rows are dropped
    if metric == "l2":
        assert not want[2][5]              # every distance overflows: no result
    assert want[2][8:].all()
    if metric == "l2":
        assert got[0][0] == 0 and got[1][0] == 0.0      # a row equal to centroid 0
    # device rows give the same answer
    _assert_assign_equal(pi.assign(lb.DeviceArray.from_numpy(rows)), want)


@pytest.mark.gpu
def test_assignment_of_normalised_cosine_columns():
    cent = ob.normalize_rows(_centroids(200, 32, 30, dup=False))
    rows = ob.normalize_rows(_rows(cent, 600, 31, special=False))
    pi = lb.PartitionIndex.build(cent, "l2", mode="hnsw", seed=9)
    _assert_assign_equal(pi.assign(rows), cg.assign(pi.export(), cent, rows, "l2"))
    with pytest.raises(lb.LanceB200Error) as e:
        lb.PartitionIndex.build(cent, "cosine", mode="hnsw")
    assert e.value.status == _lib.INVALID_ARG


@pytest.mark.gpu
@pytest.mark.parametrize("metric", ["l2", "dot"])
def test_assignment_of_u8_columns(metric):
    rng = np.random.default_rng(40)
    cent = rng.uniform(0, 255, (160, 32)).astype(np.float32)
    rows = rng.integers(0, 256, (500, 32)).astype(np.uint8)
    rows[:3] = np.clip(np.rint(cent[:3]), 0, 255).astype(np.uint8)
    pi = lb.PartitionIndex.build(cent, metric, mode="hnsw", seed=4, dtype=np.uint8)
    assert pi.has_graph
    _assert_assign_equal(pi.assign(rows), cg.assign(pi.export(), cent, rows.astype(np.float32), metric))


def _knobs(monkeypatch, chunk=None, resident_mb=None):
    for name, v in (("LB2_CHUNK_ROWS", chunk), ("LB2_MAX_RESIDENT_MB", resident_mb)):
        if v is None:
            monkeypatch.delenv(name, raising=False)
        else:
            monkeypatch.setenv(name, str(v))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.uint8])
def test_assignment_past_one_chunk_and_streamed(dtype, monkeypatch):
    cent = _centroids(256, 32, 50)
    rows = _rows(cent, 2000, 51)
    if dtype == np.uint8:
        cent = (cent * 20 + 128).astype(np.float32)
        rows = np.clip(np.nan_to_num(rows, posinf=255, neginf=0) * 20 + 128, 0, 255).astype(np.uint8)
    pi = lb.PartitionIndex.build(cent, "l2", mode="hnsw", seed=6, dtype=dtype)
    want = cg.assign(pi.export(), cent, rows.astype(np.float32), "l2")
    _knobs(monkeypatch)
    _assert_assign_equal(pi.assign(rows), want)
    _knobs(monkeypatch, chunk=333)
    _assert_assign_equal(pi.assign(rows), want)
    _knobs(monkeypatch, chunk=333, resident_mb=0)
    _assert_assign_equal(pi.assign(rows), want)
    _knobs(monkeypatch)


# ---- GPU: the exact modes, 16-bit models, AUTO and the refusals ----------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("metric", ["l2", "dot"])
def test_exact_modes_and_16bit_models_are_compute_partitions(metric):
    cent = _centroids(64, 16, 60)
    rows = _rows(cent, 400, 61)
    pi = lb.PartitionIndex.build(cent, metric, mode="exact")
    assert not pi.has_graph and pi.export() is None
    _assert_assign_equal(pi.assign(rows), lb.compute_partitions(cent, rows, metric))
    c16, r16 = cent.astype(np.float16), np.nan_to_num(rows, posinf=1e4, neginf=-1e4).astype(np.float16)
    for mode in ("exact", "auto", "hnsw"):
        pi = lb.PartitionIndex.build(c16, metric, mode=mode, dtype=np.float16)
        assert not pi.has_graph
        _assert_assign_equal(pi.assign(r16), lb.compute_partitions(c16, r16, metric))


@pytest.mark.gpu
def test_auto_mode_switches_at_one_million_values():
    rng = np.random.default_rng(70)
    rows = rng.standard_normal((300, 1000)).astype(np.float32)
    below = rng.standard_normal((999, 1000)).astype(np.float32)
    at = np.concatenate([below, rng.standard_normal((1, 1000)).astype(np.float32)])
    pi = lb.PartitionIndex.build(below, "l2", mode="auto", seed=1)
    assert not pi.has_graph
    _assert_assign_equal(pi.assign(rows), lb.compute_partitions(below, rows, "l2"))
    pi = lb.PartitionIndex.build(at, "l2", mode="auto", seed=1)
    assert pi.has_graph
    hn = lb.PartitionIndex.build(at, "l2", mode="hnsw", seed=1)
    _assert_assign_equal(pi.assign(rows), hn.assign(rows))
    _assert_assign_equal(pi.assign(rows), cg.assign(pi.export(), at, rows, "l2"))


@pytest.mark.gpu
def test_refusals():
    cent = _centroids(32, 10, 80)
    with pytest.raises(lb.LanceB200Error) as e:
        lb.PartitionIndex.build(cent, "l2", mode="hnsw")
    assert e.value.status == _lib.UNSUPPORTED           # d % 4 != 0
    assert not lb.PartitionIndex.build(cent, "l2", mode="exact").has_graph
    cent = _centroids(32, 16, 81)
    pi = lb.PartitionIndex.build(cent, "l2", mode="hnsw")
    other = lb.PartitionIndex(pi._h, cent[:16], pi._dt, "l2")
    with pytest.raises(lb.LanceB200Error) as e:
        other.assign(_rows(cent, 20, 82))
    assert e.value.status == _lib.INVALID_ARG
    other._h = None
    other = lb.PartitionIndex(pi._h, cent, pi._dt, "dot")
    with pytest.raises(lb.LanceB200Error) as e:
        other.assign(_rows(cent, 20, 82))
    assert e.value.status == _lib.INVALID_ARG
    other._h = None
