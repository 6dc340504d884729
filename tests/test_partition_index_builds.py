"""The partition index inside the index builds and the index handle (lb2_kmeans_params.partition_index,
lb2_index_set_partition_index): every build's partition ids equal PartitionIndex.assign over the exported centroids
with the documented level seed, and its payload equals lb2_index_transform's for those partitions (PQ residual codes,
RQ codes and factors from the graph's dist_v_c); AUTO switches at K · d = 10^6; the rule follows transform, optimize
and from_storage + set_partition_index; lb2_kmeans_train refuses it; and the assignment kernel over many rows per
warp (its persistent loop and the whole-bitset clear) against the restatement."""
import ctypes as C

import numpy as np
import pytest

import centroid_graph_reference as cg
import lance_b200 as lb
from lance_b200 import _lib

PI_SEED_XOR = 0x7061727469646978


def _graph_seed(seed):
    return seed ^ PI_SEED_XOR


def _data(n, d, seed, comps=24):
    rng = np.random.default_rng(seed)
    means = rng.standard_normal((comps, d)).astype(np.float32) * np.float32(3.0)
    x = means[rng.integers(0, comps, n)] + rng.standard_normal((n, d)).astype(np.float32)
    x = x.astype(np.float32)
    x[5, 1] = np.nan   # dropped by every build
    return x


def _parts_by_row(ex, n):
    """the partition of every row id (row ids 0 .. n - 1), n for rows the index does not hold"""
    off = np.asarray(ex["part_offsets"], np.int64)
    out = np.full(n, 2 ** 32 - 1, np.uint64)
    rid = np.asarray(ex["row_ids"], np.int64)
    out[rid] = np.repeat(np.arange(len(off) - 1), np.diff(off))
    return out


def _check_parts(ex, data, metric, seed, dtype=np.float32):
    cent = ex["centroids"]
    rows = data
    if metric == "cosine":
        rows = lb.normalize_fsl(data)
        metric = "l2"
    pi = lb.PartitionIndex.build(cent, metric, mode="hnsw", seed=_graph_seed(seed), dtype=dtype)
    part, _, valid = pi.assign(rows)
    got = _parts_by_row(ex, data.shape[0])
    assert np.array_equal(got[valid], part[valid].astype(np.uint64))
    assert (got[~valid] == 2 ** 32 - 1).all()
    return part, valid


def _row_payload(ex, key, n):
    rid = np.asarray(ex["row_ids"], np.int64)
    arr = np.asarray(ex[key])
    out = np.zeros((n,) + arr.shape[1:], arr.dtype)
    out[rid] = arr
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("metric", ["l2", "dot", "cosine"])
def test_ivf_flat_build_assigns_through_the_graph(metric):
    data = _data(6000, 16, 1)
    ix = lb.IvfFlatIndex.build(data, metric, num_partitions=96, max_iters=5, seed=4, partition_index="hnsw")
    ex = ix.export()
    _check_parts(ex, data, metric, 4)
    exact = lb.IvfFlatIndex.build(data, metric, num_partitions=96, max_iters=5, seed=4).export()
    assert np.array_equal(exact["centroids"], ex["centroids"])   # training never uses the graph
    # transform of the built index uses its graph too
    t = ix.transform(data)
    part, valid = _check_parts(ex, data, metric, 4)
    assert np.array_equal(t["part_ids"][valid], part[valid]) and np.array_equal(t["valid"], valid)


@pytest.mark.gpu
@pytest.mark.parametrize("metric", ["l2", "dot"])
@pytest.mark.parametrize("nbits", [8, 4])
def test_ivf_pq_build_assigns_and_encodes_through_the_graph(metric, nbits):
    data = _data(6000, 32, 2)
    p = lb.IvfBuildParams(num_partitions=80, num_sub_vectors=8, num_bits=nbits, max_iters=5, pq_max_iters=5, seed=7,
                          partition_index="hnsw")
    ix = lb.IvfPqIndex.build(data, metric, p)
    ex = ix.export()
    part, valid = _check_parts(ex, data, metric, 7)
    t = ix.transform(data)      # the index's own transform: the graph's partitions and their residual codes
    assert np.array_equal(t["part_ids"][valid], part[valid])
    codes = _row_payload(ex, "codes", data.shape[0])
    assert np.array_equal(codes[valid], t["payload"][valid])


@pytest.mark.gpu
def test_ivf_sq_and_hnsw_flat_builds_assign_through_the_graph():
    data = _data(5000, 16, 3)
    ix = lb.IvfSqIndex.build(data, "l2", num_partitions=64, max_iters=5, seed=2, partition_index="hnsw",
                             partition_index_batch=16)
    ex = ix.export()
    pi = lb.PartitionIndex.build(ex["centroids"], "l2", mode="hnsw", seed=_graph_seed(2), insert_batch=16)
    part, _, valid = pi.assign(data)
    assert np.array_equal(_parts_by_row(ex, len(data))[valid], part[valid].astype(np.uint64))
    t = ix.transform(data)
    assert np.array_equal(_row_payload(ex, "codes", len(data))[valid], t["payload"][valid])
    hx = lb.IvfHnswFlatIndex.build(data, "l2", num_partitions=64, max_iters=5, seed=2, partition_index="hnsw",
                                   hnsw_params=lb.HnswBuildParams(m=8, ef_construction=20))
    _check_parts(hx.export(), data, "l2", 2)


@pytest.mark.gpu
@pytest.mark.parametrize("metric", ["l2", "dot"])
def test_ivf_rq_build_codes_and_factors_follow_the_graph(metric):
    data = _data(5000, 32, 4)
    ix = lb.IvfRqIndex.build(data, metric, num_partitions=64, max_iters=5, seed=3, partition_index="hnsw")
    ex = ix.export()
    part, valid = _check_parts(ex, data, metric, 3)
    t = ix.transform(data)
    assert np.array_equal(t["part_ids"][valid], part[valid])
    n = len(data)
    assert np.array_equal(_row_payload(ex, "codes", n)[valid], t["payload"][valid])
    for key in ("add_factors", "scale_factors"):
        assert np.array_equal(_row_payload(ex, key, n)[valid].view(np.uint32), t[key][valid].view(np.uint32))


@pytest.mark.gpu
def test_auto_builds_switch_at_one_million_values():
    d = 1000
    data = _data(3000, d, 5)
    for k, graph in ((999, False), (1000, True)):
        auto = lb.IvfFlatIndex.build(data, "l2", num_partitions=k, max_iters=1, seed=1, partition_index="auto").export()
        want = lb.IvfFlatIndex.build(data, "l2", num_partitions=k, max_iters=1, seed=1,
                                     partition_index="hnsw" if graph else "exact").export()
        for key in ("centroids", "part_offsets", "row_ids", "vectors"):
            assert np.array_equal(auto[key], want[key]), (k, key)
    assert cg.uses_graph(1000, d, "f32", "auto") and not cg.uses_graph(999, d, "f32", "auto")


@pytest.mark.gpu
def test_optimize_keeps_the_rule_over_its_new_centroids():
    data = _data(5000, 16, 6)
    ix = lb.IvfFlatIndex.build(data[:4000], "l2", num_partitions=48, max_iters=5, seed=9, partition_index="hnsw")
    rng = np.random.default_rng(0)
    new_c = ix.export()["centroids"] + rng.standard_normal((48, 16)).astype(np.float32) * np.float32(0.2)
    opt = ix.optimize(add_vectors=data[4000:], add_row_ids=np.arange(4000, 5000, dtype=np.uint64), new_centroids=new_c)
    want, _, valid = lb.PartitionIndex.build(new_c, "l2", mode="hnsw", seed=_graph_seed(9)).assign(data)
    t = opt.transform(data)
    assert np.array_equal(t["part_ids"][valid], want[valid])
    ex = opt.export()
    got = _parts_by_row(ex, 5000)
    # appended rows went through the old index's graph (transform before the merge)
    old_part, _, v_old = lb.PartitionIndex.build(ix.export()["centroids"], "l2", mode="hnsw",
                                                 seed=_graph_seed(9)).assign(data[4000:])
    assert np.array_equal(got[4000:][v_old[:]], old_part[v_old].astype(np.uint64))


@pytest.mark.gpu
def test_set_partition_index_on_an_index_opened_from_storage():
    data = _data(4000, 16, 7)
    ex_ix = lb.IvfFlatIndex.build(data, "l2", num_partitions=40, max_iters=5, seed=1)
    cent = ex_ix.export()["centroids"]
    opened = lb.IvfFlatIndex.from_storage(cent, ex_ix.export_storage())
    exact = opened.transform(data)
    ref_exact = lb.compute_partitions(cent, data, "l2")
    assert np.array_equal(exact["part_ids"][ref_exact[2]], ref_exact[0][ref_exact[2]])
    opened.set_partition_index("hnsw", seed=21, insert_batch=4)
    want, _, valid = lb.PartitionIndex.build(cent, "l2", mode="hnsw", seed=21, insert_batch=4).assign(data)
    assert np.array_equal(opened.transform(data)["part_ids"][valid], want[valid])
    opened.set_partition_index("exact")
    assert np.array_equal(opened.transform(data)["part_ids"], exact["part_ids"])


@pytest.mark.gpu
def test_kmeans_train_refuses_a_partition_index():
    data = _data(2000, 16, 8)
    p = _lib.KMeansParams()
    _lib.lib().lb2_kmeans_params_default(C.byref(p))
    p.partition_index = 2
    cent = np.empty((8, 16), np.float32)
    st = _lib.lib().lb2_kmeans_train(C.c_void_p(data.ctypes.data), C.c_uint64(2000), C.c_uint32(16), C.c_int(0),
                                     C.c_uint32(8), C.byref(p), C.c_void_p(cent.ctypes.data), None, None)
    assert st == _lib.INVALID_ARG
    p.partition_index = 0
    st = _lib.lib().lb2_kmeans_train(C.c_void_p(data.ctypes.data), C.c_uint64(2000), C.c_uint32(16), C.c_int(0),
                                     C.c_uint32(8), C.byref(p), C.c_void_p(cent.ctypes.data), None, None)
    assert st == _lib.OK


@pytest.mark.gpu
@pytest.mark.parametrize("metric", ["l2", "dot"])
def test_many_rows_per_warp_against_the_restatement(metric):
    """20 000 rows at K = 4096: far more rows than resident warps, so every warp runs its persistent loop and reuses
    its bitset.  Zero rows tie every centroid under dot (1 - 0), so their beam search visits all 4096 nodes, more than
    the 512 a warp records, and the warp clears its whole bitset"""
    rng = np.random.default_rng(11)
    cent = rng.standard_normal((4096, 8)).astype(np.float32)
    rows = (cent[rng.integers(0, 4096, 20000)] + rng.standard_normal((20000, 8)).astype(np.float32) * np.float32(0.4))
    rows = rows.astype(np.float32)
    rows[::50] = rng.standard_normal((400, 8)).astype(np.float32) * np.float32(40.0)   # far from every centroid
    rows[7, 3] = np.inf
    rows[1::997] = 0.0
    pi = lb.PartitionIndex.build(cent, metric, mode="hnsw", seed=12, insert_batch=16)
    got = pi.assign(rows)
    want = cg.assign(pi.export(), cent, rows, metric)
    gp, gd, gv = got
    wp, wd, wv = want
    assert np.array_equal(gv, wv) and np.array_equal(gp, wp)
    assert np.array_equal(gd[wv].view(np.uint32), wd[wv].view(np.uint32))
