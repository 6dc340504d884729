"""IVF_SQ on the device against the restatement of the reference (tests/sq_reference.py): the quantizer bit for bit,
the build equal to IVF_FLAT's IVF stage plus scale_to_u8 of its stored vectors, and every search result (ids,
distances, counts) bit-identical, ties at the k-th distance included."""
import numpy as np
import pytest

import lance_b200 as lb
from oracle import binding as ob
from sq_reference import bf16_to_f32, ivfsq_search, sq_bounds, sq_encode

pytestmark = pytest.mark.gpu

SIZES = (0, 1, 4095, 4096, 4097, 12003)     # around the scan's 4096-row chunk


def _bf16_bits(x):
    """f32 -> bfloat16 bit patterns (round to nearest even), so the values are exact bf16 numbers"""
    b = np.ascontiguousarray(x, np.float32).view(np.uint32).astype(np.uint64)
    return ((b + 0x7FFF + ((b >> 16) & 1)) >> 16).astype(np.uint16)


# ---- quantizer ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", ["f32", "f16", "bf16", "u8"])
def test_quantizer_bit_exact(dt):
    rng = np.random.default_rng(5)
    d = 16
    x = (rng.standard_normal((257, d)) * 3).astype(np.float32)
    if dt != "u8":
        x[3, 2], x[7, 0], x[9, 5], x[11, 11] = np.nan, np.inf, -np.inf, np.nan
    if dt == "f32":
        arr, vals, kw = x, x, {}
    elif dt == "f16":
        arr = x.astype(np.float16)
        vals, kw = arr.astype(np.float32), {}
    elif dt == "bf16":
        arr = _bf16_bits(x)
        vals, kw = bf16_to_f32(arr), {"bf16": True}
    else:
        arr = rng.integers(0, 256, size=(257, d), dtype=np.uint8)
        vals, kw = arr.astype(np.float32), {}
    sq = lb.ScalarQuantizer(d)
    assert sq.build(arr, **kw) == sq_bounds(vals)
    finite = vals[np.isfinite(vals)]
    for b in (sq_bounds(vals), (-1.25, 2.5), (float(finite.min()) / 2, float(finite.max()) / 2), (0.5, 0.5),
              (0.0, 3.0)):
        sq.bounds = b
        assert np.array_equal(sq.transform(arr, **kw), sq_encode(vals, *b)), b


def test_quantizer_reference_literals():
    # test_f16_sq8 / test_f32_sq8 (sq.rs:296-350) and test_scale_to_u8_with_nan (sq.rs:372-389)
    for a in (np.arange(16, dtype=np.float32), np.arange(16, dtype=np.float16)):
        sq = lb.ScalarQuantizer(16)
        assert sq.build(a) == (0.0, 15.0)
        assert np.array_equal(sq.transform(a)[0], (np.arange(16) * 17).astype(np.uint8))
    sq = lb.ScalarQuantizer(4, bounds=(0.0, 3.0))
    assert sq.transform(np.array([[0, 1, 2, 3], [np.nan, 0, 0, 0]], np.float32))[:, 0].tolist() == [0, 0]
    assert sq.transform(np.array([[0, 1, 2, 3]], np.float32))[0].tolist() == [0, 85, 170, 255]
    assert sq.transform(np.array([[np.nan, 4, -1, 3]], np.float32))[0].tolist() == [0, 255, 0, 255]


# ---- build -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("metric", ["l2", "cosine", "dot"])
@pytest.mark.parametrize("dt", ["f32", "f16"])
def test_build_equals_ivf_flat_stage_and_scale_to_u8(metric, dt):
    rng = np.random.default_rng(11)
    n, d, K = 6000, 32, 8
    from lance_b200 import synth
    x = synth.gaussian_mixture(n, d, n_components=16, seed=3)
    x[rng.choice(n, 20, replace=False)] = 0.0                     # zero rows: dropped under cosine
    x[rng.choice(n, 5, replace=False), 3] = np.nan                # dropped in every metric
    if dt == "f16":
        x = x.astype(np.float16)
    kw = dict(num_partitions=K, max_iters=10, seed=7)
    sq = lb.IvfSqIndex.build(x, metric, **kw)
    fl = lb.IvfFlatIndex.build(x, metric, **kw)
    s, f = sq.export(), fl.export()
    assert np.array_equal(s["centroids"], f["centroids"])
    assert np.array_equal(s["part_offsets"], f["part_offsets"])
    assert np.array_equal(s["row_ids"], f["row_ids"])
    stored = f["vectors"].astype(np.float32)
    assert s["bounds"] == sq_bounds(stored)                       # n <= 65 536: the sample is every stored row
    assert np.array_equal(s["codes"], sq_encode(stored, *s["bounds"]))
    info = sq.info()
    assert (info["num_sub_vectors"], info["num_bits"], info["num_rows"]) == (0, 8, stored.shape[0])
    assert sq.stats.ms_pq_train > 0


def test_build_past_the_sq_sample():
    from lance_b200 import synth
    n, d = 70000, 16
    x = synth.gaussian_mixture(n, d, n_components=32, seed=9)
    sq = lb.IvfSqIndex.build(x, "l2", num_partitions=16, max_iters=5, seed=2)
    fl = lb.IvfFlatIndex.build(x, "l2", num_partitions=16, max_iters=5, seed=2)
    s, f = sq.export(), fl.export()
    assert np.array_equal(s["part_offsets"], f["part_offsets"]) and np.array_equal(s["row_ids"], f["row_ids"])
    lo, hi = s["bounds"]
    assert lo >= float(f["vectors"].min()) and hi <= float(f["vectors"].max())
    assert np.array_equal(s["codes"], sq_encode(f["vectors"], lo, hi))


def test_build_rejects_what_is_not_implemented():
    x = np.random.default_rng(0).random((300, 16), dtype=np.float32)
    with pytest.raises(lb.LanceB200Error) as e:
        lb.IvfSqIndex.build(x, "l2", num_partitions=4, sq_params=lb.SQBuildParams(num_bits=4))
    assert e.value.status == lb._lib.UNSUPPORTED
    with pytest.raises(lb.LanceB200Error) as e:
        lb.IvfSqIndex.build(np.zeros((300, 18), np.float32), "l2", num_partitions=4)
    assert e.value.status == lb._lib.INVALID_ARG
    for bounds in ((1.0, 0.0), (0.0, np.inf), (np.nan, 1.0)):
        with pytest.raises(lb.LanceB200Error) as e:
            lb.IvfSqIndex.from_parts(np.zeros((2, 16), np.float32), bounds, np.zeros(3, np.uint32),
                                     np.zeros((3, 16), np.uint8))
        assert e.value.status == lb._lib.INVALID_ARG
    ix = lb.IvfSqIndex.from_parts(np.zeros((2, 16), np.float32), (0.0, 1.0), np.zeros(3, np.uint32),
                                  np.zeros((3, 16), np.uint8))
    with pytest.raises(lb.LanceB200Error):
        ix.update(add_part_ids=[0], add_codes=np.zeros((1, 16), np.uint8), add_row_ids=[9])
    for call in (lambda: lb.lib().lb2_index_export(ix._h, None, None, None, None, None),
                 lambda: lb.lib().lb2_index_load(ix._h, None, None, None, lb.C.c_uint64(0)),
                 lambda: lb.lib().lb2_index_export_partition(ix._h, 0, None, None, None)):
        assert call() == lb._lib.INVALID_ARG


# ---- search ------------------------------------------------------------------------------------------------------
def _index(d, metric, sizes=SIZES, seed=0, bounds=(-1.5, 2.0), dtype=np.float32, bf16=False, extremes=False):
    """from_parts at exact partition sizes: random centroids, codes and (shuffled) row ids"""
    rng = np.random.default_rng(seed + d)
    K = len(sizes)
    cent = rng.standard_normal((K, d)).astype(np.float32)
    if metric == "cosine":
        cent = ob.normalize_rows(cent)
    n = int(sum(sizes))
    part = np.repeat(np.arange(K, dtype=np.uint32), sizes)
    codes = rng.integers(0, 256, size=(n, d), dtype=np.uint8)
    if extremes:
        codes = np.where(rng.random((n, d)) < 0.5, 0, 255).astype(np.uint8)
    perm = rng.permutation(n)                                    # rows arrive unsorted; the load groups them
    rid = rng.permutation(n).astype(np.uint64)
    if bf16:
        cent = bf16_to_f32(_bf16_bits(cent))
    elif dtype == np.float16:
        cent = cent.astype(np.float16).astype(np.float32)
    ix = lb.IvfSqIndex.from_parts(cent if not bf16 else _bf16_bits(cent), bounds, part[perm], codes[perm],
                                  rid[perm], metric, dtype=dtype, bf16=bf16)
    offs = np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint64)
    order = perm[np.argsort(part[perm], kind="stable")]         # the storage order the load produces
    return ix, cent, offs, codes[order], rid[order]


def _queries(nq, d, seed, extremes=False):
    rng = np.random.default_rng(seed)
    q = (rng.random((nq, d)) * 4.5 - 2.25).astype(np.float32)   # partly outside the bounds (-1.5, 2.0)
    if extremes:
        q = np.where(rng.random((nq, d)) < 0.5, -3.0, 3.0).astype(np.float32)
    return q


def _same(got, want):
    (gi, gd), (wi, wd, wc) = got, want
    for i in range(wi.shape[0]):
        c = int(wc[i])
        assert np.array_equal(gi[i, :c], wi[i, :c]), i
        assert np.array_equal(gd[i, :c].view(np.uint32), wd[i, :c].view(np.uint32)), i
        assert (gi[i, c:] == np.iinfo(np.uint64).max).all() and np.isinf(gd[i, c:]).all(), i


@pytest.mark.parametrize("metric", ["l2", "cosine", "dot"])
@pytest.mark.parametrize("d", [4, 8, 20, 128, 140, 512])
def test_search_bit_exact(metric, d):
    extremes = d == 512                      # codes at 0 and 255: the u32 sums pass 2^24 and `s as f32` rounds
    ix, cent, offs, codes, rid = _index(d, metric, extremes=extremes)
    q = _queries(6, d, 100 + d, extremes=extremes)
    bounds = (-1.5, 2.0)
    for k, nprobes in ((1, 6), (10, 3), (17, 6), (100, 6), (1024, 2), (1024, 6)):   # np * k on both sides of 2048
        want = ivfsq_search(cent, bounds, offs, codes, rid, q, k, nprobes, metric=metric)
        _same(ix.search(q, k=k, nprobes=nprobes), want)


@pytest.mark.parametrize("qdt", ["f16", "bf16"])
@pytest.mark.parametrize("metric", ["l2", "cosine", "dot"])
def test_search_16bit_queries(qdt, metric):
    d = 128
    kw = {"bf16": True} if qdt == "bf16" else {"dtype": np.float16}
    ix, cent, offs, codes, rid = _index(d, metric, seed=3, **kw)
    q32 = _queries(5, d, 7)
    if qdt == "bf16":
        qn = _bf16_bits(q32)
        qv = bf16_to_f32(qn)
    else:
        qn = q32.astype(np.float16)
        qv = qn.astype(np.float32)
    for k in (10, 100):
        _same(ix.search(qn, k=k, nprobes=4), ivfsq_search(cent, (-1.5, 2.0), offs, codes, rid, qv, k, 4, metric=metric))


@pytest.mark.parametrize("metric", ["l2", "dot"])
def test_search_ties_at_the_kth_distance(metric):
    d, sizes = 16, (4097, 12003, 5)
    rng = np.random.default_rng(1)
    # a constant column: equal bounds, every code 0, every distance 0 -> the heap's sift order decides
    ix, cent, offs, codes, rid = _index(d, metric, sizes=sizes, bounds=(0.75, 0.75))
    z = np.zeros_like(codes)
    ix = lb.IvfSqIndex.from_parts(cent, (0.75, 0.75), np.repeat(np.arange(3, dtype=np.uint32), sizes), z, rid, metric)
    q = _queries(3, d, 2)
    for k in (1, 10, 100, 1024):
        _same(ix.search(q, k=k, nprobes=3), ivfsq_search(cent, (0.75, 0.75), offs, z, rid, q, k, 3, metric=metric))
    # duplicated rows: a few distinct codes repeated many times
    base = rng.integers(0, 256, size=(7, d), dtype=np.uint8)
    dup = base[rng.integers(0, 7, size=int(sum(sizes)))]
    ix = lb.IvfSqIndex.from_parts(cent, (-1.5, 2.0), np.repeat(np.arange(3, dtype=np.uint32), sizes), dup, rid, metric)
    for k in (10, 17, 100, 1024):
        _same(ix.search(q, k=k, nprobes=3), ivfsq_search(cent, (-1.5, 2.0), offs, dup, rid, q, k, 3, metric=metric))


@pytest.mark.parametrize("metric", ["l2", "cosine", "dot"])
def test_search_prefilter_range_async_sharded_repartition(metric):
    d = 20
    ix, cent, offs, codes, rid = _index(d, metric, seed=4)
    q = _queries(4, d, 9)
    bounds = (-1.5, 2.0)
    rng = np.random.default_rng(2)
    allow = rng.choice(int(offs[-1]), 9000, replace=False).astype(np.uint64)
    bm = ix.row_mask(allow_row_ids=allow)
    for k in (10, 100):
        _same(ix.search_ex(q, k=k, nprobes=6, allow_bitmap=bm),
              ivfsq_search(cent, bounds, offs, codes, rid, q, k, 6, metric=metric, allow=allow))
    _, d0 = ix.search(q, k=200, nprobes=6)
    lo, hi = float(d0[0, 20]), float(d0[0, 150])
    for k in (10, 100):
        _same(ix.search_ex(q, k=k, nprobes=6, lower_bound=lo, upper_bound=hi),
              ivfsq_search(cent, bounds, offs, codes, rid, q, k, 6, metric=metric, lower=lo, upper=hi))
        _same(ix.search_ex(q, k=k, nprobes=6, allow_bitmap=bm, upper_bound=hi),
              ivfsq_search(cent, bounds, offs, codes, rid, q, k, 6, metric=metric, allow=allow, upper=hi))
    want_i, want_d = ix.search(q, k=50, nprobes=5)
    qd = lb.DeviceArray.from_numpy(q)
    oi, od = lb.DeviceArray((4, 50), np.uint64), lb.DeviceArray((4, 50), np.float32)
    ix.search_async(qd, (oi, od), k=50, nprobes=5)
    lb.synchronize()
    assert np.array_equal(oi.numpy(), want_i) and np.array_equal(od.numpy().view(np.uint32), want_d.view(np.uint32))
    si, sd = ix.search_sharded(q, k=50, nprobes=5)
    assert np.array_equal(si, want_i) and np.array_equal(sd.view(np.uint32), want_d.view(np.uint32))
    rp = ix.repartition()
    ri, rd = rp.search(q, k=50, nprobes=5)
    assert np.array_equal(ri, want_i) and np.array_equal(rd.view(np.uint32), want_d.view(np.uint32))
    assert rp.export()["bounds"] == ix.export()["bounds"]


@pytest.mark.parametrize("metric", ["l2", "dot"])
def test_search_refine(metric):
    d = 128
    ix, cent, offs, codes, rid = _index(d, metric, seed=6)
    n = int(offs[-1])
    raw = np.random.default_rng(8).standard_normal((n, d)).astype(np.float32)   # the column, row id = row number
    q = _queries(3, d, 12)
    dist = ob.l2 if metric == "l2" else (lambda a, b: np.float32(1.0) - np.float32(ob.dot(a, b)))
    for k, rf in ((10, 10), (100, 4)):
        cands, _, cc = ivfsq_search(cent, (-1.5, 2.0), offs, codes, rid, q, k * rf, 6, metric=metric)
        ids, dists = ix.search_refine(raw, q, k=k, nprobes=6, refine_factor=rf)
        for i in range(q.shape[0]):
            c = cands[i, :cc[i]]
            ex = np.array([dist(q[i], raw[j]) for j in c], np.float32)
            order = np.lexsort((c, ex))[:k]
            assert np.array_equal(ids[i], c[order]), (k, rf, i)
            assert np.allclose(dists[i], ex[order], rtol=1e-6, atol=1e-6), (k, rf, i)


# ---- recall ------------------------------------------------------------------------------------------------------
def test_recall_on_sift_shaped_data_at_least_ivf_pq():
    from lance_b200 import synth
    n, d, K, nq = 1_000_000, 128, 256, 1000
    x = synth.sift_like(n, d)
    q = synth.sift_like_queries(nq, d)
    xd = lb.DeviceArray.from_numpy(x)
    sq = lb.IvfSqIndex.build(xd, "l2", num_partitions=K, max_iters=20, seed=0)
    cent = sq.export()["centroids"]
    pq = lb.IvfPqIndex.build(xd, "l2", lb.IvfBuildParams(num_partitions=K, num_sub_vectors=16, max_iters=20, seed=0))
    assert np.array_equal(pq.export()["centroids"], cent)        # same data, same IVF stage, same centroids
    fl = lb.IvfFlatIndex.build(xd, "l2", num_partitions=K, max_iters=20, seed=0)
    gt, _ = fl.search(q, k=10, nprobes=K)

    def recall(ix):
        ids, _ = ix.search(q, k=10, nprobes=10)
        return np.mean([len(set(a.tolist()) & set(b.tolist())) / 10 for a, b in zip(ids, gt)])

    r_sq, r_pq = recall(sq), recall(pq)
    print(f"recall@10 at nprobes 10: IVF_SQ {r_sq:.4f}, IVF_PQ(256, 16) {r_pq:.4f}")
    assert r_sq >= r_pq
