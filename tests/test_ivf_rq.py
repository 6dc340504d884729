"""IVF_RQ on the device against the restatement of the reference (tests/rq_reference.py): the transform's codes and
factors, the build (IVF_FLAT's IVF stage plus the transform of its stored vectors) and every search result (ids,
distances, counts) bit for bit, ties at the k-th distance included."""
import numpy as np
import pytest

import lance_b200 as lb
from oracle import binding as ob
from rq_reference import ivfrq_search, rq_transform

pytestmark = pytest.mark.gpu

SIZES = (0, 1, 31, 32, 33, 4097)        # around the 32-row blocks and the scan's 4096-row chunk


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _rotation(code_dim, seed=1):
    return lb.RabitQuantizer(code_dim, 1).build(seed)


# ---- transform ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("metric", ["l2", "cosine", "dot"])
@pytest.mark.parametrize("num_bits", [1, 2])
@pytest.mark.parametrize("d", [8, 16, 120, 128, 1024, 1032])
def test_transform_bit_exact(metric, num_bits, d):
    rng = np.random.default_rng(d * 10 + num_bits)
    n, K = (300 if d <= 128 else 40), 4
    cent = rng.standard_normal((K, d)).astype(np.float32)
    if metric == "cosine":
        cent = ob.normalize_rows(cent)
    x = rng.standard_normal((n, d)).astype(np.float32)
    x[3, 1] = np.nan                   # dropped
    x[4] = 0.0                         # dropped under cosine
    x[5] = cent[2]                     # a row equal to its centroid: ip = 0
    rq = lb.RabitQuantizer(d, num_bits)
    rq.build(seed=d)
    got = rq.transform(cent, x, metric)
    part, codes, add, scale, valid = rq_transform(cent, rq.rotation, x, metric, num_bits)
    assert np.array_equal(got["valid"], valid)
    assert not valid[3] and valid[5] and valid[4] == (metric != "cosine")
    assert np.array_equal(got["part_ids"][valid], part[valid])
    assert np.array_equal(got["codes"], codes)
    assert np.array_equal(_bits(got["add_factors"]), _bits(add))
    assert np.array_equal(_bits(got["scale_factors"]), _bits(scale))
    if metric != "cosine":
        assert scale[5] == 0 and got["scale_factors"][5] == 0


def test_rotation_is_orthogonal_and_seeded():
    r1, r2, r3 = _rotation(128, 5), _rotation(128, 5), _rotation(128, 6)
    assert np.array_equal(r1, r2) and not np.array_equal(r1, r3)
    r = r1.astype(np.float64)
    assert np.allclose(r @ r.T, np.eye(128), atol=1e-5, rtol=0)


# ---- build -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("metric", ["l2", "cosine", "dot"])
def test_build_equals_ivf_flat_stage_and_the_transform(metric):
    from lance_b200 import synth
    rng = np.random.default_rng(11)
    n, d, K = 6000, 32, 8
    x = synth.gaussian_mixture(n, d, n_components=16, seed=3)
    x[rng.choice(n, 20, replace=False)] = 0.0
    x[rng.choice(n, 5, replace=False), 3] = np.nan
    kw = dict(num_partitions=K, max_iters=10, seed=7)
    rq = lb.IvfRqIndex.build(x, metric, **kw)
    fl = lb.IvfFlatIndex.build(x, metric, **kw)
    r, f = rq.export(), fl.export()
    assert np.array_equal(r["centroids"], f["centroids"])
    assert np.array_equal(r["part_offsets"], f["part_offsets"])
    assert np.array_equal(r["row_ids"], f["row_ids"])
    rows = f["row_ids"].astype(np.int64)
    part, codes, add, scale, valid = rq_transform(f["centroids"], r["rotation"], x[rows], metric)
    assert valid.all()
    assert np.array_equal(r["codes"], codes)
    assert np.array_equal(_bits(r["add_factors"]), _bits(add)) and np.array_equal(_bits(r["scale_factors"]), _bits(scale))
    assert np.array_equal(r["rotation"], _rotation(d, 8))       # the rotation comes from seed + 1
    rr = r["rotation"].astype(np.float64)
    assert np.allclose(rr @ rr.T, np.eye(d), atol=1e-5, rtol=0)
    info = rq.info()
    assert (info["num_sub_vectors"], info["num_bits"], info["num_rows"]) == (0, 1, rows.size)
    assert rq.stats.ms_pq_train > 0 and rq.stats.ms_transform > 0


def test_build_and_create_reject_what_is_not_implemented():
    x = np.random.default_rng(0).random((300, 16), dtype=np.float32)
    cases = [(lambda: lb.IvfRqIndex.build(x.astype(np.float16), "l2", num_partitions=4), lb._lib.UNSUPPORTED),
             (lambda: lb.IvfRqIndex.build(x.astype(np.uint8), "l2", num_partitions=4), lb._lib.INVALID_ARG),
             (lambda: lb.IvfRqIndex.build(x[:, :12], "l2", num_partitions=4), lb._lib.INVALID_ARG),
             (lambda: lb.IvfRqIndex.from_parts(np.zeros((2, 12), np.float32), np.eye(12), [0], np.zeros((1, 1)),
                                               [0], [0]), lb._lib.INVALID_ARG),
             (lambda: lb.IvfRqIndex.from_parts(np.zeros((2, 16), np.float16), np.eye(16), [0], np.zeros((1, 2)), [0],
                                               [0], dtype=np.float16), lb._lib.UNSUPPORTED),
             (lambda: lb.IvfRqIndex.from_parts(np.zeros((2, 16)), np.eye(16), [0], np.zeros((1, 2)), [0], [0],
                                               dtype=np.uint8), lb._lib.INVALID_ARG),
             # code_dim 16 * 1024: the tables do not fit shared memory (checked before the rotation is read)
             (lambda: lb.IvfRqIndex.from_parts(np.zeros((2, 16)), np.zeros((1, 1)), [], np.zeros((0, 2048)), [], [],
                                               num_bits=1024), lb._lib.UNSUPPORTED)]
    for call, status in cases:
        with pytest.raises(lb.LanceB200Error) as e:
            call()
        assert e.value.status == status
    # bf16 columns: rejected like u8
    h = lb.C.c_void_p()
    z = np.zeros(2 * 16, np.uint16)
    assert lb.lib().lb2_index_create_rq(lb.C.c_void_p(z.ctypes.data), 2, 16, lb._lib.BF16, 0,
                                        lb.C.c_void_p(z.ctypes.data), 1, lb.C.byref(h)) == lb._lib.INVALID_ARG
    ix = lb.IvfRqIndex.from_parts(np.zeros((2, 16), np.float32), np.eye(16), np.zeros(3, np.uint32),
                                  np.zeros((3, 2), np.uint8), np.ones(3), np.ones(3))
    with pytest.raises(lb.LanceB200Error) as e:
        ix.update(add_part_ids=[0], add_codes=np.zeros((1, 2), np.uint8), add_row_ids=[9])
    assert e.value.status == lb._lib.INVALID_ARG
    with pytest.raises(lb.LanceB200Error) as e:
        ix.repartition()
    assert e.value.status == lb._lib.UNSUPPORTED
    for call in (lambda: lb.lib().lb2_index_export(ix._h, None, None, None, None, None),
                 lambda: lb.lib().lb2_index_load(ix._h, None, None, None, lb.C.c_uint64(0)),
                 lambda: lb.lib().lb2_index_export_partition(ix._h, 0, None, None, None)):
        assert call() == lb._lib.INVALID_ARG


# ---- search ------------------------------------------------------------------------------------------------------
def _index(d, metric, sizes=SIZES, seed=0, num_bits=1, dup=None):
    """from_parts at exact partition sizes: the transform of random rows around random centroids"""
    rng = np.random.default_rng(seed + d)
    K = len(sizes)
    cent = rng.standard_normal((K, d)).astype(np.float32)
    if metric == "cosine":
        cent = ob.normalize_rows(cent)
    n = int(sum(sizes))
    part = np.repeat(np.arange(K, dtype=np.uint32), sizes)
    rot = _rotation(d * num_bits, seed + 3)
    x = cent[part] + np.float32(0.5) * rng.standard_normal((n, d)).astype(np.float32)
    if dup is not None:                                          # a few distinct rows repeated: ties
        x = x[rng.integers(0, dup, size=n)]
    _, codes, add, scale, _ = rq_transform(cent, rot, x, "dot" if metric == "dot" else "l2", num_bits)
    perm = rng.permutation(n)                                    # rows arrive unsorted; the load groups them
    rid = rng.permutation(n).astype(np.uint64)
    ix = lb.IvfRqIndex.from_parts(cent, rot, part[perm], codes[perm], add[perm], scale[perm], rid[perm], metric,
                                  num_bits=num_bits)
    offs = np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint64)
    order = perm[np.argsort(part[perm], kind="stable")]         # the storage order the load produces
    return ix, (cent, rot, offs, codes[order], add[order], scale[order], rid[order])


def _same(got, want):
    (gi, gd), (wi, wd, wc) = got, want
    for i in range(wi.shape[0]):
        c = int(wc[i])
        assert np.array_equal(gi[i, :c], wi[i, :c]), i
        assert np.array_equal(gd[i, :c].view(np.uint32), wd[i, :c].view(np.uint32)), i
        assert (gi[i, c:] == np.iinfo(np.uint64).max).all() and np.isinf(gd[i, c:]).all(), i


@pytest.mark.parametrize("metric", ["l2", "cosine", "dot"])
@pytest.mark.parametrize("d,num_bits", [(16, 1), (16, 2), (128, 1), (120, 1)])
def test_search_bit_exact(metric, d, num_bits):
    ix, m = _index(d, metric, num_bits=num_bits)
    q = np.random.default_rng(100 + d).standard_normal((5, d)).astype(np.float32)
    for k, nprobes in ((1, 6), (10, 3), (17, 6), (100, 6), (1024, 2), (1024, 6)):
        _same(ix.search(q, k=k, nprobes=nprobes), ivfrq_search(*m, q, k, nprobes, metric=metric))


def test_search_zero_query_under_cosine():
    ix, m = _index(16, "cosine")
    q = np.zeros((2, 16), np.float32)
    q[1, 0] = 1.0
    _same(ix.search(q, k=10, nprobes=6), ivfrq_search(*m, q, 10, 6, metric="cosine"))


@pytest.mark.parametrize("metric", ["l2", "dot"])
def test_search_ties_at_the_kth_distance(metric):
    ix, m = _index(16, metric, sizes=(4097, 33, 64), dup=5)
    q = np.random.default_rng(2).standard_normal((3, 16)).astype(np.float32)
    for k in (1, 10, 17, 100, 1024):
        _same(ix.search(q, k=k, nprobes=3), ivfrq_search(*m, q, k, 3, metric=metric))


@pytest.mark.parametrize("metric", ["l2", "cosine", "dot"])
def test_search_prefilter_range_async_sharded(metric):
    d = 32
    ix, m = _index(d, metric, seed=4)
    q = np.random.default_rng(9).standard_normal((4, d)).astype(np.float32)
    rng = np.random.default_rng(2)
    n = int(m[2][-1])
    allow = rng.choice(n, n // 2, replace=False).astype(np.uint64)
    bm = ix.row_mask(allow_row_ids=allow)
    for k in (10, 100):
        _same(ix.search_ex(q, k=k, nprobes=6, allow_bitmap=bm), ivfrq_search(*m, q, k, 6, metric=metric, allow=allow))
    _, d0 = ix.search(q, k=200, nprobes=6)
    lo, hi = float(d0[0, 20]), float(d0[0, 150])
    for k in (10, 100):
        _same(ix.search_ex(q, k=k, nprobes=6, lower_bound=lo, upper_bound=hi),
              ivfrq_search(*m, q, k, 6, metric=metric, lower=lo, upper=hi))
        _same(ix.search_ex(q, k=k, nprobes=6, allow_bitmap=bm, upper_bound=hi),
              ivfrq_search(*m, q, k, 6, metric=metric, allow=allow, upper=hi))
    want_i, want_d = ix.search(q, k=50, nprobes=5)
    qd = lb.DeviceArray.from_numpy(q)
    oi, od = lb.DeviceArray((4, 50), np.uint64), lb.DeviceArray((4, 50), np.float32)
    ix.search_async(qd, (oi, od), k=50, nprobes=5)
    lb.synchronize()
    assert np.array_equal(oi.numpy(), want_i) and np.array_equal(od.numpy().view(np.uint32), want_d.view(np.uint32))
    si, sd = ix.search_sharded(q, k=50, nprobes=5)
    assert np.array_equal(si, want_i) and np.array_equal(sd.view(np.uint32), want_d.view(np.uint32))


@pytest.mark.parametrize("metric", ["l2", "dot"])
def test_search_refine(metric):
    d = 64
    ix, m = _index(d, metric, seed=6)
    n = int(m[2][-1])
    raw = np.random.default_rng(8).standard_normal((n, d)).astype(np.float32)   # the column, row id = row number
    q = np.random.default_rng(12).standard_normal((3, d)).astype(np.float32)
    dist = ob.l2 if metric == "l2" else (lambda a, b: np.float32(1.0) - np.float32(ob.dot(a, b)))
    for k, rf in ((10, 10), (100, 4)):
        cands, _, cc = ivfrq_search(*m, q, k * rf, 6, metric=metric)
        ids, dists = ix.search_refine(raw, q, k=k, nprobes=6, refine_factor=rf)
        for i in range(q.shape[0]):
            c = cands[i, :cc[i]]
            ex = np.array([dist(q[i], raw[j]) for j in c], np.float32)
            order = np.lexsort((c, ex))[:k]
            assert np.array_equal(ids[i], c[order]), (k, rf, i)
            assert np.allclose(dists[i], ex[order], rtol=1e-6, atol=1e-6), (k, rf, i)


def test_round_trip_from_parts_export():
    ix, (cent, rot, offs, codes, add, scale, rid) = _index(16, "l2", num_bits=2)
    e = ix.export()
    assert np.array_equal(e["centroids"], cent) and np.array_equal(e["rotation"], rot)
    assert np.array_equal(e["part_offsets"], offs) and np.array_equal(e["codes"], codes)
    assert np.array_equal(_bits(e["add_factors"]), _bits(add)) and np.array_equal(_bits(e["scale_factors"]), _bits(scale))
    assert np.array_equal(e["row_ids"], rid)
    back = lb.IvfRqIndex.from_parts(e["centroids"], e["rotation"], np.repeat(np.arange(len(SIZES)), SIZES), e["codes"],
                                    e["add_factors"], e["scale_factors"], e["row_ids"], num_bits=2)
    q = np.random.default_rng(1).standard_normal((3, 16)).astype(np.float32)
    a, b = ix.search(q, k=20, nprobes=6), back.search(q, k=20, nprobes=6)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1].view(np.uint32), b[1].view(np.uint32))


# ---- recall ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nlist", [1, 4])
@pytest.mark.parametrize("metric", ["l2", "cosine", "dot"])
def test_recall_floor(metric, nlist):
    """test_build_ivf_rq (rust/lance/src/index/vector/ivf/v2.rs:1423-1449, test_recall :1962-2007): 512 x 32 rows
    uniform in [0, 1), k = 100, nprobes = nlist, recall >= 0.5 against exact ground truth (IVF_FLAT, every
    partition).  The reference queries with row 0; the first 16 rows are used here, each held to the floor."""
    x = np.random.default_rng(nlist).random((512, 32), dtype=np.float32)
    q = x[:16]
    rq = lb.IvfRqIndex.build(x, metric, num_partitions=nlist, seed=0)
    fl = lb.IvfFlatIndex.build(x, metric, num_partitions=nlist, seed=0)
    gt, _ = fl.search(q, k=100, nprobes=nlist)
    ids, _ = rq.search(q, k=100, nprobes=nlist)
    r = np.array([len(set(a.tolist()) & set(b.tolist())) / 100 for a, b in zip(ids, gt)])
    print(f"IVF_RQ recall@100 ({metric}, nlist {nlist}): min {r.min():.2f}, mean {r.mean():.3f}")
    assert r.min() >= 0.5
