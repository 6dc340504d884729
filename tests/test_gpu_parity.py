"""GPU parity tests: the CUDA path (through the C ABI) against the CPU oracle on the same seeded
inputs.  Integer outputs (partition ids, PQ codes, probe ids) and f32 L2/Dot/ADC distances must be
BIT-EXACT; trained models are bit-exact given the same initial centroids (our training is
deterministic by construction, see lance_b200/csrc/lloyd.cu)."""
import numpy as np
import pytest

import lance_b200 as lb
from lance_b200 import synth
from oracle import binding as ob

pytestmark = pytest.mark.gpu
NT = 16


def test_device_present_and_native_library_loaded():
    assert lb.device_count() >= 1, "no GPU: -m gpu tests must run on an H100"
    lb.set_device(0)
    assert lb.launch_count(reset=True) >= 0


@pytest.mark.parametrize("d", [8, 5, 16, 32, 128, 100, 768])
def test_l2_distance_batch_bit_exact(d):
    rng = np.random.default_rng(d)
    x = rng.standard_normal(d).astype(np.float32)
    y = rng.standard_normal((77, d)).astype(np.float32)
    assert np.array_equal(lb.l2_distance_batch(x, y, d), ob.l2_batch(x, y, d))


def test_dot_distance_batch_bit_exact():
    rng = np.random.default_rng(0)
    for d in (8, 24, 128):
        x = rng.standard_normal(d).astype(np.float32)
        y = rng.standard_normal((33, d)).astype(np.float32)
        exp = np.array([np.float32(1.0) - np.float32(ob.dot(x, v)) for v in y], np.float32)
        assert np.array_equal(lb.dot_distance_batch(x, y, d), exp)


def test_reference_known_answers_on_gpu():
    import json, os
    cases = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "reference_known_answers.json")))
    for c in cases:
        if c["op"] == "l2_u8":      # l2.rs:431-447: the u8 kernel sums in u32
            x, y = np.asarray(c["x"], np.uint8), np.asarray(c["y"], np.uint8)
            assert float(lb.l2_distance_batch(x, y, x.size)[0]) == c["expect"] == float(lb.l2_distance_batch(y, x, x.size)[0])
            continue
        if c["op"] == "cosine":     # cosine.rs:361-393
            got = float(lb.cosine_distance_batch(np.asarray(c["x"], np.float32), np.asarray(c["y"], np.float32), len(c["x"]))[0])
            tol = c["abs"] if "abs" in c else c["rel"] * abs(c["expect"])
            assert abs(got - c["expect"]) <= tol, c["name"]
            continue
        if c["op"] != "l2_batch":
            continue
        got = lb.l2_distance_batch(c["frm"], c["to"], c["d"])
        exp = np.asarray(c["expect"], np.float64)
        if c.get("exact"):
            assert np.array_equal(got.astype(np.float64), exp), c["name"]
        else:
            assert np.all(np.abs(got - exp) <= c["rel"] * np.abs(exp)), c["name"]


@pytest.mark.parametrize("n,d,k", [(1000, 128, 256), (777, 128, 100), (513, 64, 17), (300, 8, 16),
                                   (300, 4, 256), (257, 40, 33), (100, 200, 7), (64, 768, 50)])
def test_compute_partitions_bit_exact(n, d, k):
    rng = np.random.default_rng(n + d + k)
    cent = rng.standard_normal((k, d)).astype(np.float32)
    data = rng.standard_normal((n, d)).astype(np.float32)
    p, dist, valid = lb.compute_partitions(cent, data)
    po, do, vo = ob.compute_membership(cent, data, nthreads=NT)
    assert np.array_equal(valid, vo) and valid.all()
    assert np.array_equal(p, po)
    assert np.array_equal(dist, do)


def test_compute_partitions_sift_shaped_integers_have_ties():
    # SIFT-like small integers -> many exactly equal distances: first-minimum rule must hold
    data = synth.sift_like(5000, 128, n_components=32, seed=3)
    cent = data[:256].copy()
    cent[10] = cent[3]  # duplicate centroid: index 3 must always win over 10
    p, dist, _ = lb.compute_partitions(cent, data)
    po, do, _ = ob.compute_membership(cent, data, nthreads=NT)
    assert np.array_equal(p, po) and np.array_equal(dist, do)
    assert not (p == 10).any()


def test_compute_partitions_nan_inf_rows_are_none():
    # kmeans.rs:1447-1486
    rng = np.random.default_rng(9)
    cent = rng.standard_normal((20, 32)).astype(np.float32)
    data = rng.standard_normal((50, 32)).astype(np.float32)
    data[3, 5] = np.nan
    data[7, :] = np.nan
    data[11, 0] = np.inf
    p, dist, valid = lb.compute_partitions(cent, data)
    po, do, vo = ob.compute_membership(cent, data)
    assert np.array_equal(valid, vo) and not valid[3] and not valid[7] and not valid[11]
    assert np.array_equal(p[valid], po[vo]) and np.array_equal(dist[valid], do[vo])


def test_compute_partitions_dot_metric():
    rng = np.random.default_rng(10)
    cent = rng.standard_normal((40, 64)).astype(np.float32)
    data = rng.standard_normal((333, 64)).astype(np.float32)
    p, dist, _ = lb.compute_partitions(cent, data, "dot")
    po, do, _ = ob.compute_membership(cent, data, metric="dot", nthreads=NT)
    assert np.array_equal(p, po) and np.array_equal(dist, do)


@pytest.mark.parametrize("n,d,k", [(6000, 32, 16), (20000, 128, 64), (3000, 8, 256)])
def test_kmeans_training_bit_exact_given_init(n, d, k):
    data = synth.gaussian_mixture(n, d, n_components=k, seed=n)
    init = data[np.random.default_rng(1).choice(n, k, replace=False)].copy()
    km = lb.train_kmeans(data, d, k, max_iters=20, centroids=init, balance_factor=1.0)
    nn = min(n, 256 * k)
    co, loss_o, it_o = ob.kmeans_train(data[:nn], k, max_iters=20,
                                       balance_factor=float(np.float32(1.0) / np.float32(nn)),
                                       init_centroids=init, nthreads=NT)
    assert km.iters == it_o
    assert np.array_equal(km.centroids, co)
    assert km.loss == loss_o


def test_kmeans_training_seeded_random_init_matches_oracle():
    data = synth.gaussian_mixture(8000, 32, n_components=32, seed=5)
    km = lb.train_kmeans(data, 32, 32, max_iters=15, seed=42)
    co, loss_o, it_o = ob.kmeans_train(data, 32, max_iters=15, seed=42, nthreads=NT)
    assert km.iters == it_o and np.array_equal(km.centroids, co) and km.loss == loss_o


def test_kmeans_empty_cluster_split():
    # duplicate init centroids force empty clusters -> split_clusters path (kmeans.rs:174-207)
    data = synth.gaussian_mixture(4000, 16, n_components=4, seed=8)
    init = np.repeat(data[:4], 4, axis=0).copy()  # 16 centroids, only 4 distinct
    km = lb.train_kmeans(data, 16, 16, max_iters=8, centroids=init, seed=3)
    co, loss_o, it_o = ob.kmeans_train(data, 16, max_iters=8, init_centroids=init, seed=3, nthreads=NT)
    assert km.iters == it_o and np.array_equal(km.centroids, co)
    assert np.isfinite(km.centroids).all()


def test_pq_training_bit_exact_given_codebook_init():
    rng = np.random.default_rng(4)
    n, d, M = 8000, 64, 8
    data = synth.gaussian_mixture(n, d, n_components=300, seed=4)
    init = np.stack([data[rng.choice(n, 256, replace=False)][:, m * 8:(m + 1) * 8] for m in range(M)])
    pq = lb.PQBuildParams(M, 8, max_iters=12, codebook=init).build(data)
    cbo, iters_o = ob.pq_train(data, M, max_iters=12, init_codebook=init, nthreads=NT)
    assert np.array_equal(pq.train_iters.astype(np.int32), iters_o)
    assert np.array_equal(pq.codebook, cbo)


def test_pq_training_seeded_random_init_matches_oracle():
    data = synth.gaussian_mixture(5000, 32, n_components=300, seed=6)
    pq = lb.PQBuildParams(8, 8, max_iters=6, seed=11).build(data)
    cbo, iters_o = ob.pq_train(data, 8, max_iters=6, seed=11, nthreads=NT)
    assert np.array_equal(pq.codebook, cbo)


@pytest.mark.parametrize("d,M", [(128, 16), (64, 16), (32, 32), (96, 8)])
def test_pq_encode_bit_exact(d, M):
    rng = np.random.default_rng(d + M)
    cb = rng.standard_normal((M, 256, d // M)).astype(np.float32)
    vec = rng.standard_normal((1500, d)).astype(np.float32)
    pq = lb.ProductQuantizer(M, 8, d, cb)
    assert np.array_equal(pq.quantize(vec), ob.pq_encode(cb, vec, nthreads=NT))


def test_pq_encode_fused_residual_bit_exact():
    rng = np.random.default_rng(77)
    d, M, K = 128, 16, 50
    cent = rng.standard_normal((K, d)).astype(np.float32)
    cb = (rng.standard_normal((M, 256, d // M)) * 0.5).astype(np.float32)
    vec = rng.standard_normal((2000, d)).astype(np.float32)
    part, _, _ = ob.compute_membership(cent, vec, nthreads=NT)
    res = ob.compute_residual(cent, vec, part, nthreads=NT)
    assert np.array_equal(lb.compute_residual(cent, vec, part), res)
    pq = lb.ProductQuantizer(M, 8, d, cb)
    assert np.array_equal(pq.quantize(vec, centroids=cent, part_ids=part), ob.pq_encode(cb, res, nthreads=NT))
    p2, c2, v2 = lb.ivfpq_transform(cent, cb, vec)
    assert np.array_equal(p2, part) and np.array_equal(c2, ob.pq_encode(cb, res, nthreads=NT)) and v2.all()


def test_lut_and_scan_bit_exact():
    rng = np.random.default_rng(12)
    d, M = 128, 16
    cb = rng.standard_normal((M, 256, d // M)).astype(np.float32)
    q = rng.standard_normal(d).astype(np.float32)
    lut = lb.build_distance_table_l2(cb, 8, M, q)
    assert np.array_equal(lut, ob.build_lut(cb, q))
    codes = rng.integers(0, 256, size=(5000, M), dtype=np.uint8)
    ct = ob.transpose_codes(codes)
    assert np.array_equal(lb.compute_pq_distance(lut, 8, M, ct), ob.pq_scan(lut, ct))
    lut_dot = lb.build_distance_table_l2(cb, 8, M, q, "dot")
    assert np.array_equal(lut_dot, ob.build_lut(cb, q, metric="dot"))
    assert np.array_equal(lb.compute_pq_distance(lut_dot, 8, M, ct, "dot"), ob.pq_scan(lut_dot, ct, metric="dot"))


def test_pq_scan_reference_deterministic_case():
    # lance-index/src/vector/pq/distance.rs:337-365
    nv, M, d = 100, 4, 16
    codebook = np.arange(256 * d, dtype=np.float32).reshape(M, 256, d // M)
    query = np.arange(d, dtype=np.float32)
    lut = lb.build_distance_table_l2(codebook, 8, M, query)
    codes = (np.arange(nv * M) % 256).astype(np.uint8).reshape(nv, M)
    got = lb.compute_pq_distance(lut, 8, M, ob.transpose_codes(codes))
    exp = np.zeros(nv, np.float32)
    for m in range(M):
        exp = (exp + lut[m * 256 + codes[:, m].astype(np.int64)]).astype(np.float32)
    assert np.array_equal(got, exp)


def _check_topk(ids, dists, oi, od, k):
    """the SET of (distance, row id) pairs equals the final content of the reference's BinaryHeap --
    rows tied at the k-th distance included (which of them survive depends on the heap's sift order,
    flat/index.rs:116-126; the product replays that loop whenever such ties overflow the k-th place)."""
    got = sorted(zip(np.asarray(dists).view(np.uint32).tolist(), np.asarray(ids).tolist()))
    exp = sorted(zip(np.asarray(od).view(np.uint32).tolist(), np.asarray(oi).tolist()))
    assert got == exp


def test_flat_topk_matches_heap_semantics():
    rng = np.random.default_rng(13)
    d = rng.integers(0, 50, size=3000).astype(np.float32)  # lots of ties
    rid = rng.permutation(3000).astype(np.uint64)
    for k in (1, 10, 100, 500):
        ids, dist = lb.flat_topk(d, rid, k)
        oi, od = ob.flat_topk(d, rid, k)
        _check_topk(ids, dist, oi, od, k)
    ids, dist = lb.flat_topk(d[:5], rid[:5], 10)
    assert len(ids) == 5


def test_find_partitions_bit_exact():
    rng = np.random.default_rng(14)
    cent = rng.standard_normal((300, 128)).astype(np.float32)
    q = rng.standard_normal((40, 128)).astype(np.float32)
    ids, dists = lb.kmeans_find_partitions(cent, q, 20)
    for i in range(40):
        oi, od = ob.find_partitions(cent, q[i], 20)
        assert np.array_equal(ids[i], oi) and np.array_equal(dists[i], od)


@pytest.mark.parametrize("metric", ["l2", "cosine", "dot"])
def test_index_search_matches_oracle(metric):
    rng = np.random.default_rng(15)
    n, d, K, M = 30000, 64, 40, 16
    data = synth.gaussian_mixture(n, d, n_components=K, seed=15)
    if metric == "dot":
        data /= np.linalg.norm(data, axis=1, keepdims=True)
    ix = lb.IvfPqIndex.build(data, metric, lb.IvfBuildParams(num_partitions=K, num_sub_vectors=M, max_iters=10, pq_max_iters=8))
    parts = ix.export()
    assert parts["part_offsets"][-1] == n and sorted(parts["row_ids"].tolist()) == list(range(n))
    q = synth.gaussian_mixture(50, d, n_components=K, seed=16)
    for k, nprobes in ((10, 1), (10, 8), (100, 5)):
        ids, dists = ix.search(q, k=k, nprobes=nprobes)
        oi, od, oc = ob.ivfpq_search(parts["centroids"], parts["codebook"], parts["part_offsets"],
                                     parts["codes"], parts["row_ids"], q, k, nprobes, metric=metric, nthreads=NT)
        for i in range(len(q)):
            c = int(oc[i])
            assert np.isinf(dists[i, c:]).all()
            _check_topk(ids[i, :c], dists[i, :c], oi[i, :c], od[i, :c], k)
            assert np.all(np.diff(dists[i, :c]) >= 0)
        # the merged output is sorted by (_distance, _rowid) like the reference's SortExec: arrays are equal
        assert np.array_equal(ids, oi) and np.array_equal(dists, od)


# ---- 4-bit PQ (a19): 16 codewords per sub-space, packed codes, u8-quantised table scan -----------
@pytest.mark.parametrize("metric", ["l2", "dot"])
def test_pq_4bit_train_encode_lut_scan_bit_exact(metric):
    rng = np.random.default_rng(404)
    n, d, M = 6000, 64, 16
    data = synth.gaussian_mixture(n, d, n_components=32, seed=404)
    if metric == "dot":
        data /= np.linalg.norm(data, axis=1, keepdims=True)
    init = np.stack([data[rng.choice(n, 16, replace=False)][:, m * 4:(m + 1) * 4] for m in range(M)])
    pq = lb.PQBuildParams(M, 4, max_iters=12, codebook=init).build(data, metric)
    cbo, iters_o = ob.pq_train(data, M, nbits=4, max_iters=12, init_codebook=init, metric=metric, nthreads=NT)
    assert pq.codebook.shape == (M, 16, 4)
    assert np.array_equal(pq.codebook, cbo) and np.array_equal(pq.train_iters.astype(np.int32), iters_o)
    codes = pq.quantize(data)
    assert codes.shape == (n, M // 2)
    assert np.array_equal(codes, ob.pq_encode(cbo, data, nbits=4, metric=metric, nthreads=NT))
    q = data[17] + 0.01
    lut = lb.build_distance_table_l2(pq.codebook, 4, M, q, metric)
    assert np.array_equal(lut, ob.build_lut(cbo, q, nbits=4, metric=metric))
    for rows in (1, 50, 199, 200, 216, 1000, 4099):          # < 200: all flat; n % 16 != 0: exact remainder rows
        ct = np.ascontiguousarray(codes[:rows].T)
        for k_hint in (10, 300):
            got = lb.compute_pq_distance_4bit(lut, M, ct, k_hint, metric)
            want = ob.pq_scan_4bit(lut, ct, rows, k_hint, metric)
            assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (rows, k_hint)
    with pytest.raises(lb.LanceB200Error, match="divisible by 2"):
        lb.ProductQuantizer(3, 4, 12, np.zeros((3, 16, 4), np.float32)).quantize(np.zeros((4, 12), np.float32))


@pytest.mark.parametrize("metric", ["l2", "dot"])
def test_index_4bit_build_search_matches_oracle(metric):
    # create_index(IVF_PQ, num_bits=4): 16 codewords, packed codes, quantised-table scan inside the index
    rng = np.random.default_rng(414)
    n, d, K, M = 20000, 64, 16, 16
    data = synth.gaussian_mixture(n, d, n_components=K, seed=414)
    if metric == "dot":
        data /= np.linalg.norm(data, axis=1, keepdims=True)
    ix = lb.IvfPqIndex.build(data, metric, lb.IvfBuildParams(num_partitions=K, num_sub_vectors=M, num_bits=4,
                                                             max_iters=8, pq_max_iters=6))
    parts = ix.export()
    assert parts["codebook"].shape == (M, 16, d // M) and parts["codes"].shape == (n, M // 2)
    assert ix.info()["num_bits"] == 4
    # the stored codes are the reference's codes for the stored model
    order = np.argsort(parts["row_ids"])
    p_ref, _, _ = ob.compute_membership(parts["centroids"], data, metric=metric, nthreads=NT)
    res = data if metric == "dot" else ob.compute_residual(parts["centroids"], data, p_ref, nthreads=NT)
    # codes are L2 codes whatever the index metric (builder.rs:460: the quantizer is built with DistanceType::L2)
    assert np.array_equal(parts["codes"][order], ob.pq_encode(parts["codebook"], res, nbits=4, metric="l2", nthreads=NT))
    q = synth.gaussian_mixture(16, d, n_components=K, seed=415)
    for k, nprobes in ((10, 3), (250, 2)):                    # k > 200 moves flat_num
        ids, dists = ix.search(q, k=k, nprobes=nprobes)
        oi, od, oc = ob.ivfpq_search(parts["centroids"], parts["codebook"], parts["part_offsets"], parts["codes"],
                                     parts["row_ids"], q, k, nprobes, metric=metric, nbits=4, nthreads=NT)
        for i in range(len(q)):
            c = int(oc[i])
            _check_topk(ids[i, :c], dists[i, :c], oi[i, :c], od[i, :c], k)
    # prefilter: the reference scores the selected rows exactly (DistCalculator::distance)
    allow = parts["row_ids"][rng.choice(n, n // 3, replace=False)]
    bm = ix.row_mask(allow, None)
    ids, dists = ix.search_ex(q, k=10, nprobes=3, allow_bitmap=bm)
    oi, od, oc = ob.ivfpq_search(parts["centroids"], parts["codebook"], parts["part_offsets"], parts["codes"],
                                 parts["row_ids"], q, 10, 3, metric=metric, nbits=4, nthreads=NT, allow=allow)
    for i in range(len(q)):
        c = int(oc[i])
        _check_topk(ids[i, :c], dists[i, :c], oi[i, :c], od[i, :c], 10)
    # from_parts with packed codes == build
    i2 = lb.IvfPqIndex.from_parts(parts["centroids"], parts["codebook"],
                                  np.repeat(np.arange(K, dtype=np.uint32), np.diff(parts["part_offsets"]).astype(np.int64)),
                                  parts["codes"], parts["row_ids"], metric, num_bits=4)
    a, b = ix.search(q, k=10, nprobes=3), i2.search(q, k=10, nprobes=3)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


# ---- prefilter: PreFilter / RowIdMask (prefilter.rs:27-51, flat/index.rs:129-165) --------------
@pytest.mark.parametrize("kind", ["pq", "flat", "pq_pinned_ids"])
def test_index_search_with_row_mask_matches_oracle(kind):
    rng = np.random.default_rng(115)
    n, d, K, M = 24000, 64, 24, 8
    data = synth.gaussian_mixture(n, d, n_components=K, seed=115)
    rid = (rng.permutation(n).astype(np.uint64) * 3 + 7)          # sparse, shuffled row ids
    pin = None
    if kind == "pq_pinned_ids":                                    # the same row ids from pinned host memory
        kind, pin = "pq", lb.PinnedArray(rid.shape, np.uint64)
        pin.array[...] = rid
    if kind == "pq":
        ix = lb.IvfPqIndex.build(data, "l2", lb.IvfBuildParams(num_partitions=K, num_sub_vectors=M, max_iters=8,
                                                               pq_max_iters=6), row_ids=rid if pin is None else pin)
    else:
        ix = lb.IvfFlatIndex.build(data, "l2", num_partitions=K, max_iters=8, row_ids=rid)
    parts = ix.export()
    q = synth.gaussian_mixture(24, d, n_components=K, seed=116)
    allow = rng.choice(rid, n // 3, replace=False)
    block = rng.choice(rid, n // 2, replace=False)
    few = rng.choice(rid, 25, replace=False)                       # fewer allowed rows than k in most probes
    cases = [(allow, None), (None, block), (allow, block), (few, None), (np.zeros(0, np.uint64), None)]
    for a, b in cases:
        bm = ix.row_mask(a, b)
        sel = np.ones(n, bool) if a is None else np.isin(parts["row_ids"], a)
        if b is not None:
            sel &= ~np.isin(parts["row_ids"], b)
        bits = np.unpackbits(bm.view(np.uint8), bitorder="little")[:n].astype(bool)
        assert np.array_equal(bits, sel)                           # lb2_index_row_mask == RowIdMask::selected
        for k, nprobes in ((10, 4), (40, 6)):
            ids, dists = ix.search_ex(q, k=k, nprobes=nprobes, allow_bitmap=bm)
            if kind == "pq":
                oi, od, oc = ob.ivfpq_search(parts["centroids"], parts["codebook"], parts["part_offsets"],
                                             parts["codes"], parts["row_ids"], q, k, nprobes, nthreads=NT,
                                             allow=a, block=b)
            else:
                oi, od, oc = ob.ivfflat_search(parts["centroids"], parts["part_offsets"], parts["vectors"],
                                               parts["row_ids"], q, k, nprobes, nthreads=NT, allow=a, block=b)
            for i in range(len(q)):
                c = int(oc[i])
                assert np.isinf(dists[i, c:]).all() and (ids[i, c:] == np.uint64(2**64 - 1)).all()
                _check_topk(ids[i, :c], dists[i, :c], oi[i, :c], od[i, :c], k)
                assert sel[np.searchsorted(np.sort(parts["row_ids"]), ids[i, :c])].shape[0] == c
                assert np.isin(ids[i, :c], parts["row_ids"][sel]).all()
    # no mask == plain search; mask + refine composes
    i0, d0 = ix.search(q, k=10, nprobes=4)
    i1, d1 = ix.search_ex(q, k=10, nprobes=4)
    assert np.array_equal(i0, i1) and np.array_equal(d0, d1)
    # a NaN query: every distance's order key is the one filtered rows carry.  With the first 5 rows of every
    # partition blocked, the k + 1 smallest (key, position) of a slot (k + 1 > 16: the radix path for IVF_PQ) end in
    # an admitted row, so the slot is replayed through the reference's heap and keeps k admitted rows.
    off = parts["part_offsets"].astype(np.int64)
    b = np.concatenate([parts["row_ids"][o:o + 5] for o in off[:-1]])
    bm = ix.row_mask(None, b)
    qn = q[:1].copy()
    qn[0, 0] = np.nan
    ids, dists = ix.search_ex(qn, k=40, nprobes=6, allow_bitmap=bm)
    if kind == "pq":
        oi, od, oc = ob.ivfpq_search(parts["centroids"], parts["codebook"], parts["part_offsets"], parts["codes"],
                                     parts["row_ids"], qn, 40, 6, nthreads=NT, block=b)
    else:
        oi, od, oc = ob.ivfflat_search(parts["centroids"], parts["part_offsets"], parts["vectors"], parts["row_ids"],
                                       qn, 40, 6, nthreads=NT, block=b)
    assert int(oc[0]) == 40 and np.isnan(od).all()
    assert np.array_equal(ids, oi) and np.isnan(dists).all()


def test_build_transform_equals_oracle_and_recall():
    # v2.rs:1310-1384: IVF_PQ recall floor on random data; here against exact brute force
    n, d, K, M = 50000, 128, 64, 16
    data = synth.sift_like(n, d, n_components=256, seed=21)
    ix = lb.IvfPqIndex.build(data, "l2", lb.IvfBuildParams(num_partitions=K, num_sub_vectors=M))
    parts = ix.export()
    order = np.argsort(parts["row_ids"])
    p_ref, _, _ = ob.compute_membership(parts["centroids"], data, nthreads=NT)
    sizes = np.diff(parts["part_offsets"]).astype(np.int64)
    assert np.array_equal(np.repeat(np.arange(K, dtype=np.uint32), sizes)[order], p_ref)
    res = ob.compute_residual(parts["centroids"], data, p_ref, nthreads=NT)
    assert np.array_equal(parts["codes"][order], ob.pq_encode(parts["codebook"], res, nthreads=NT))
    # rows inside a partition keep input order (stable grouping)
    for p in range(0, K, 7):
        r = parts["row_ids"][parts["part_offsets"][p]:parts["part_offsets"][p + 1]]
        assert np.all(np.diff(r.astype(np.int64)) > 0)
    q = synth.sift_like_queries(100, d, n_components=256, seed=21)
    gt, _ = ob.brute_force_topk(data, q, 10, nthreads=NT)
    ids, _ = ix.search(q, k=10, nprobes=K)
    recall = np.mean([len(set(ids[i].tolist()) & set(gt[i].tolist())) / 10 for i in range(len(q))])
    assert recall >= 0.5, recall  # PQ-only ceiling on SIFT-like data is ~0.6 (BASELINE.md)
    ids100, _ = ix.search(q, k=100, nprobes=K)
    r100 = np.mean([len(set(ids100[i].tolist()) & set(gt[i].tolist())) / 10 for i in range(len(q))])
    assert r100 >= 0.95, r100


def test_device_resident_inputs():
    rng = np.random.default_rng(30)
    cent = rng.standard_normal((64, 128)).astype(np.float32)
    data = rng.standard_normal((4096, 128)).astype(np.float32)
    dd = lb.DeviceArray.from_numpy(data)
    p1, d1, _ = lb.compute_partitions(cent, dd)
    p2, d2, _ = lb.compute_partitions(cent, data)
    assert np.array_equal(p1, p2) and np.array_equal(d1, d2)
    assert np.array_equal(dd.numpy(), data)


def test_unsupported_is_surfaced_not_masked():
    ixs = lb.IvfPqIndex.from_parts(np.zeros((2, 16), np.float32), np.zeros((4, 256, 4), np.float32),
                                   np.zeros(4, np.uint32), np.zeros((4, 4), np.uint8))
    with pytest.raises(lb.LanceB200Error) as e:      # k beyond what the scan kernels select: surfaced
        ixs.search(np.zeros((1, 16), np.float32), k=2000, nprobes=1)
    assert e.value.status == 2
    with pytest.raises(lb.LanceB200Error) as e:      # the reference only has 4 and 8 bits
        lb.PQBuildParams(4, 6).build(np.zeros((300, 16), np.float32))
    assert e.value.status == 1
    with pytest.raises(lb.LanceB200Error):
        lb.train_kmeans(np.zeros((10, 8), np.float32), 8, 20)


def test_edge_cases_empty_ragged_and_error_messages():
    rng = np.random.default_rng(77)
    cent = rng.standard_normal((7, 24)).astype(np.float32)
    # empty batch (transform.rs: empty record batches pass through)
    p, dd, v = lb.compute_partitions(cent, np.zeros((0, 24), np.float32))
    assert p.shape == (0,) and dd.shape == (0,) and v.shape == (0,)
    # one row, K not a multiple of anything, d not a multiple of 16 (sequential tail of l2.rs:69-79)
    x = rng.standard_normal((1, 24)).astype(np.float32)
    p, dd, v = lb.compute_partitions(cent, x)
    po, do, vo = ob.compute_membership(cent, x)
    assert np.array_equal(p, po) and np.array_equal(dd, do)
    # tiny index: more partitions than rows -> empty partitions; k larger than the probed rows
    n, d, K, M = 40, 16, 8, 4
    data = rng.standard_normal((n, d)).astype(np.float32)
    cb = rng.standard_normal((M, 256, d // M)).astype(np.float32)
    cents = data[:K].copy()
    part, codes = lb.ivfpq_transform(cents, cb, data)[:2]
    part = np.where(part == 3, 2, part).astype(np.uint32)      # partition 3 is empty
    ix = lb.IvfPqIndex.from_parts(cents, cb, part, codes)
    parts = ix.export()
    assert parts["part_offsets"][4] == parts["part_offsets"][3]
    q = rng.standard_normal((5, d)).astype(np.float32)
    for k, nprobes in ((10, 1), (64, 8), (1, 3)):
        ids, dists = ix.search(q, k=k, nprobes=nprobes)
        oi, od, oc = ob.ivfpq_search(parts["centroids"], parts["codebook"], parts["part_offsets"], parts["codes"],
                                     parts["row_ids"], q, k, nprobes)
        for i in range(len(q)):
            c = int(oc[i])
            assert np.isinf(dists[i, c:]).all()
            _check_topk(ids[i, :c], dists[i, :c], oi[i, :c], od[i, :c], k)
    ids, dists = ix.search(np.zeros((0, d), np.float32), k=5, nprobes=2)   # empty query batch
    assert ids.shape == (0, 5)
    # the reference's error texts (kmeans.rs:1014-1022, pq/builder.rs:96-110) come back through lb2_last_error
    with pytest.raises(lb.LanceB200Error, match="can not train 20 centroids with 10 vectors") as e:
        lb.train_kmeans(np.zeros((10, 8), np.float32), 8, 20)
    assert e.value.status == 1
    with pytest.raises(lb.LanceB200Error, match="num_sub_vectors must divide vector dimension"):
        lb.PQBuildParams(5, 8).build(np.zeros((300, 16), np.float32))
    with pytest.raises(lb.LanceB200Error, match="nprobes"):
        lb.kmeans_find_partitions(cent, x, 8)


def test_concurrent_host_threads_share_an_index():
    """SURVEY 8b threading: every symbol is re-entrant, each calling thread gets its own stream; the
    reference searches partitions from many spawn_cpu threads at once (knn.rs:881, v2.rs:483)."""
    import threading
    n, d, K, M = 30000, 64, 32, 8
    data = synth.gaussian_mixture(n, d, n_components=K, seed=501)
    ix = lb.IvfPqIndex.build(data, "l2", lb.IvfBuildParams(num_partitions=K, num_sub_vectors=M, max_iters=6, pq_max_iters=4))
    cent = ix.export()["centroids"]
    qs = [synth.gaussian_mixture(200, d, n_components=K, seed=600 + t) for t in range(6)]
    want = [(ix.search(q, k=10, nprobes=4), lb.compute_partitions(cent, q)) for q in qs]
    got, errs = [None] * len(qs), []

    def work(t):
        try:
            for _ in range(5):
                got[t] = (ix.search(qs[t], k=10, nprobes=4), lb.compute_partitions(cent, qs[t]))
        except Exception as e:  # noqa: BLE001 - reported below
            errs.append(e)

    th = [threading.Thread(target=work, args=(t,)) for t in range(len(qs))]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errs, errs
    for (s1, p1), (s2, p2) in zip(want, got):
        assert np.array_equal(s1[0], s2[0]) and np.array_equal(s1[1], s2[1])
        assert all(np.array_equal(a, b) for a, b in zip(p1, p2))


# ---- tensor-core filter path (wgmma) must be bit-identical to the exact path -----------------
def _both_paths(fn):
    import os
    os.environ.pop("LB2_DISABLE_TC", None)
    a = fn()
    os.environ["LB2_DISABLE_TC"] = "1"
    try:
        b = fn()
    finally:
        os.environ.pop("LB2_DISABLE_TC", None)
    return a, b


@pytest.mark.parametrize("n,d,k", [(256, 128, 256), (1000, 128, 256), (5000, 128, 100), (4097, 64, 256),
                                   (3000, 96, 33), (129, 32, 2), (20000, 128, 255)])
def test_tc_filter_equals_exact_path(n, d, k):
    rng = np.random.default_rng(n * 7 + d + k)
    cent = (rng.standard_normal((k, d)) * 3).astype(np.float32)
    data = (cent[rng.integers(0, k, n)] + rng.standard_normal((n, d))).astype(np.float32)
    (p1, d1, v1), (p2, d2, v2) = _both_paths(lambda: lb.compute_partitions(cent, data))
    assert np.array_equal(p1, p2) and np.array_equal(d1, d2) and np.array_equal(v1, v2)
    po, do, vo = ob.compute_membership(cent, data, nthreads=NT)
    assert np.array_equal(p1, po) and np.array_equal(d1, do)


@pytest.mark.parametrize("n,d,k", [(3000, 768, 300), (2000, 768, 1000), (5000, 64, 1000), (2500, 128, 4096),
                                   (700, 256, 256), (1500, 1536, 64), (4000, 160, 513), (300, 32, 257)])
def test_tc_filter_general_shapes_equal_exact_path(n, d, k):
    # d > 128 and/or K > 256: centroid tiles streamed through the TMA ring, running top-3 across tiles
    rng = np.random.default_rng(n * 3 + d + k)
    cent = (rng.standard_normal((k, d)) * 3).astype(np.float32)
    cent[k - 1] = cent[0]       # duplicate in the LAST centroid tile: index 0 must win
    data = (cent[rng.integers(0, k, n)] + rng.standard_normal((n, d))).astype(np.float32)
    data[7] = np.nan
    data[11] = ((cent[1] + cent[k - 2]) * 0.5).astype(np.float32)   # half-way across tiles
    (p1, d1, v1), (p2, d2, v2) = _both_paths(lambda: lb.compute_partitions(cent, data))
    assert np.array_equal(v1, v2) and not v1[7]
    assert np.array_equal(p1[v1], p2[v2]) and np.array_equal(d1[v1], d2[v2])
    po, do, vo = ob.compute_membership(cent, data, nthreads=NT)
    assert np.array_equal(p1[v1], po[vo]) and np.array_equal(d1[v1], do[vo])


def test_tc_filter_general_training_with_balance_bias():
    # direct Lloyd at K > 256 (hierarchical off): the bias/balance term goes through the streamed path
    data = synth.sift_like(40000, 64, seed=77)
    init = data[np.random.default_rng(5).choice(40000, 320, replace=False)].copy()
    (k1, k2) = _both_paths(lambda: lb.train_kmeans(data, 64, 320, max_iters=6, centroids=init,
                                                   balance_factor=1.0))
    assert k1.iters == k2.iters and k1.loss == k2.loss and np.array_equal(k1.centroids, k2.centroids)


def test_tc_filter_adversarial_near_ties():
    # centroids in tight groups (differences far below the TF32 resolution), exact duplicates, and
    # rows exactly half-way between two centroids: every row must still match the exact path
    rng = np.random.default_rng(99)
    d, k, n = 128, 256, 6000
    base = (rng.standard_normal((32, d)) * 50).astype(np.float32)
    cent = np.repeat(base, 8, axis=0)
    cent += (rng.standard_normal((k, d)) * 1e-3).astype(np.float32)
    cent[17] = cent[16]          # exact duplicate
    cent[40:44] = cent[40]       # 4 identical -> top-3 all tied -> exact fallback
    data = (cent[rng.integers(0, k, n)] + rng.standard_normal((n, d)) * 0.5).astype(np.float32)
    data[:100] = ((cent[0] + cent[9]) * 0.5).astype(np.float32)
    data[100] = np.nan
    data[101, 5] = np.inf
    (p1, d1, v1), (p2, d2, v2) = _both_paths(lambda: lb.compute_partitions(cent, data))
    assert np.array_equal(v1, v2) and not v1[100] and not v1[101]
    assert np.array_equal(p1[v1], p2[v2]) and np.array_equal(d1[v1], d2[v2])
    po, do, vo = ob.compute_membership(cent, data, nthreads=NT)
    assert np.array_equal(p1[v1], po[vo]) and np.array_equal(d1[v1], do[vo])


def _tight_groups(rng, k, d, dtype=np.float32):
    """centroids in groups of 8 that differ by ~1e-3 (far below the TF32 / accumulate resolution), duplicates"""
    base = (rng.standard_normal((k // 8, d)) * 20).astype(np.float32)
    cent = np.repeat(base, 8, axis=0) + (rng.standard_normal((k, d)) * 1e-3).astype(np.float32)
    cent = cent.astype(dtype).astype(np.float32)
    cent[17] = cent[16]
    cent[40:44] = cent[40]
    cent[k - 40:k - 20] = cent[k - 40]      # 20 identical: more candidates than slots -> full exact scan
    return cent


@pytest.mark.parametrize("n,d,k", [(5000, 128, 256), (6000, 96, 600), (3000, 768, 1024)])
def test_tc_candidate_pass_matches_oracle(n, d, k, monkeypatch):
    # LB2_FORCE_REFINE: the 3xTF32 top-3 pass + candidate pass + exact decision among candidates run even
    # on small inputs (production takes them when n * K >= 2^26); every row must still match the oracle
    monkeypatch.setenv("LB2_FORCE_REFINE", "1")
    rng = np.random.default_rng(n + k)
    cent = _tight_groups(rng, k, d)
    data = (cent[rng.integers(0, k, n)] + rng.standard_normal((n, d)) * 0.3).astype(np.float32)
    data[:64] = ((cent[0] + cent[9]) * 0.5).astype(np.float32)
    data[64:96] = cent[k - 30]               # exactly on the 20-fold duplicate
    data[100] = np.nan
    data[101, 5] = np.inf
    p1, d1, v1 = lb.compute_partitions(cent, data)
    po, do, vo = ob.compute_membership(cent, data, nthreads=NT)
    assert np.array_equal(v1, vo) and not v1[100] and not v1[101]
    assert np.array_equal(p1[v1], po[vo]) and np.array_equal(d1[v1], do[vo])
    # balance bias goes through the same passes
    km = lb.train_kmeans(data[:2000], d, 16, max_iters=3, balance_factor=1.0, seed=3)
    monkeypatch.delenv("LB2_FORCE_REFINE")
    km2 = lb.train_kmeans(data[:2000], d, 16, max_iters=3, balance_factor=1.0, seed=3)
    assert np.array_equal(km.centroids, km2.centroids)


@pytest.mark.parametrize("dtype", ["f16", "bf16"])
@pytest.mark.parametrize("n,d,k", [(5000, 128, 512), (3000, 1536, 304)])
def test_native_16bit_operands_match_oracle(dtype, n, d, k, monkeypatch):
    # f16 / bf16 rows (the model has the same element type, so it is exact in it): the tensor-core passes read the
    # native rows (f16 / bf16 wgmma).  Results must equal the oracle on the converted values -- with and without the
    # candidate pass -- and the f32-staged path (LB2_NO_NATIVE16).
    rng = np.random.default_rng(n + d + len(dtype))
    if dtype == "f16":
        to_t = lambda a: a.astype(np.float16)
        to_f = lambda t: t.astype(np.float32)
    else:
        to_t = lambda a: (np.ascontiguousarray(a, np.float32).view(np.uint32) >> 16).astype(np.uint16)
        to_f = lambda t: (t.astype(np.uint32) << 16).view(np.float32)
    cent_t = to_t(_tight_groups(rng, k, d) * np.float32(0.05 if dtype == "f16" else 1.0))
    cent = to_f(cent_t)
    data = (cent[rng.integers(0, k, n)] + rng.standard_normal((n, d)) * 0.3).astype(np.float32)
    data[:64] = ((cent[0] + cent[9]) * 0.5).astype(np.float32)
    data[64:96] = cent[k - 30]
    data[100] = np.nan
    data_t = to_t(data)
    data32 = to_f(data_t)
    po, do, vo = ob.compute_membership(cent, data32, nthreads=NT)
    run = lambda: lb.compute_partitions(cent_t, data_t, bf16=(dtype == "bf16"))
    for force in ("", "1"):
        monkeypatch.setenv("LB2_FORCE_REFINE", force)
        p1, d1, v1 = run()
        assert np.array_equal(v1, vo) and not v1[100]
        assert np.array_equal(p1[v1], po[vo]) and np.array_equal(d1[v1], do[vo])
    lb.profile.enable(True)
    lb.profile.reset()
    run()
    lb.profile.enable(False)
    assert lb.profile.get("tc_filter_general16")[0] == 1 and lb.profile.get("tc_candidates")[0] == 1
    monkeypatch.setenv("LB2_NO_NATIVE16", "1")
    p2, d2, v2 = run()
    assert np.array_equal(p1[v1], p2[v2]) and np.array_equal(d1[v1], d2[v2])


def test_tc_filter_sift_shaped_and_training():
    data = synth.sift_like(70000, 128, seed=31)
    init = data[np.random.default_rng(2).choice(70000, 256, replace=False)].copy()
    (k1, k2) = _both_paths(lambda: lb.train_kmeans(data, 128, 256, max_iters=12, centroids=init, balance_factor=1.0))
    assert k1.iters == k2.iters and k1.loss == k2.loss and np.array_equal(k1.centroids, k2.centroids)
    nn = 65536
    co, loss_o, it_o = ob.kmeans_train(data[:nn], 256, max_iters=12, init_centroids=init,
                                       balance_factor=float(np.float32(1.0) / np.float32(nn)), nthreads=NT)
    assert k1.iters == it_o and np.array_equal(k1.centroids, co) and k1.loss == loss_o


@pytest.mark.parametrize("n,d,M", [(1500, 128, 16), (4097, 64, 8), (300, 32, 4), (20000, 128, 16),
                                   (3000, 768, 96), (1000, 256, 32), (700, 1536, 192), (40000, 160, 20)])
def test_tc_pq_encode_equals_exact_path(n, d, M):
    rng = np.random.default_rng(n + d)
    cb = (rng.standard_normal((M, 256, 8)) * 2).astype(np.float32)
    cb[0, 7] = cb[0, 3]            # duplicate codeword: index 3 must win
    cb[1, 100:104] = cb[1, 100]    # 4-way tie -> exact fallback
    vec = (rng.standard_normal((n, d)) * 2).astype(np.float32)
    vec[5, :8] = cb[0, 3]          # exactly on a duplicated codeword
    pq = lb.ProductQuantizer(M, 8, d, cb)
    c1, c2 = _both_paths(lambda: pq.quantize(vec))
    assert np.array_equal(c1, c2)
    assert np.array_equal(c1, ob.pq_encode(cb, vec, nthreads=NT))
    assert c1[5, 0] == 3


def test_tc_pq_fused_residual_and_training_equal_exact_path():
    rng = np.random.default_rng(123)
    n, d, M, K = 30000, 128, 16, 64
    data = synth.sift_like(n, d, seed=9)
    cent = data[rng.choice(n, K, replace=False)].copy()
    cb0 = (rng.standard_normal((M, 256, 8)) * 20).astype(np.float32)
    (a1, a2) = _both_paths(lambda: lb.ivfpq_transform(cent, cb0, data))
    assert np.array_equal(a1[0], a2[0]) and np.array_equal(a1[1], a2[1])
    part, _, _ = ob.compute_membership(cent, data, nthreads=NT)
    res = ob.compute_residual(cent, data, part, nthreads=NT)
    assert np.array_equal(a1[1], ob.pq_encode(cb0, res, nthreads=NT))
    init = np.stack([res[rng.choice(n, 256, replace=False)][:, m * 8:(m + 1) * 8] for m in range(M)])
    (p1, p2) = _both_paths(lambda: lb.PQBuildParams(M, 8, max_iters=10, codebook=init).build(res))
    assert np.array_equal(p1.train_iters, p2.train_iters) and np.array_equal(p1.codebook, p2.codebook)
    cbo, iters_o = ob.pq_train(res, M, max_iters=10, init_codebook=init, nthreads=NT)
    assert np.array_equal(p1.codebook, cbo) and np.array_equal(p1.train_iters.astype(np.int32), iters_o)


def test_tc_pq_streamed_codebook_training_equals_exact_path():
    # M > 16: codebook chunks are streamed; sub-spaces converge at different iterations (active flags)
    rng = np.random.default_rng(321)
    n, d, M = 20000, 384, 48
    res = (rng.standard_normal((n, d)) * np.linspace(0.5, 4.0, d)).astype(np.float32)
    res[:, :8] = np.round(res[:, :8])          # a coarse sub-space: converges early, many exact ties
    init = np.stack([res[rng.choice(n, 256, replace=False)][:, m * 8:(m + 1) * 8] for m in range(M)])
    (p1, p2) = _both_paths(lambda: lb.PQBuildParams(M, 8, max_iters=8, codebook=init).build(res))
    assert np.array_equal(p1.train_iters, p2.train_iters) and np.array_equal(p1.codebook, p2.codebook)
    cbo, iters_o = ob.pq_train(res, M, max_iters=8, init_codebook=init, nthreads=NT)
    assert np.array_equal(p1.codebook, cbo) and np.array_equal(p1.train_iters.astype(np.int32), iters_o)


# ---- IVF_FLAT (flat/index.rs, flat/storage.rs; recall floor 1.0 in v2.rs:1310-1332) ------------
@pytest.mark.parametrize("metric", ["l2", "dot", "cosine"])
def test_ivf_flat_matches_oracle_and_full_probe_recall_is_one(metric):
    n, d, K = 20000, 64, 32
    data = synth.gaussian_mixture(n, d, n_components=K, seed=41)
    if metric == "dot":
        data /= np.linalg.norm(data, axis=1, keepdims=True)
    ix = lb.IvfFlatIndex.build(data, metric, num_partitions=K, max_iters=10)
    parts = ix.export()
    assert parts["part_offsets"][-1] == n and sorted(parts["row_ids"].tolist()) == list(range(n))
    stored = ob.normalize_rows(data, nthreads=NT) if metric == "cosine" else data
    assert np.array_equal(parts["vectors"], stored[parts["row_ids"].astype(np.int64)])
    q = synth.gaussian_mixture(40, d, n_components=K, seed=42)
    for k, nprobes in ((10, 1), (10, 5), (64, 3)):
        ids, dists = ix.search(q, k=k, nprobes=nprobes)
        oi, od, oc = ob.ivfflat_search(parts["centroids"], parts["part_offsets"], parts["vectors"],
                                       parts["row_ids"], q, k, nprobes, metric=metric, nthreads=NT)
        qn = ob.normalize_rows(q, nthreads=NT)
        off = parts["part_offsets"].astype(np.int64)
        for i in range(len(q)):
            c = int(oc[i])
            if metric == "cosine":
                # FMA lanes + shuffle tree, not the reference's scalar order: every distance within
                # B = 3 (ceil(d/16) + 4) 2^-24 S + 2^-24 of its f64 value (S = sum|q y| / |q||y|, derived in
                # tests/test_exact_search_variants.py::_cosine_bound), the ids the f64 top-k up to rows within 2B
                # of the k-th, ascending by (distance, id)
                def f64(r):
                    y, x = stored[r].astype(np.float64), qn[i].astype(np.float64)
                    nrm = np.linalg.norm(x) * np.linalg.norm(y, axis=-1)
                    return 1.0 - (y @ x) / nrm, 3.0 * (-(-d // 16) + 4) * 2.0 ** -24 * np.abs(y * x).sum(-1) / nrm + 2.0 ** -24
                got = ids[i, :c].astype(np.int64)
                ex, bnd = f64(got)
                assert np.all(np.abs(dists[i, :c] - ex) <= bnd), i
                assert all((dists[i, j], got[j]) < (dists[i, j + 1], got[j + 1]) for j in range(c - 1)), i
                pids, _ = ob.find_partitions(parts["centroids"], qn[i], nprobes)
                cand = np.concatenate([parts["row_ids"][off[p]:off[p + 1]] for p in pids]).astype(np.int64)
                all_ex, all_b = f64(cand)
                kth, b2 = np.sort(all_ex)[c - 1], 2 * all_b.max()
                assert set(cand[all_ex < kth - b2].tolist()) <= set(got.tolist()) and np.all(ex <= kth + b2), i
            else:
                _check_topk(ids[i, :c], dists[i, :c], oi[i, :c], od[i, :c], k)
    gt, _ = ob.brute_force_topk(stored if metric == "cosine" else data, q if metric != "cosine" else ob.normalize_rows(q), 10,
                                metric="l2" if metric == "cosine" else metric, nthreads=NT)
    ids, _ = ix.search(q, k=10, nprobes=K)
    recall = np.mean([len(set(ids[i].tolist()) & set(gt[i].tolist())) / 10 for i in range(len(q))])
    assert recall >= 0.999, recall


# ---- element types: f16 / u8 buffers are converted to f32 on the device, then f32 semantics -----
def test_f16_and_u8_inputs_equal_f32_path_on_converted_values():
    rng = np.random.default_rng(77)
    n, d, K = 5000, 128, 64
    x8 = rng.integers(0, 256, size=(n, d), dtype=np.uint8)
    cent = x8[:K].astype(np.float32) + 0.25
    p8, d8, _ = lb.compute_partitions(cent, x8)
    pf, df, _ = lb.compute_partitions(cent, x8.astype(np.float32))
    assert np.array_equal(p8, pf) and np.array_equal(d8, df)
    x16 = (rng.standard_normal((n, d)) * 4).astype(np.float16)
    c16 = x16[:K].copy()
    p16, d16, _ = lb.compute_partitions(c16, x16)
    pr, dr, _ = lb.compute_partitions(c16.astype(np.float32), x16.astype(np.float32))
    assert np.array_equal(p16, pr) and np.array_equal(d16, dr)
    # the oracle's f16 scalar path (convert each element to f32, 16 lanes: l2.rs:100-106,156)
    for i in range(0, 50, 7):
        assert d16[i] == np.float32(ob.l2_f16(x16[i], c16[p16[i]]))
    # trained model comes back in the input's element type
    km = lb.train_kmeans(x16, d, 16, max_iters=4, centroids=c16[:16])
    assert km.centroids.dtype == np.float16
    kf = lb.train_kmeans(x16.astype(np.float32), d, 16, max_iters=4, centroids=c16[:16].astype(np.float32))
    assert np.array_equal(km.centroids, kf.centroids.astype(np.float16))
    # whole index from u8 vectors == index from the same values as f32
    i8 = lb.IvfPqIndex.build(x8, "l2", lb.IvfBuildParams(num_partitions=16, num_sub_vectors=16, max_iters=5, pq_max_iters=4))
    i32 = lb.IvfPqIndex.build(x8.astype(np.float32), "l2", lb.IvfBuildParams(num_partitions=16, num_sub_vectors=16, max_iters=5, pq_max_iters=4))
    e8, e32 = i8.export(), i32.export()
    assert np.array_equal(e8["codes"], e32["codes"]) and np.array_equal(e8["part_offsets"], e32["part_offsets"])
    r8 = i8.search(x8[:20], k=5, nprobes=4)
    r32 = i32.search(x8[:20].astype(np.float32), k=5, nprobes=4)
    assert np.array_equal(r8[0], r32[0]) and np.array_equal(r8[1], r32[1])


# ---- full-size (BASELINE config 1: 1M x 128, IVF_PQ 256/16) size-independent properties ----------
def test_full_size_sift1m_properties():
    import ctypes as C
    n, d, K, M = 1_000_000, 128, 256, 16
    pin = lb.PinnedArray((n, d), np.float32)
    rng = np.random.default_rng(5)
    W, cm = synth.sift_model(d)
    for s in range(0, n, 1 << 16):  # generate in place (host allocations are slow on these VMs)
        e = min(n, s + (1 << 16))
        z = cm[rng.integers(0, cm.shape[0], e - s)] + rng.standard_normal((e - s, 24), dtype=np.float32)
        x = np.maximum(z @ W * 12.0 + 20.0, 0.0) + rng.standard_normal((e - s, d), dtype=np.float32) * 3.0
        pin.array[s:e] = np.clip(np.rint(x), 0, 255)
    data = pin.array
    ix = lb.IvfPqIndex.build(pin, "l2", lb.IvfBuildParams(num_partitions=K, num_sub_vectors=M, seed=3))
    parts = ix.export()
    off, rid, codes = parts["part_offsets"].astype(np.int64), parts["row_ids"].astype(np.int64), parts["codes"]
    # every row exactly once; rows inside a partition in input order; offsets monotone
    assert off[0] == 0 and off[-1] == n and np.all(np.diff(off) >= 0)
    assert np.array_equal(np.sort(rid), np.arange(n))
    part_of_pos = np.repeat(np.arange(K), np.diff(off))
    same = part_of_pos[1:] == part_of_pos[:-1]
    assert np.all(np.diff(rid)[same] > 0)
    # idempotence: re-assigning with the trained model reproduces the stored partition of every row,
    # and re-encoding reproduces every code (tensor-core path == stored result of the same path)
    p2, c2, v2 = lb.ivfpq_transform(parts["centroids"], parts["codebook"], data[:200000])
    part_of_row = np.empty(n, np.int64)
    part_of_row[rid] = part_of_pos
    code_of_row = np.empty((n, M), np.uint8)
    code_of_row[rid] = codes
    assert np.array_equal(p2, part_of_row[:200000]) and np.array_equal(c2, code_of_row[:200000]) and v2.all()
    # a sample of rows against the oracle (exactness at full size)
    sel = rng.choice(n, 4000, replace=False)
    po, _, _ = ob.compute_membership(parts["centroids"], data[sel], nthreads=NT)
    assert np.array_equal(po, part_of_row[sel])
    res = ob.compute_residual(parts["centroids"], data[sel], po, nthreads=NT)
    assert np.array_equal(ob.pq_encode(parts["codebook"], res, nthreads=NT), code_of_row[sel])
    # reconstruction: decode(code) + centroid is closer to the row than the bare centroid (PQ helps)
    recon = parts["centroids"][po] + np.concatenate([parts["codebook"][m][code_of_row[sel][:, m]] for m in range(M)], axis=1)
    assert ((data[sel] - recon) ** 2).sum(1).mean() < 0.6 * ((data[sel] - parts["centroids"][po]) ** 2).sum(1).mean()
    # search: distances ascending, ids unique, counts full, and equal to the oracle on a few queries
    q = data[rng.choice(n, 64, replace=False)] + rng.integers(-2, 3, size=(64, d)).astype(np.float32)
    ids, dd = ix.search(q, k=10, nprobes=16)
    assert np.all(np.diff(dd, axis=1) >= 0) and all(len(set(r.tolist())) == 10 for r in ids)
    oi, od, _ = ob.ivfpq_search(parts["centroids"], parts["codebook"], parts["part_offsets"], codes,
                                parts["row_ids"], q[:8], 10, 16, nthreads=NT)
    assert np.array_equal(np.sort(dd[:8], axis=1), np.sort(od, axis=1))
    pin.free()


def test_search_with_refine_matches_exact_rerank_of_oracle_candidates():
    n, d, K, M = 40000, 128, 32, 16
    data = synth.sift_like(n, d, seed=61)
    q = synth.sift_like_queries(60, d, seed=61)
    ix = lb.IvfPqIndex.build(data, "l2", lb.IvfBuildParams(num_partitions=K, num_sub_vectors=M, max_iters=10, pq_max_iters=8))
    parts = ix.export()
    k, nprobes, rf = 10, 8, 10
    ids, dists = ix.search_refine(data, q, k=k, nprobes=nprobes, refine_factor=rf)
    oi, od, oc = ob.ivfpq_search(parts["centroids"], parts["codebook"], parts["part_offsets"], parts["codes"],
                                 parts["row_ids"], q, k * rf, nprobes, nthreads=NT)
    for i in range(len(q)):
        cand = oi[i, :oc[i]].astype(np.int64)
        ex = np.array([ob.l2(q[i], data[c]) for c in cand], np.float32)
        order = np.lexsort((cand, ex))[:k]
        assert np.array_equal(dists[i], ex[order]) and np.array_equal(ids[i].astype(np.int64), cand[order]), i
    gt, _ = ob.brute_force_topk(data, q, 10, nthreads=NT)
    recall = np.mean([len(set(ids[i].tolist()) & set(gt[i].tolist())) / 10 for i in range(len(q))])
    plain, _ = ix.search(q, k=10, nprobes=nprobes)
    r0 = np.mean([len(set(plain[i].tolist()) & set(gt[i].tolist())) / 10 for i in range(len(q))])
    assert recall > r0 + 0.1 and recall >= 0.85, (recall, r0)


def test_hierarchical_kmeans_for_k_above_256_matches_oracle():
    # kmeans.rs:1511-1537 (k = 257 produces K finite centroids) + bit parity with the restated scheme
    n, d, k = 30000, 32, 300
    data = synth.gaussian_mixture(n, d, n_components=400, seed=71)
    km = lb.train_kmeans(data, d, k, max_iters=10, seed=9, balance_factor=1.0)
    assert km.centroids.shape == (k, d) and np.isfinite(km.centroids).all()
    co, got = ob.hierarchical_kmeans(data, k, max_iters=10, seed=9,
                                     balance_factor=float(np.float32(1.0) / np.float32(n)), nthreads=NT)
    assert got == k
    assert np.array_equal(km.centroids, co)
    # sanity of the scheme itself: within ~20 % of a flat Lloyd run of the same budget (the ratio depends on the
    # seed: 1.14 .. 1.21 over seeds 1, 2, 3, 9, 11 on this data)
    _, d_h, _ = ob.compute_membership(km.centroids, data, nthreads=NT)
    flat, _, _ = ob.kmeans_train(data, k, max_iters=10, seed=9, nthreads=NT)
    _, d_f, _ = ob.compute_membership(flat, data, nthreads=NT)
    assert d_h.sum() <= 1.3 * d_f.sum()


# ---- scaled-down shapes of the other BASELINE.json configs (parity cases, not bench lines) ------
def test_config2_shape_768d_k300_m96():
    # C2: 768-d f32, K > 256 (hierarchical training), M = 96 (8-wide sub-vectors, 98 KB LUT)
    n, d, K, M = 12000, 768, 300, 96
    data = synth.gaussian_mixture(n, d, n_components=64, seed=81)
    ix = lb.IvfPqIndex.build(data, "l2", lb.IvfBuildParams(num_partitions=K, num_sub_vectors=M, max_iters=4, pq_max_iters=3))
    parts = ix.export()
    order = np.argsort(parts["row_ids"])
    p_ref, _, _ = ob.compute_membership(parts["centroids"], data, nthreads=NT)
    sizes = np.diff(parts["part_offsets"]).astype(np.int64)
    assert np.array_equal(np.repeat(np.arange(K, dtype=np.uint32), sizes)[order], p_ref)
    res = ob.compute_residual(parts["centroids"], data, p_ref, nthreads=NT)
    assert np.array_equal(parts["codes"][order], ob.pq_encode(parts["codebook"], res, nthreads=NT))
    q = synth.gaussian_mixture(10, d, n_components=64, seed=82)
    ids, dists = ix.search(q, k=10, nprobes=6)
    oi, od, oc = ob.ivfpq_search(parts["centroids"], parts["codebook"], parts["part_offsets"], parts["codes"],
                                 parts["row_ids"], q, 10, 6, nthreads=NT)
    for i in range(len(q)):
        _check_topk(ids[i, :oc[i]], dists[i, :oc[i]], oi[i, :oc[i]], od[i, :oc[i]], 10)


def _bf16_to_f32(bits):
    return (np.asarray(bits, np.uint16).astype(np.uint32) << 16).view(np.float32)


def test_config3_shape_f16_cosine():
    # C3: f16 vectors, cosine (normalise, then L2).  The model of an f16 column is f16-valued like the reference's
    # (kmeans.rs:405-418 keeps centroids in T); given that model every integer output equals the oracle's on the
    # converted values, and the search equals the oracle's search
    n, d, K, M = 20000, 128, 64, 16
    data16 = (synth.gaussian_mixture(n, d, n_components=K, seed=83) * 0.25).astype(np.float16)
    p = lb.IvfBuildParams(num_partitions=K, num_sub_vectors=M, max_iters=6, pq_max_iters=4)
    i16 = lb.IvfPqIndex.build(data16, "cosine", p)
    e16 = i16.export()
    for name in ("centroids", "codebook"):
        assert np.array_equal(e16[name], e16[name].astype(np.float16).astype(np.float32)), name
    unit = ob.normalize_rows(data16.astype(np.float32), nthreads=NT)
    order = np.argsort(e16["row_ids"])
    p_ref, _, _ = ob.compute_membership(e16["centroids"], unit, nthreads=NT)
    sizes = np.diff(e16["part_offsets"]).astype(np.int64)
    assert np.array_equal(np.repeat(np.arange(K, dtype=np.uint32), sizes)[order], p_ref)
    res = ob.compute_residual(e16["centroids"], unit, p_ref, nthreads=NT)
    assert np.array_equal(e16["codes"][order], ob.pq_encode(e16["codebook"], res, nthreads=NT))
    q16 = data16[:30]
    r16 = i16.search(q16, k=10, nprobes=5)
    # (cosine index = L2 on unit vectors, _distance = squared L2 of unit vectors)
    oi, od, oc = ob.ivfpq_search(e16["centroids"], e16["codebook"], e16["part_offsets"], e16["codes"],
                                 e16["row_ids"], q16.astype(np.float32), 10, 5, metric="cosine", nthreads=NT)
    assert np.array_equal(r16[0], oi) and np.array_equal(r16[1], od)


def test_f16_normalize_and_centroid_update_vs_reference_f16_arithmetic():
    """The reference normalises and sums centroids IN THE ELEMENT TYPE (kernels.rs:141-146: norm = sqrt of a
    sequential f16 sum, x / norm in f16; kmeans.rs:405-418: centroid += row in f16, * 1/cnt in f16).  We compute
    in f32 and round once.  This bounds the distance between the two: the f16 loops below restate the reference
    (numpy float16, one rounding per operation); the tolerance is what f16 accumulation itself loses."""
    rng = np.random.default_rng(90)
    d, n = 128, 64
    x = (rng.standard_normal((n, d)) * 0.5).astype(np.float16)
    ours = lb.normalize_fsl(x.astype(np.float32))                   # f32 arithmetic on the converted values
    ref = np.empty((n, d), np.float16)
    for r in range(n):
        s = np.float16(0)
        for i in range(d):
            s = np.float16(s + np.float16(x[r, i] * x[r, i]))
        ref[r] = (x[r] / np.sqrt(s, dtype=np.float16)).astype(np.float16)
    # a 128-term f16 sum carries up to ~sqrt(128) * 2^-11 relative error (0.6 %), worst case 128 * 2^-11 (6 %)
    assert np.max(np.abs(ours - ref.astype(np.float32))) <= 0.02 * np.max(np.abs(ours))
    assert np.mean(np.abs(ours - ref.astype(np.float32))) <= 0.003 * np.max(np.abs(ours))
    # one centroid update: 200 members summed in f16 vs our f32 sum rounded to f16
    members = (rng.standard_normal((200, d)) * 0.5 + 1.0).astype(np.float16)
    km = lb.train_kmeans(members, d, 1, max_iters=1, centroids=members[:1])
    acc = np.zeros(d, np.float16)
    for r in range(200):
        acc = (acc + members[r]).astype(np.float16)
    ref_c = (acc * np.float16(1.0 / 200)).astype(np.float16)
    rel = np.abs(km.centroids[0].astype(np.float32) - ref_c.astype(np.float32)) / np.maximum(np.abs(ref_c.astype(np.float32)), 1e-3)
    assert km.centroids.dtype == np.float16 and np.max(rel) <= 0.05, np.max(rel)   # f16 sums near 200 have 0.125 ulps


def test_config4_shape_bf16_ivf_flat_1536d():
    # C4: 1536-d bf16 column, IVF_FLAT (no PQ): coarse assignment through the streamed tensor-core filter, exact
    # partition scan over vectors STORED AS bf16; bf16 -> f32 is exact, so with the (bf16-valued) model the index
    # equals the oracle's on the converted values
    n, d, K = 6000, 1536, 48
    f = synth.gaussian_mixture(n, d, n_components=K, seed=87).astype(np.float32)
    bits = (f.view(np.uint32) >> 16).astype(np.uint16)               # truncate to bf16
    f = _bf16_to_f32(bits)                                           # the exact f32 value of every element
    ib = lb.IvfFlatIndex.build(bits, "l2", num_partitions=K, max_iters=6, bf16=True)
    eb = ib.export()
    assert eb["vectors"].dtype == np.uint16 and eb["vectors"].shape == (n, d)
    order = np.argsort(eb["row_ids"])
    assert np.array_equal(eb["vectors"][order], bits)                # the rows themselves, regrouped
    cb = eb["centroids"]
    assert np.array_equal(cb, _bf16_to_f32((cb.view(np.uint32) >> 16).astype(np.uint16)))   # bf16-valued model
    p_ref, _, _ = ob.compute_membership(cb, f, nthreads=NT)
    sizes = np.diff(eb["part_offsets"]).astype(np.int64)
    assert np.array_equal(np.repeat(np.arange(K, dtype=np.uint32), sizes)[order], p_ref)
    q = f[:20]
    ids, dists = ib.search(bits[:20], k=10, nprobes=4)
    oi, od, oc = ob.ivfflat_search(cb, eb["part_offsets"], _bf16_to_f32(eb["vectors"]), eb["row_ids"], q, 10, 4, nthreads=NT)
    assert np.array_equal(ids, oi) and np.array_equal(dists, od)
    # an f16 column keeps f16 storage
    h = (f[:2000, :64] * 0.1).astype(np.float16)
    ih = lb.IvfFlatIndex.build(h, "cosine", num_partitions=8, max_iters=4)
    eh = ih.export()
    assert eh["vectors"].dtype == np.float16
    unit = ob.normalize_rows(h.astype(np.float32), nthreads=NT).astype(np.float16)   # normalised, then stored in T
    assert np.array_equal(eh["vectors"][np.argsort(eh["row_ids"])], unit)


def test_config5_shape_u8_m32():
    # C5: u8 vectors, M = 32 (4-wide sub-vectors -> exact small-d kernel), many partitions
    rng = np.random.default_rng(85)
    n, d, K, M = 30000, 128, 200, 32
    data8 = np.clip(synth.sift_like(n, d, seed=85), 0, 255).astype(np.uint8)
    ix = lb.IvfPqIndex.build(data8, "l2", lb.IvfBuildParams(num_partitions=K, num_sub_vectors=M, max_iters=6, pq_max_iters=4))
    parts = ix.export()
    f = data8.astype(np.float32)
    order = np.argsort(parts["row_ids"])
    p_ref, _, _ = ob.compute_membership(parts["centroids"], f, nthreads=NT)
    sizes = np.diff(parts["part_offsets"]).astype(np.int64)
    assert np.array_equal(np.repeat(np.arange(K, dtype=np.uint32), sizes)[order], p_ref)
    res = ob.compute_residual(parts["centroids"], f, p_ref, nthreads=NT)
    assert np.array_equal(parts["codes"][order], ob.pq_encode(parts["codebook"], res, nthreads=NT))
    ids, dists = ix.search(data8[:16], k=10, nprobes=8)
    oi, od, oc = ob.ivfpq_search(parts["centroids"], parts["codebook"], parts["part_offsets"], parts["codes"],
                                 parts["row_ids"], f[:16], 10, 8, nthreads=NT)
    for i in range(16):
        _check_topk(ids[i, :oc[i]], dists[i, :oc[i]], oi[i, :oc[i]], od[i, :oc[i]], 10)


# ---- round 2: parity loose ends -----------------------------------------------------------------------
def test_flat_topk_ties_and_range_equal_reference_heap():
    rng = np.random.default_rng(2001)
    for n in (5000, 12003):                                       # 12003: three 4096-row chunks, ties across them
        d = rng.integers(0, 12, size=n).astype(np.float32)         # at most 12 distinct values: ties everywhere
        rid = rng.permutation(n).astype(np.uint64)
        for k in (1, 2, 7, 15, 16, 17, 100, 127, 128, 500, 1024):
            ids, dist = lb.flat_topk(d, rid, k)
            oi, od = ob.flat_topk(d, rid, k)
            _check_topk(ids, dist, oi, od, k)
            assert np.all(np.diff(dist) >= 0)
        for lo, hi in ((2.0, 7.0), (None, 3.0), (5.0, None), (3.0, 3.0), (11.0, 100.0)):
            for k in (5, 40):
                ids, dist = lb.flat_topk(d, rid, k, lower_bound=lo, upper_bound=hi)
                oi, od = ob.flat_topk(d, rid, k, lower=lo, upper=hi)
                _check_topk(ids, dist, oi, od, k)
    x = np.array([np.inf, -np.inf, 1.0, 2.0], np.float32)          # an absent bound is f32::MIN / f32::MAX
    assert lb.flat_topk(x, None, 4, upper_bound=5.0)[1].tolist() == [1.0, 2.0]
    assert lb.flat_topk(x, None, 4, lower_bound=-5.0)[1].tolist() == [1.0, 2.0]


@pytest.mark.parametrize("kind", ["pq", "flat", "pq4"])
def test_index_search_boundary_ties_equal_reference_heap(kind):
    """Duplicate rows -> identical codes / distances -> ties at the k-th place inside a partition: the
    survivors must be the ones the reference's BinaryHeap keeps (flat/index.rs:116-126)."""
    rng = np.random.default_rng(2002)
    distinct, d, K, M = 220, 32, 6, 8
    base = synth.gaussian_mixture(distinct, d, n_components=K, seed=2002)
    n = 9000
    data = base[rng.integers(0, distinct, n)]                       # every vector ~40 times
    q = base[rng.integers(0, distinct, 40)] + 0.01
    if kind == "flat":
        ix = lb.IvfFlatIndex.build(data, "l2", num_partitions=K, max_iters=6)
    else:
        ix = lb.IvfPqIndex.build(data, "l2", lb.IvfBuildParams(num_partitions=K, num_sub_vectors=M, max_iters=6, pq_max_iters=5,
                                                               num_bits=4 if kind == "pq4" else 8))
    parts = ix.export()
    for k, nprobes in ((1, 1), (5, 2), (10, 3), (15, 6), (16, 2), (60, 3), (300, 6)):
        ids, dists = ix.search(q, k=k, nprobes=nprobes)
        if kind == "flat":
            oi, od, oc = ob.ivfflat_search(parts["centroids"], parts["part_offsets"], parts["vectors"],
                                           parts["row_ids"], q, k, nprobes, nthreads=NT)
        else:
            oi, od, oc = ob.ivfpq_search(parts["centroids"], parts["codebook"], parts["part_offsets"], parts["codes"],
                                         parts["row_ids"], q, k, nprobes, nbits=4 if kind == "pq4" else 8, nthreads=NT)
        assert np.array_equal(ids, oi) and np.array_equal(dists, od), (kind, k, nprobes)
    # ... and under a prefilter
    allow = rng.choice(parts["row_ids"], n // 2, replace=False)
    bm = ix.row_mask(allow, None)
    ids, dists = ix.search_ex(q, k=10, nprobes=3, allow_bitmap=bm)
    if kind == "flat":
        oi, od, oc = ob.ivfflat_search(parts["centroids"], parts["part_offsets"], parts["vectors"], parts["row_ids"], q, 10, 3,
                                       nthreads=NT, allow=allow)
    else:
        oi, od, oc = ob.ivfpq_search(parts["centroids"], parts["codebook"], parts["part_offsets"], parts["codes"],
                                     parts["row_ids"], q, 10, 3, nbits=4 if kind == "pq4" else 8, nthreads=NT, allow=allow)
    assert np.array_equal(ids, oi) and np.array_equal(dists, od)


@pytest.mark.parametrize("kind", ["pq", "flat"])
def test_index_search_range_query_matches_oracle(kind):
    rng = np.random.default_rng(2003)
    n, d, K, M = 20000, 64, 16, 8
    data = synth.gaussian_mixture(n, d, n_components=K, seed=2003)
    q = synth.gaussian_mixture(30, d, n_components=K, seed=2004)
    if kind == "pq":
        ix = lb.IvfPqIndex.build(data, "l2", lb.IvfBuildParams(num_partitions=K, num_sub_vectors=M, max_iters=8, pq_max_iters=6))
    else:
        ix = lb.IvfFlatIndex.build(data, "l2", num_partitions=K, max_iters=8)
    parts = ix.export()
    i0, d0 = ix.search(q, k=50, nprobes=4)
    lo, hi = float(np.median(d0[:, 5])), float(np.median(d0[:, 30]))
    allow = rng.choice(parts["row_ids"], n // 2, replace=False)
    bm = ix.row_mask(allow, None)
    for lower, upper, a in ((lo, hi, None), (None, hi, None), (lo, None, None), (lo, hi, allow), (hi, lo, None)):
        for k in (10, 40):
            ids, dists = ix.search_ex(q, k=k, nprobes=4, lower_bound=lower, upper_bound=upper,
                                      allow_bitmap=None if a is None else bm)
            if kind == "pq":
                oi, od, oc = ob.ivfpq_search(parts["centroids"], parts["codebook"], parts["part_offsets"], parts["codes"],
                                             parts["row_ids"], q, k, 4, nthreads=NT, allow=a, lower=lower, upper=upper)
            else:
                oi, od, oc = ob.ivfflat_search(parts["centroids"], parts["part_offsets"], parts["vectors"], parts["row_ids"],
                                               q, k, 4, nthreads=NT, allow=a, lower=lower, upper=upper)
            assert np.array_equal(ids, oi) and np.array_equal(dists, od), (kind, lower, upper, k)
            fin = np.isfinite(dists)
            if lower is not None:
                assert np.all(dists[fin] >= lower)
            if upper is not None:
                assert np.all(dists[fin] < upper)
    if kind == "pq":  # with refine the plan filters the EXACT distances afterwards (scanner.rs:3342-3377)
        k, rf = 10, 5
        ids, dists = ix.search_ex(q, k=k, nprobes=4, refine_factor=rf, vectors=data, lower_bound=lo, upper_bound=hi)
        oi, od, oc = ob.ivfpq_search(parts["centroids"], parts["codebook"], parts["part_offsets"], parts["codes"],
                                     parts["row_ids"], q, k * rf, 4, nthreads=NT, lower=lo, upper=hi)
        for i in range(len(q)):
            cand = oi[i, :oc[i]].astype(np.int64)
            ex = np.array([ob.l2(q[i], data[c]) for c in cand], np.float32)
            keep = (ex >= np.float32(lo)) & (ex < np.float32(hi))
            cand, ex = cand[keep], ex[keep]
            order = np.lexsort((cand, ex))[:k]
            c = len(order)
            assert np.array_equal(dists[i, :c], ex[order]) and np.array_equal(ids[i, :c].astype(np.int64), cand[order])
            assert np.isinf(dists[i, c:]).all()


@pytest.mark.parametrize("metric", ["l2", "cosine"])
def test_builds_drop_non_finite_rows_like_keep_finite_vectors(metric):
    """transform.rs:112-159 (KeepFiniteVectors) and builder.rs:436 (is_finite filter on the sample): NaN / Inf
    rows -- and zero vectors under cosine, which normalise to NaN -- never enter the index or the training."""
    rng = np.random.default_rng(2005)
    n, d, K, M = 6000, 32, 8, 8
    data = synth.gaussian_mixture(n, d, n_components=K, seed=2005)
    bad = np.sort(rng.choice(n, 40, replace=False))
    data[bad[:15], 3] = np.nan
    data[bad[15:30], 7] = np.inf
    if metric == "cosine":
        data[bad[30:]] = 0.0
        dropped = set(bad.tolist())
    else:
        data[bad[30:], 0] = -np.inf
        dropped = set(bad.tolist())
    q = synth.gaussian_mixture(20, d, n_components=K, seed=2006)
    # sample_rate large enough that the training sample is the whole dataset (bad rows included)
    ix = lb.IvfPqIndex.build(data, metric, lb.IvfBuildParams(num_partitions=K, num_sub_vectors=M, max_iters=6, pq_max_iters=5,
                                                            sample_rate=n))
    info, parts = ix.info(), ix.export()
    assert info["num_rows"] == n - len(dropped) == int(parts["part_offsets"][-1])
    assert dropped.isdisjoint(parts["row_ids"].tolist())
    assert np.isfinite(parts["centroids"]).all() and np.isfinite(parts["codebook"]).all()
    ids, dists = ix.search(q, k=20, nprobes=K)
    assert dropped.isdisjoint(ids.ravel().tolist()) and np.isfinite(dists).all()
    fx = lb.IvfFlatIndex.build(data, metric, num_partitions=K, max_iters=6, sample_rate=n)
    fparts = fx.export()
    assert fx.info()["num_rows"] == n - len(dropped) and dropped.isdisjoint(fparts["row_ids"].tolist())
    assert np.isfinite(fparts["vectors"]).all() and np.isfinite(fparts["centroids"]).all()
    ids, dists = fx.search(q, k=20, nprobes=K)
    assert dropped.isdisjoint(ids.ravel().tolist()) and np.isfinite(dists).all()
    # rows the index holds are exactly the oracle's kept rows with the oracle's partition ids
    src = ob.normalize_rows(data) if metric == "cosine" else data
    keep = np.isfinite(src).all(axis=1)
    assert np.array_equal(np.sort(fparts["row_ids"]), np.flatnonzero(keep).astype(np.uint64))
    p_ref, _, _ = ob.compute_membership(fparts["centroids"], src[keep], nthreads=NT)
    order = np.argsort(fparts["row_ids"])
    sizes = np.diff(fparts["part_offsets"]).astype(np.int64)
    assert np.array_equal(np.repeat(np.arange(K, dtype=np.uint32), sizes)[order], p_ref)


def test_part_ids_out_of_range_are_rejected():
    rng = np.random.default_rng(2007)
    d, K, M, n = 16, 4, 4, 50
    cent = rng.standard_normal((K, d)).astype(np.float32)
    cb = rng.standard_normal((M, 256, d // M)).astype(np.float32)
    data = rng.standard_normal((n, d)).astype(np.float32)
    part = rng.integers(0, K, n).astype(np.uint32)
    codes = rng.integers(0, 256, (n, M)).astype(np.uint8)
    bad = part.copy()
    bad[17] = K
    with pytest.raises(lb.LanceB200Error, match="out of range") as e:
        lb.IvfPqIndex.from_parts(cent, cb, bad, codes)
    assert e.value.status == 1
    with pytest.raises(lb.LanceB200Error, match="out of range"):
        lb.IvfFlatIndex.from_parts(cent, bad, data)
    with pytest.raises(lb.LanceB200Error, match="out of range"):
        lb.compute_residual(cent, data, bad)
    with pytest.raises(lb.LanceB200Error, match="out of range"):
        lb.ProductQuantizer(M, 8, d, cb).quantize(data, centroids=cent, part_ids=bad)
    lb.IvfPqIndex.from_parts(cent, cb, part, codes)                 # in range: fine


def test_kmeans_redos_semantics():
    """kmeans.rs:643-716: every redo restarts from rng.clone() -> identical runs without a balance bias (PQ);
    with a bias redos > 1 is not implemented and says so."""
    data = synth.gaussian_mixture(3000, 16, n_components=8, seed=2008)
    a = lb.train_kmeans(data, 16, 8, max_iters=10, redos=1, seed=5)
    b = lb.train_kmeans(data, 16, 8, max_iters=10, redos=3, seed=5)
    assert np.array_equal(a.centroids, b.centroids) and a.loss == b.loss
    with pytest.raises(lb.LanceB200Error) as e:
        lb.train_kmeans(data, 16, 8, max_iters=10, redos=2, balance_factor=1.0, seed=5)
    assert e.value.status == 2
    p1 = lb.PQBuildParams(4, 8, max_iters=6, kmeans_redos=1, seed=3).build(data)
    p2 = lb.PQBuildParams(4, 8, max_iters=6, kmeans_redos=4, seed=3).build(data)
    assert np.array_equal(p1.codebook, p2.codebook)


@pytest.mark.parametrize("d", [3, 8, 32, 100, 768])
def test_normalize_fsl_bit_exact(d):
    rng = np.random.default_rng(2009 + d)
    x = rng.standard_normal((257, d)).astype(np.float32)
    x[5] = 0.0                                                     # 0 / 0 -> NaN like the reference
    got, exp = lb.normalize_fsl(x), ob.normalize_rows(x)
    assert np.array_equal(got.view(np.uint32)[np.isfinite(exp)], exp.view(np.uint32)[np.isfinite(exp)])
    assert np.isnan(got[5]).all() and np.isnan(exp[5]).all()


def test_reference_fixture_pq_in_schema_on_gpu():
    """The reference's own index fixture (tests/golden/pq_in_schema.npz, see make_pq_in_schema_fixture.py): the device
    reproduces the codes Lance 0.27.1 stored, consumes the stored transposed bytes, and searches like the oracle."""
    import os
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", "pq_in_schema.npz"))
    M, n = int(z["num_sub_vectors"]), len(z["row_ids"])
    codes = z["codes_transposed"].reshape(M, n).T.copy()
    v = z["vectors"][z["row_ids"].astype(np.int64)]
    part, pcodes, valid = lb.ivfpq_transform(z["centroids"], z["codebook"], v)
    assert valid.all() and (part == 0).all() and np.array_equal(pcodes, codes)
    assert np.array_equal(lb.ProductQuantizer(M, 8, 32, z["codebook"]).quantize(v, centroids=z["centroids"], part_ids=part), codes)
    q = np.zeros((1, 32), np.float32)
    lut = lb.build_distance_table_l2(z["codebook"], 8, M, q[0] - z["centroids"][0])
    assert np.array_equal(lut, ob.build_lut(z["codebook"], q[0] - z["centroids"][0]))
    d_t = lb.compute_pq_distance(lut, 8, M, z["codes_transposed"])
    assert np.array_equal(d_t, ob.pq_scan(lut, z["codes_transposed"].reshape(M, n)))
    ix = lb.IvfPqIndex.from_parts(z["centroids"], z["codebook"], part, codes, row_ids=z["row_ids"])
    ids, dd = ix.search(q, k=5, nprobes=1)
    oi, od, oc = ob.ivfpq_search(z["centroids"], z["codebook"], np.array([0, n], np.uint64), codes, z["row_ids"], q, 5, 1)
    assert oc[0] == 5 and np.array_equal(ids, oi) and np.array_equal(dd, od)
    # the partition goes back out in the reference's storage layout: the bytes of the `__pq_code` column
    ct, rid = ix.export_partition_transposed(0)
    assert np.array_equal(ct.reshape(-1), z["codes_transposed"]) and np.array_equal(rid, z["row_ids"])


# ---- the conflict-free ("skewed") scan kernel: same bits as the classic kernel and the oracle ----------------
def _with_scan(mode, fn):
    """mode: classic | skew (two teams of 8 warps, two LUT copies) | skew4 (four teams of 4 warps, one copy)"""
    import os
    old = {k: os.environ.get(k) for k in ("LB2_SCAN", "LB2_SCAN_TEAMS")}
    os.environ["LB2_SCAN"] = "classic" if mode == "classic" else "skew"
    os.environ["LB2_SCAN_TEAMS"] = "4" if mode == "skew4" else "2"
    try:
        return fn()
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


@pytest.mark.parametrize("metric", ["l2", "cosine", "dot"])
def test_skew_scan_kernel_matches_oracle_and_classic(metric):
    """ivfpq_scan_skew_kernel (8-bit, 16 sub-spaces x 8 dims): partitions that are empty, shorter than a warp,
    shorter than a slab, several chunks long; k = 1 .. 15; plain, prefiltered and range searches."""
    rng = np.random.default_rng(3101)
    d, M = 128, 16
    sizes = [0, 1, 17, 31, 32, 33, 500, 512, 513, 1000, 4095, 4096, 4097, 9000, 0, 700]
    K = len(sizes)
    cent = (rng.standard_normal((K, d)) * 4).astype(np.float32)
    part = np.repeat(np.arange(K, dtype=np.uint32), sizes)
    n = len(part)
    data = (cent[part] + rng.standard_normal((n, d))).astype(np.float32)
    if metric == "dot":
        data /= np.linalg.norm(data, axis=1, keepdims=True)
        cent /= np.linalg.norm(cent, axis=1, keepdims=True)
    perm = rng.permutation(n)
    data, part = data[perm], part[perm]
    res = data - cent[part]
    pq = lb.PQBuildParams(M, 8, max_iters=4, seed=5).build(res[rng.choice(n, 8000, replace=False)])
    codes = pq.quantize(res)
    rid = (rng.permutation(n).astype(np.uint64) * 5 + 3)
    ix = lb.IvfPqIndex.from_parts(cent, pq.codebook, part, codes, rid, metric)
    parts = ix.export()
    q = (cent[rng.integers(0, K, 48)] + rng.standard_normal((48, d))).astype(np.float32)
    allow = rng.choice(rid, n // 3, replace=False)
    bm = ix.row_mask(allow, None)
    lb.profile.reset()
    lb.profile.enable(True)
    for k, nprobes in ((1, 3), (10, K), (15, 7), (5, 1), (100, 6), (135, K), (40, 2)):   # k > 15: the radix slot
        oi, od, oc = ob.ivfpq_search(parts["centroids"], parts["codebook"], parts["part_offsets"], parts["codes"],
                                     parts["row_ids"], q, k, nprobes, metric=metric, nthreads=NT)
        for mode in ("skew", "skew4", "classic"):
            ids, dists = _with_scan(mode, lambda: ix.search(q, k=k, nprobes=nprobes))
            assert np.array_equal(ids, oi) and np.array_equal(dists, od), (mode, k, nprobes)
        oi, od, oc = ob.ivfpq_search(parts["centroids"], parts["codebook"], parts["part_offsets"], parts["codes"],
                                     parts["row_ids"], q, k, nprobes, metric=metric, nthreads=NT, allow=allow)
        for mode in ("skew", "skew4"):
            ids, dists = _with_scan(mode, lambda: ix.search_ex(q, k=k, nprobes=nprobes, allow_bitmap=bm))
            assert np.array_equal(ids, oi) and np.array_equal(dists, od), (mode + "+mask", k, nprobes)
    i0, d0 = ix.search(q, k=15, nprobes=K)
    lo, hi = float(np.median(d0[:, 2])), float(np.median(d0[:, 12]))
    oi, od, oc = ob.ivfpq_search(parts["centroids"], parts["codebook"], parts["part_offsets"], parts["codes"],
                                 parts["row_ids"], q, 10, K, metric=metric, nthreads=NT, lower=lo, upper=hi)
    for mode in ("skew", "skew4"):
        ids, dists = _with_scan(mode, lambda: ix.search_ex(q, k=10, nprobes=K, lower_bound=lo, upper_bound=hi))
        assert np.array_equal(ids, oi) and np.array_equal(dists, od), mode
    lb.profile.enable(False)
    prof = lb.profile.dump()
    assert prof.get("search:pq_scan_skew", (0, 0))[0] >= 18 and prof.get("search:pq_scan", (0, 0))[0] >= 4, prof


def test_skew_scan_kernel_ties_and_non_finite_lut_go_to_the_replay():
    """duplicated rows tie at the k-th place (reference heap order decides); a query with an Inf component makes
    the LUT non-finite, which the skewed kernel must hand to the exact replay instead of poisoning its sums."""
    rng = np.random.default_rng(3102)
    d, M, K, distinct, n = 128, 16, 5, 150, 7000
    base = (rng.integers(0, 6, (distinct, d))).astype(np.float32)
    data = base[rng.integers(0, distinct, n)]
    ix = lb.IvfPqIndex.build(data, "l2", lb.IvfBuildParams(num_partitions=K, num_sub_vectors=M, max_iters=5, pq_max_iters=4))
    parts = ix.export()
    q = base[rng.integers(0, distinct, 64)] + np.float32(0.25)
    q[3, 7] = np.inf
    q[9, 100] = 3.0e38
    for k, nprobes in ((1, 1), (7, 3), (15, 5), (60, 4), (120, 2)):
        oi, od, oc = ob.ivfpq_search(parts["centroids"], parts["codebook"], parts["part_offsets"], parts["codes"],
                                     parts["row_ids"], q, k, nprobes, nthreads=NT)
        for mode in ("skew", "skew4", "classic"):
            ids, dists = _with_scan(mode, lambda: ix.search(q, k=k, nprobes=nprobes))
            assert np.array_equal(ids, oi), (mode, k, nprobes)
            assert np.array_equal(dists, od, equal_nan=True), (mode, k, nprobes)


# ---- stream / async variants of the boundary (SURVEY 8b "Threading") ------------------------------------------
def test_search_async_and_set_stream_equal_blocking_calls():
    """lb2_index_search_async only enqueues: several searches on two caller-owned streams, results read after the
    streams finish, equal the blocking lb2_index_search results; lb2_set_stream routes blocking calls to a caller
    stream (same results) and NULL restores the private stream."""
    import torch  # CUDA stream / event handles only
    from lance_b200._lib import DeviceArray, PinnedArray
    rng = np.random.default_rng(3201)
    n, d, K, M = 40000, 128, 32, 16
    data = synth.sift_like(n, d, n_components=64, seed=3201)
    ix = lb.IvfPqIndex.build(data, "l2", lb.IvfBuildParams(num_partitions=K, num_sub_vectors=M, max_iters=6, pq_max_iters=5))
    batches = [synth.sift_like_queries(nq, d, n_components=64, seed=3300 + i) for i, nq in enumerate((400, 7, 256, 64))]
    want = [ix.search(q, k=10, nprobes=6) for q in batches]
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    ev = torch.cuda.Event()
    ev.record()                                                       # torch creates the cudaEvent_t lazily
    qs, outs = [], []
    for i, q in enumerate(batches):                                   # device buffers and pinned host buffers
        qd = DeviceArray.from_numpy(q)
        if i % 2 == 0:
            o = (DeviceArray((len(q), 10), np.uint64), DeviceArray((len(q), 10), np.float32))
        else:
            o = (PinnedArray((len(q), 10), np.uint64), PinnedArray((len(q), 10), np.float32))
        qs.append(qd)
        outs.append(o)
        ix.search_async(qd, o, k=10, nprobes=6, cuda_stream=streams[i % 2].cuda_stream,
                        done_event=ev.cuda_event if i == len(batches) - 1 else None)
    ev.synchronize()
    for s in streams:
        s.synchronize()
    for (wi, wd), o in zip(want, outs):
        gi = o[0].numpy() if isinstance(o[0], DeviceArray) else o[0].array
        gd = o[1].numpy() if isinstance(o[1], DeviceArray) else o[1].array
        assert np.array_equal(gi, wi) and np.array_equal(gd, wd)
    lb.set_stream(streams[0].cuda_stream)
    try:
        gi, gd = ix.search(batches[0], k=10, nprobes=6)
        p, dd, v = lb.compute_partitions(ix.export()["centroids"], data[:5000])
    finally:
        lb.set_stream(None)
    assert np.array_equal(gi, want[0][0]) and np.array_equal(gd, want[0][1])
    p2, dd2, v2 = lb.compute_partitions(ix.export()["centroids"], data[:5000])
    assert np.array_equal(p, p2) and np.array_equal(dd, dd2)


def test_index_repartition_without_communicator_is_a_copy():
    """lb2_index_repartition on one rank owns every partition: same storage, same search (the N-rank exchange is
    checked by tools/nccl_check.py under torchrun)."""
    for kind in ("pq", "flat"):
        data = synth.gaussian_mixture(12000, 128 if kind == "pq" else 32, n_components=20, seed=3301)
        if kind == "pq":
            ix = lb.IvfPqIndex.build(data, "l2", lb.IvfBuildParams(num_partitions=20, num_sub_vectors=16, max_iters=5, pq_max_iters=4))
        else:
            ix = lb.IvfFlatIndex.build(data, "l2", num_partitions=20, max_iters=5)
        own = ix.repartition()
        a, b = ix.export(), own.export()
        for key in a:
            assert np.array_equal(a[key], b[key]), (kind, key)
        q = data[:40] + np.float32(0.1)
        for mode in ("skew", "classic"):
            r0 = _with_scan(mode, lambda: ix.search(q, k=10, nprobes=5))
            r1 = _with_scan(mode, lambda: own.search(q, k=10, nprobes=5))
            assert np.array_equal(r0[0], r1[0]) and np.array_equal(r0[1], r1[1])


# ---- incremental update: the data path of optimize / split / join (builder.rs:1152-1650) ----------------------
def test_index_update_append_remove_and_remap_equal_a_fresh_load():
    rng = np.random.default_rng(3401)
    n, d, K, M = 30000, 128, 24, 16
    data = synth.gaussian_mixture(n, d, n_components=K, seed=3401)
    ix = lb.IvfPqIndex.build(data[:20000], "l2", lb.IvfBuildParams(num_partitions=K, num_sub_vectors=M, max_iters=6, pq_max_iters=5),
                             row_ids=np.arange(20000, dtype=np.uint64) * 2)
    parts = ix.export()
    sizes = np.diff(parts["part_offsets"]).astype(np.int64)
    old_part = np.repeat(np.arange(K, dtype=np.uint32), sizes)
    # (1) append (optimize without retraining): new rows are transformed with the index's model and merged
    add_p, add_c, _ = lb.ivfpq_transform(parts["centroids"], parts["codebook"], data[20000:])
    add_r = np.arange(20000, n, dtype=np.uint64) * 2
    up = ix.update(add_part_ids=add_p, add_codes=add_c, add_row_ids=add_r)
    want = lb.IvfPqIndex.from_parts(parts["centroids"], parts["codebook"], np.concatenate([old_part, add_p]),
                                    np.concatenate([parts["codes"], add_c]), np.concatenate([parts["row_ids"], add_r]))
    a, b = up.export(), want.export()
    for key in a:
        assert np.array_equal(a[key], b[key]), ("append", key)
    # (2) remove row ids (AssignOp::Remove / deletions) + drop partition 3 entirely + shift the later ids down (join)
    removed = rng.choice(parts["row_ids"], 3000, replace=False)
    pm = np.arange(K, dtype=np.uint32)
    pm[3] = 0xFFFFFFFF
    pm[4:] -= 1
    cent2 = np.delete(parts["centroids"], 3, axis=0)
    keep = ~np.isin(parts["row_ids"], removed) & (old_part != 3)
    moved = np.flatnonzero(old_part == 3)                             # the joined partition's rows re-enter via the add list
    mp = rng.integers(0, K - 1, len(moved)).astype(np.uint32)
    up2 = ix.update(new_centroids=cent2, part_map=pm, remove_row_ids=removed, add_part_ids=mp,
                    add_codes=parts["codes"][moved], add_row_ids=parts["row_ids"][moved] + np.uint64(1))
    want2 = lb.IvfPqIndex.from_parts(cent2, parts["codebook"], np.concatenate([pm[old_part[keep]], mp]),
                                     np.concatenate([parts["codes"][keep], parts["codes"][moved]]),
                                     np.concatenate([parts["row_ids"][keep], parts["row_ids"][moved] + np.uint64(1)]))
    a, b = up2.export(), want2.export()
    assert up2.info()["num_partitions"] == K - 1
    for key in a:
        assert np.array_equal(a[key], b[key]), ("join", key)
    q = data[:64] + np.float32(0.05)
    r0, r1 = up2.search(q, k=10, nprobes=6), want2.search(q, k=10, nprobes=6)
    assert np.array_equal(r0[0], r1[0]) and np.array_equal(r0[1], r1[1])
    with pytest.raises(lb.LanceB200Error):                             # a map beyond the new partition count is rejected
        ix.update(part_map=np.full(K, K + 5, np.uint32))


def test_split_partition_flow_on_device_primitives():
    """split_partition_impl (builder.rs:1219-1333) on the device primitives: k-means with k = 2 on the partition's raw
    vectors, distances to the old and the two new centroids, the reference's assign rule, then lb2_index_update.  The
    result must equal an index loaded from the same decisions computed with the oracle's distances."""
    n, d, K, M = 24000, 128, 12, 16
    data = synth.gaussian_mixture(n, d, n_components=K + 1, seed=3402)
    ix = lb.IvfPqIndex.build(data, "l2", lb.IvfBuildParams(num_partitions=K, num_sub_vectors=M, max_iters=8, pq_max_iters=5))
    parts = ix.export()
    sizes = np.diff(parts["part_offsets"]).astype(np.int64)
    ps = int(np.argmax(sizes))                                          # should_split picks the largest partition
    lo, hi = int(parts["part_offsets"][ps]), int(parts["part_offsets"][ps + 1])
    rows = parts["row_ids"][lo:hi].astype(np.int64)
    vec = data[rows]
    km = lb.train_kmeans(vec, d, 2, max_iters=50, seed=3)
    c0, c1, c2 = parts["centroids"][ps], km.centroids[0], km.centroids[1]
    d0, d1, d2 = (lb.l2_distance_batch(c, vec, d) for c in (c0, c1, c2))
    assert all(np.array_equal(g, ob.l2_batch(c, vec, d)) for g, c in ((d0, c0), (d1, c1), (d2, c2)))
    # rows of the split partition: the closer of the two new centroids (no reassign candidates in this test)
    to2 = ~(d1 <= d2)
    newc = np.concatenate([parts["centroids"], c2[None]], 0)
    newc[ps] = c1
    npart = np.where(to2, K, ps).astype(np.uint32)
    codes = lb.ProductQuantizer(M, 8, d, parts["codebook"]).quantize(vec, centroids=newc, part_ids=npart)
    pm = np.arange(K, dtype=np.uint32)
    pm[ps] = 0xFFFFFFFF
    up = ix.update(new_centroids=newc, part_map=pm, add_part_ids=npart, add_codes=codes, add_row_ids=rows.astype(np.uint64))
    old_part = np.repeat(np.arange(K, dtype=np.uint32), sizes)
    keep = old_part != ps
    res = vec - newc[npart]
    want = lb.IvfPqIndex.from_parts(newc, parts["codebook"], np.concatenate([old_part[keep], npart]),
                                    np.concatenate([parts["codes"][keep], ob.pq_encode(parts["codebook"], res, nthreads=NT)]),
                                    np.concatenate([parts["row_ids"][keep], rows.astype(np.uint64)]))
    a, b = up.export(), want.export()
    assert up.info()["num_partitions"] == K + 1 and up.info()["num_rows"] == n
    for key in a:
        assert np.array_equal(a[key], b[key]), key


# ---- the bulk-copy staging cache (staging.cuh StagingCache): repeated host-sourced builds reuse one landing buffer --
def test_host_sourced_builds_reuse_staging_buffer_and_equal_device_builds():
    n, d, K, M = 30000, 64, 16, 8
    prm = lb.IvfBuildParams(num_partitions=K, num_sub_vectors=M, max_iters=6, pq_max_iters=5, seed=11)
    pin = lb.PinnedArray((n, d), np.float32)
    exports = []
    for rep, (rows, seed) in enumerate(((n, 1), (n, 2), (n // 2, 3), (n, 4))):  # same, same size, smaller, larger again
        x = synth.sift_like(rows, d, seed=seed)
        pin.array[:rows] = x
        src = pin if rows == n else np.ascontiguousarray(pin.array[:rows])   # pinned (zero-copy gathers) and pageable
        e_host = lb.IvfPqIndex.build(src, "l2", prm).export()
        e_dev = lb.IvfPqIndex.build(lb.DeviceArray.from_numpy(x), "l2", prm).export()
        for key in ("centroids", "codebook", "part_offsets", "codes", "row_ids"):
            assert np.array_equal(e_host[key], e_dev[key]), (rep, key)
        exports.append(e_host["codes"])
    assert not np.array_equal(exports[0], exports[1])  # the second build did read its own rows, not stale ones
    # rows that are not finite: the PQ sample gathered on the copy stream reports them and the build falls back
    # to the synchronous gather that drops them (builder.rs:436) -- same index as from device-resident rows
    x = synth.sift_like(n, d, seed=9)
    x[::7, 3] = np.nan
    x[5::11, 0] = np.inf
    pin.array[:] = x
    e_host = lb.IvfPqIndex.build(pin, "l2", prm).export()
    e_dev = lb.IvfPqIndex.build(lb.DeviceArray.from_numpy(x), "l2", prm).export()
    for key in ("centroids", "codebook", "part_offsets", "codes", "row_ids"):
        assert np.array_equal(e_host[key], e_dev[key]), ("non-finite", key)
    bad = np.flatnonzero(~np.isfinite(x).all(1))
    assert len(e_host["row_ids"]) == n - len(bad) and not np.isin(bad, e_host["row_ids"]).any()
    pin.array[:] = synth.sift_like(n, d, seed=4)
    e_host = lb.IvfPqIndex.build(pin, "l2", prm).export()
    # transform through the same cache, then give everything back and build once more
    p_h, c_h, _ = lb.ivfpq_transform(e_dev["centroids"], e_dev["codebook"], pin.array[:5000])
    p_d, c_d, _ = lb.ivfpq_transform(e_dev["centroids"], e_dev["codebook"], lb.DeviceArray.from_numpy(pin.array[:5000].copy()))
    assert np.array_equal(p_h, p_d) and np.array_equal(c_h, c_d)
    lb.trim_memory()
    e_again = lb.IvfPqIndex.build(pin, "l2", prm).export()
    assert np.array_equal(e_again["codes"], e_host["codes"])
