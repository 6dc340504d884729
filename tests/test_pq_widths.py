"""PQ code assignment and training at every sub-vector width ds = d / num_sub_vectors, pinned bit for bit to the CPU
oracle.

Every width has an exact device route (`pq_assign_f32`, lance_b200/csrc/assign.cu):
  * ds < 16: `small_d_kernel`, the reference's tail-only sum (l2.rs:69-79);
  * 16 <= ds <= 256: `pq_wide_kernel` (launches named `pq_assign_wide`): 16 lane sums in chunk order, added in lane
    order, plus the sequential tail;
  * ds > 256: each sub-space's rows copied out and assigned by the exact IVF assignment (`assign_f32_ex`);
  * ds = 8 keeps the tensor-core filter `tc_pq` for 8-bit codes.
The tests cover encode (plain, fused residual, f16 rows, non-finite rows, duplicated codewords, unaligned rows), a
case where the reference's 16-lane order and a plain sequential sum choose different codes, PQ training, and the
index layers above: IVF_PQ builds at the default num_sub_vectors, maintenance of an index opened from parts, and
IVF_HNSW_PQ graphs."""
import os

import numpy as np
import pytest

import hnsw_pq_reference as pr
import lance_b200 as lb
from lance_b200 import synth
from oracle import binding as ob
from test_ivf_hnsw_sq import _assert_graph_equal

pytestmark = pytest.mark.gpu
NT = 16
# the tail-only widths, the wide kernel's (chunk only, chunk + tail, up to its 256 bound) and two past the bound:
# 520 (not a multiple of 32: the exact kernel) and 1536 (the tensor-core filter with exact re-rank)
WIDTHS = [3, 5, 6, 7, 9, 10, 11, 13, 14, 15, 16, 17, 20, 24, 31, 32, 33, 48, 64, 96, 128, 256, 520, 1536]
ROWS = (1, 63, 65, 5000)


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _unpack(codes, nbits):
    """[n][M] codes from the stored bytes (4-bit: byte i = code[2i+1] << 4 | code[2i])"""
    if nbits == 8:
        return codes
    return np.stack([codes & 15, codes >> 4], axis=2).reshape(codes.shape[0], -1)


def _profiled(fn):
    lb.profile.enable(True)
    lb.profile.reset()
    try:
        out = fn()
    finally:
        lb.profile.enable(False)
    prof = lb.profile.dump()
    return out, lambda name: sum(v[0] for key, v in prof.items() if key.split(":")[-1] == name)


def _subspaces(ds):
    return 4 if ds <= 256 else 2


def _case(ds, nbits, n, seed):
    """codebook [M][2^nbits][ds] with codeword K-1 a duplicate of codeword 1 in every sub-space, and rows around the
    codewords: row 0 sits on the duplicated codeword, row 3 has a NaN in sub-space 0, row 4 an inf in the last
    sub-space and row 5 is all -inf"""
    rng = np.random.default_rng(seed)
    M, K = _subspaces(ds), 1 << nbits
    cb = rng.standard_normal((M, K, ds)).astype(np.float32)
    cb[:, K - 1] = cb[:, 1]
    pick = rng.integers(0, K, (n, M))
    x = cb[np.arange(M)[None, :], pick] + (rng.standard_normal((n, M, ds)) * 0.4).astype(np.float32)
    x = np.ascontiguousarray(x.reshape(n, M * ds), np.float32)
    x[0] = cb[:, K - 1].reshape(-1)
    x[3, 1] = np.nan
    x[4, -1] = np.inf
    x[5] = -np.inf
    return cb, x


def _route(ds, nbits):
    if ds == 8 and nbits == 8:
        return "tc_pq_filter"
    return "pq_assign_exact" if ds < 16 else "pq_assign_wide" if ds <= 256 else "pq_subspace_copy"


# ---- 1. encode ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("metric", ["l2", "dot"])
@pytest.mark.parametrize("nbits", [8, 4])
@pytest.mark.parametrize("ds", WIDTHS)
def test_encode_equals_oracle(ds, nbits, metric):
    cb, x = _case(ds, nbits, ROWS[-1], seed=10 * ds + nbits)
    M = cb.shape[0]
    pq = lb.ProductQuantizer(M, nbits, M * ds, cb, metric)
    for n in ROWS:
        got = pq.quantize(x[:n])
        assert np.array_equal(got, ob.pq_encode(cb, x[:n], nbits=nbits, metric=metric, nthreads=NT)), n
    codes = _unpack(got, nbits)
    assert codes[3, 0] == 0   # a NaN sub-vector has no winner: unwrap_or(0)
    if metric == "l2":
        assert (codes[0] == 1).all()   # on codewords 1 and K-1 at distance 0: the lower index wins
        assert codes[4, -1] == 0 and (codes[5] == 0).all()   # infinite distances never win either
    _, launched = _profiled(lambda: pq.quantize(x[:ROWS[-1]]))
    assert launched(_route(ds, nbits)) > 0


@pytest.mark.parametrize("nbits", [8, 4])
@pytest.mark.parametrize("ds", [5, 13, 16, 20, 48, 256, 520])
def test_fused_residual_equals_oracle(ds, nbits):
    n = 3000
    cb, x = _case(ds, nbits, n, seed=7 * ds + nbits)
    M, d = cb.shape[0], cb.shape[0] * ds
    rng = np.random.default_rng(ds)
    cent = (rng.standard_normal((40, d)) * 0.2).astype(np.float32)
    part = rng.integers(0, 40, n).astype(np.uint32)
    res = ob.compute_residual(cent, x, part, nthreads=NT)
    got = lb.ProductQuantizer(M, nbits, d, cb).quantize(x, cent, part)
    assert np.array_equal(got, ob.pq_encode(cb, res, nbits=nbits, nthreads=NT))


class _Offset(lb.DeviceArray):
    """a view of `base`'s memory starting `offset` bytes in (owns nothing)"""

    def __init__(self, base, offset, shape):
        self.base, self.ptr = base, base.ptr + offset
        self.shape, self.dtype = tuple(shape), np.dtype(np.float32)
        self.nbytes = int(np.prod(self.shape)) * 4

    def free(self):
        pass


@pytest.mark.parametrize("ds", [6, 16, 24, 520, 1536])
def test_unaligned_device_rows(ds):
    n, nbits = 2000, 8
    cb, x = _case(ds, nbits, n, seed=ds + 3)
    M, d = cb.shape[0], cb.shape[0] * ds
    buf = lb.DeviceArray.from_numpy(np.concatenate([np.zeros(1, np.float32), x.ravel()]))
    view = _Offset(buf, 4, (n, d))
    assert view.ptr % 16 == 4
    got = lb.ProductQuantizer(M, nbits, d, cb).quantize(view)
    assert np.array_equal(got, ob.pq_encode(cb, x, nbits=nbits, nthreads=NT))


@pytest.mark.parametrize("nbits", [8, 4])
@pytest.mark.parametrize("ds", [5, 16, 48])
def test_f16_rows_through_ivfpq_transform(ds, nbits):
    """an f16 column: partition, residual and code in one call, the model in f16 too"""
    n, K = 3000, 32
    cb, x = _case(ds, nbits, n, seed=ds + 50)
    x = np.nan_to_num(x, nan=0.0, posinf=0.0, neginf=0.0)
    x[7, 2] = np.nan                                     # a row KeepFiniteVectors drops
    rng = np.random.default_rng(ds)
    cent16 = (x[rng.choice(np.arange(10, n), K, replace=False)] * np.float32(0.9)).astype(np.float16)
    cb16, x16 = (cb * np.float32(0.5)).astype(np.float16), (x * np.float32(0.5)).astype(np.float16)
    cent16 = (cent16.astype(np.float32) * np.float32(0.5)).astype(np.float16)
    part, codes, valid = lb.ivfpq_transform(cent16, cb16, x16, num_bits=nbits)
    x32, cent32, cb32 = x16.astype(np.float32), cent16.astype(np.float32), cb16.astype(np.float32)
    po, _, vo = ob.compute_membership(cent32, x32, nthreads=NT)
    assert np.array_equal(valid, vo) and not vo[7]
    assert np.array_equal(part[vo], po[vo])
    res = ob.compute_residual(cent32, x32[vo], po[vo], nthreads=NT)
    assert np.array_equal(codes[vo], ob.pq_encode(cb32, res, nbits=nbits, nthreads=NT))


# ---- 2. the reference's summation order ---------------------------------------------------------------------------
def _lane_order(x, cb):
    """[n][K] L2 distances in the reference's order: 16 lane sums in chunk order, added in lane order (t), the tail
    summed left to right (s), s + t; every operation rounded to f32"""
    t = (x[:, None, :] - cb[None, :, :]) ** 2
    ds = x.shape[1]
    n16 = ds & ~15
    s = np.zeros(t.shape[:2], np.float32)
    for e in range(n16, ds):
        s = s + t[..., e]
    lanes = np.zeros(t.shape[:2] + (16,), np.float32)
    for c in range(0, n16, 16):
        lanes = lanes + t[..., c:c + 16]
    tt = np.zeros(t.shape[:2], np.float32)
    for lane in range(16):
        tt = tt + lanes[..., lane]
    return s + tt


def _sequential(x, cb):
    t = (x[:, None, :] - cb[None, :, :]) ** 2
    acc = np.zeros(t.shape[:2], np.float32)
    for e in range(x.shape[1]):
        acc = acc + t[..., e]
    return acc


@pytest.mark.parametrize("ds", [20, 48, 544])
def test_reference_lane_order_decides_codes(ds):
    """Every codeword shares two large coordinates (one in the 16-lane chunks, one in the tail, or the last chunk at
    ds = 48), so each distance is ~1e6 and the codewords differ only by tiny terms that the large partial sums absorb
    differently in each order.  A kernel that sums in any other order picks other codes for some rows."""
    n, K, M = 1500, 256, 2
    rng = np.random.default_rng(ds)
    big = [0, ds - 1]
    cbs, xs = [], []
    for _ in range(M):
        cb = (rng.standard_normal((K, ds)) * 0.1).astype(np.float32)
        cb[:, big] = np.float32(1000.0)
        x = (rng.standard_normal((n, ds)) * 0.1).astype(np.float32)
        x[:, big] = (rng.standard_normal((n, len(big))) * 3).astype(np.float32)
        cbs.append(cb)
        xs.append(x)
    def codes(dist):  # first minimum per row, 100 rows at a time (bounds the [rows][K][ds] temporaries)
        return np.stack([np.concatenate([np.argmin(dist(x[r:r + 100], cb), axis=1) for r in range(0, n, 100)])
                         for x, cb in zip(xs, cbs)], axis=1)

    ref, seq = codes(_lane_order), codes(_sequential)
    differ = int((ref != seq).sum())
    assert differ > 0, "no code depends on the order: the case would not test it"
    cb, x = np.stack(cbs), np.ascontiguousarray(np.concatenate(xs, axis=1))
    assert np.array_equal(ob.pq_encode(cb, x, nthreads=NT), ref)
    got = lb.ProductQuantizer(M, 8, M * ds, cb).quantize(x)
    assert np.array_equal(got, ref)


# ---- 3. training --------------------------------------------------------------------------------------------------
def _train_data(ds, nbits, n, seed):
    """sub-space 0: tight groups around the initial codewords (under L2 it converges within a few iterations); the
    others: a Gaussian mixture that keeps moving.  Returns (data, initial codebook)"""
    rng = np.random.default_rng(seed)
    M, K = _subspaces(ds), 1 << nbits
    data = synth.gaussian_mixture(n, M * ds, n_components=300, seed=seed).reshape(n, M, ds)
    centers = (rng.standard_normal((K, ds)) * 20).astype(np.float32)
    data[:, 0] = centers[rng.integers(0, K, n)] + (rng.standard_normal((n, ds)) * 1e-3).astype(np.float32)
    data = np.ascontiguousarray(data.reshape(n, M * ds))
    init = np.stack([data[rng.choice(n, K, replace=False)][:, m * ds:(m + 1) * ds] for m in range(M)])
    init[0] = centers
    return data, init


@pytest.mark.parametrize("init", [False, True], ids=["seeded", "init"])
@pytest.mark.parametrize("metric", ["l2", "dot"])
@pytest.mark.parametrize("nbits", [8, 4])
@pytest.mark.parametrize("ds", [5, 16, 24, 48, 544])
def test_training_equals_oracle(ds, nbits, metric, init):
    """codebook bits and iteration counts equal the oracle's, replayed from the CUDA graph, eager, and eager with
    event profiling (which also names the assignment route)"""
    data, cb0 = _train_data(ds, nbits, 3000, seed=ds + nbits)
    M, max_iters = cb0.shape[0], 12
    cb0 = cb0 if init else None
    cbo, iters_o = ob.pq_train(data, M, nbits=nbits, max_iters=max_iters, metric=metric, seed=3, init_codebook=cb0,
                               nthreads=NT)
    train = lambda: lb.PQBuildParams(M, nbits, max_iters=max_iters, codebook=cb0, seed=3).build(data, metric)  # noqa
    prev = os.environ.pop("LB2_NO_GRAPH", None)
    try:
        runs = [train()]
        os.environ["LB2_NO_GRAPH"] = "1"
        runs.append(train())
        os.environ.pop("LB2_NO_GRAPH")
        pq, launched = _profiled(train)
        runs.append(pq)
    finally:
        os.environ.pop("LB2_NO_GRAPH", None)
        if prev is not None:
            os.environ["LB2_NO_GRAPH"] = prev
    for pq in runs:
        assert np.array_equal(pq.train_iters.astype(np.int32), iters_o)
        assert np.array_equal(_bits(pq.codebook), _bits(cbo))
    assert launched(_route(ds, nbits)) > 0
    if init and metric == "l2":
        assert iters_o[0] < iters_o.max(), iters_o   # sub-spaces converge at different iterations


# ---- 4. IVF_PQ builds at the default num_sub_vectors ------------------------------------------------------------
def _same_topk(ids, dists, oi, od):
    for q in range(len(ids)):
        got = sorted(zip(np.asarray(dists[q]).view(np.uint32).tolist(), np.asarray(ids[q]).tolist()))
        exp = sorted(zip(np.asarray(od[q]).view(np.uint32).tolist(), np.asarray(oi[q]).tolist()))
        assert got == exp, q


def _oracle_codes(parts, x, metric, nbits=8):
    """partition and codes of rows x under the model in `parts`: the reference's transform (L2 codes, residuals
    unless the metric is dot)"""
    po, _, _ = ob.compute_membership(parts["centroids"], x, metric=metric, nthreads=NT)
    src = x if metric == "dot" else ob.compute_residual(parts["centroids"], x, po, nthreads=NT)
    return po, ob.pq_encode(parts["codebook"], src, nbits=nbits, nthreads=NT)


@pytest.mark.parametrize("metric", ["l2", "dot"])
@pytest.mark.parametrize("d", [256, 768])
def test_ivfpq_build_default_subvectors(d, metric):
    n, K, k = 20000, 16, 10
    data = synth.gaussian_mixture(n, d, n_components=64, seed=d)
    queries = synth.gaussian_mixture(8, d, n_components=64, seed=d + 1)
    params = lb.IvfBuildParams(num_partitions=K, max_iters=10, pq_max_iters=10)
    assert params.num_sub_vectors == 16
    ix = lb.IvfPqIndex.build(data, metric, params)
    parts = ix.export()
    assert parts["codebook"].shape == (16, 256, d // 16)
    po, co = _oracle_codes(parts, data, metric)
    order = np.argsort(parts["row_ids"])
    part_of_row = np.repeat(np.arange(K, dtype=np.uint32), np.diff(parts["part_offsets"]).astype(np.int64))[order]
    assert np.array_equal(part_of_row, po)
    assert np.array_equal(parts["codes"][order], co)
    for nprobes in (1, K):
        ids, dists = ix.search(queries, k=k, nprobes=nprobes)
        oi, od, _ = ob.ivfpq_search(parts["centroids"], parts["codebook"], parts["part_offsets"], parts["codes"],
                                    parts["row_ids"], queries, k, nprobes, metric=metric, nthreads=NT)
        _same_topk(ids, dists, oi, od)


# ---- 5. maintenance of an index opened from parts (d = 128, M = 8: ds = 16) ---------------------------------------
@pytest.mark.parametrize("nbits", [8, 4])
@pytest.mark.parametrize("metric", ["l2", "dot"])
def test_transform_and_optimize_of_a_reference_shaped_index(metric, nbits):
    d, M, K, n, n_add, k = 128, 8, 12, 4000, 1500, 10
    rng = np.random.default_rng(nbits)
    data = synth.gaussian_mixture(n + n_add, d, n_components=40, seed=5)
    old, new = data[:n], data[n:]
    cent = data[rng.choice(n, K, replace=False)].copy()
    cb = (rng.standard_normal((M, 1 << nbits, d // M)) * 0.5).astype(np.float32)
    parts = dict(centroids=cent, codebook=cb)
    po_old, codes_old = _oracle_codes(parts, old, metric, nbits)
    rid_old = np.arange(n, dtype=np.uint64) * 3
    ix = lb.IvfPqIndex.from_parts(cent, cb, po_old, codes_old, rid_old, metric, num_bits=nbits)

    po, co = _oracle_codes(parts, new, metric, nbits)
    part, codes, valid = lb.ivfpq_transform(cent, cb, new, metric, num_bits=nbits)
    assert valid.all() and np.array_equal(part, po) and np.array_equal(codes, co)
    t = ix.transform(new)
    assert t["valid"].all() and np.array_equal(t["part_ids"], po) and np.array_equal(t["payload"], co)

    rid_new = np.arange(n_add, dtype=np.uint64) * 3 + 1
    opt = ix.optimize(add_vectors=new, add_row_ids=rid_new)
    got = opt.export()
    # stable grouping by partition: the old rows, then the added rows, in input order within a partition
    all_part = np.concatenate([po_old, po])
    order = np.argsort(all_part, kind="stable")
    assert np.array_equal(got["row_ids"], np.concatenate([rid_old, rid_new])[order])
    assert np.array_equal(got["codes"], np.concatenate([codes_old, co])[order])
    queries = synth.gaussian_mixture(8, d, n_components=40, seed=6)
    for nprobes in (1, K):
        ids, dists = opt.search(queries, k=k, nprobes=nprobes)
        oi, od, _ = ob.ivfpq_search(cent, cb, got["part_offsets"], got["codes"], got["row_ids"], queries, k, nprobes,
                                    metric=metric, nbits=nbits, nthreads=NT)
        _same_topk(ids, dists, oi, od)


# ---- 6. IVF_HNSW_PQ at ds = 16 ------------------------------------------------------------------------------------
@pytest.mark.parametrize("nbits", [8, 4])
@pytest.mark.parametrize("metric", ["l2", "dot"])
def test_ivf_hnsw_pq_graph_at_width_16(metric, nbits):
    d, M, m, efc = 64, 4, 12, 60
    x = synth.gaussian_mixture(1200, d, n_components=30, seed=nbits)
    x[-40:] = x[:40]
    params = lb.IvfBuildParams(num_partitions=5, num_sub_vectors=M, num_bits=nbits, max_iters=10, pq_max_iters=10,
                               seed=5)
    hp = lb.HnswBuildParams(max_level=5, m=m, ef_construction=efc)
    got = lb.IvfHnswPqIndex.build(x, metric, params, hp).export()
    pq = lb.IvfPqIndex.build(x, metric, params).export()
    for key in ("centroids", "codebook", "part_offsets", "codes", "row_ids"):
        assert np.array_equal(got[key], pq[key]), key
    order = np.argsort(got["row_ids"])
    assert np.array_equal(got["codes"][order], _oracle_codes(got, x, metric, nbits)[1])
    want = pr.build(got["codes"], got["part_offsets"], got["codebook"], nbits, metric, "f32", m=m, max_level=5,
                    efc=efc, seed=5)
    _assert_graph_equal(got["graph"], want)
