"""Every execution variant of the device Lloyd loop, and the grouping sort past its one-launch limits, pinned bit
for bit to the CPU oracle.

`lloyd_train` (lance_b200/csrc/lloyd.cu) promises the reference's model for the same initial centroids: the same
centroid bits, the same f64 loss and the same iteration count.  It reaches that promise by many routes:
  * fused: the whole run in one `lloyd_small_kernel` launch (K <= 16, n <= 16384, n*K*d <= 2^20, not profiling);
  * multi-kernel: one iteration = assignment, member sort, `update_stats_kernel`, `epilogue_kernel`, replayed from a
    CUDA graph (default), launched eagerly (LB2_NO_GRAPH=1), or launched eagerly with event profiling on (which also
    turns the fused kernel off); every one stops on the progress words at most one no-op iteration past convergence,
    which the profiled run checks by counting launches;
  * centroid sums by one warp per (cluster, 8 dims) (`update_body_warp`: d % 8 == 0 and 16-byte aligned rows) or
    one thread per (cluster, dim) (`update_body`);
  * order-independent fast paths for the centroid sums and the f64 loss, which must reject any cluster whose sum
    can round;
  * member lists by one cluster launch (K <= 1024, n <= 2^21) or hist -> scan -> offsets -> scatter;
  * the per-iteration epilogue: split_clusters, the balance bias, the loss sum in 1024-cluster chunks.
Each test compares with the oracle and checks which route ran: the fused kernel's launch count does not grow with
the iteration count (tolerance 0 runs every iteration), and the profile names the sort and update kernels."""
import os

import numpy as np
import pytest

import lance_b200 as lb
from lance_b200 import synth
from oracle import binding as ob

pytestmark = pytest.mark.gpu
NT = 16
MODES = ("graph", "eager", "profiled")


# ---- helpers ---------------------------------------------------------------------------------------------------
def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _same_model(km, ref):
    co, loss, iters = ref
    assert km.iters == iters, (km.iters, iters)
    assert np.array_equal(_bits(km.centroids), _bits(co))
    assert np.float64(km.loss).tobytes() == np.float64(loss).tobytes(), (km.loss, loss)


def _oracle(data, k, *, metric="l2", bf=0.0, init=None, max_iters=20, tol=1e-4, sample_rate=256, seed=0):
    """ob.kmeans_train on the rows train_kmeans keeps (the first sample_rate * k), balance factor after the division"""
    nn = min(len(data), sample_rate * k)
    bfo = float(np.float32(bf) / np.float32(nn)) if bf else 0.0
    return ob.kmeans_train(data[:nn], k, max_iters=max_iters, tolerance=tol, balance_factor=bfo, metric=metric,
                           seed=seed, init_centroids=init, nthreads=NT)


def _train(data, d, k, mode="graph", *, metric="l2", bf=0.0, init=None, max_iters=20, tol=1e-4, sample_rate=256,
           seed=0):
    """(KMeans, launches of the call, profile or None).  graph: default; eager: LB2_NO_GRAPH=1 (read on every call);
    profiled: event profiling on"""
    prev = os.environ.pop("LB2_NO_GRAPH", None)
    if mode == "eager":
        os.environ["LB2_NO_GRAPH"] = "1"
    if mode == "profiled":
        lb.profile.enable(True)
        lb.profile.reset()
    try:
        lb.launch_count(reset=True)
        km = lb.train_kmeans(data, d, k, max_iters=max_iters, distance_type=metric, sample_rate=sample_rate,
                             balance_factor=bf, tolerance=tol, seed=seed, centroids=init)
        launches = lb.launch_count()
    finally:
        os.environ.pop("LB2_NO_GRAPH", None)
        if prev is not None:
            os.environ["LB2_NO_GRAPH"] = prev
        if mode == "profiled":
            lb.profile.enable(False)
    return km, launches, (lb.profile.dump() if mode == "profiled" else None)


def _count(prof, name):
    """launches of kernel family `name`, whatever phase tag prefixes it"""
    return sum(v[0] for key, v in prof.items() if key.split(":")[-1] == name)


def _runs_fused(data, d, k, **kw):
    """with tolerance 0 every iteration runs: only the one-launch kernel keeps the count flat from 2 to 20"""
    kw = dict(kw, tol=0.0)
    return _train(data, d, k, max_iters=2, **kw)[1] == _train(data, d, k, max_iters=20, **kw)[1]


def _check_flat(data, d, k, *, fused, host=None, modes=MODES, **kw):
    """every mode equals the oracle; the profiled run went through the multi-kernel loop with the cluster sort
    (K <= 1024) or the four-kernel sort (K > 1024); `fused` says whether the default run is one launch"""
    ref = _oracle(data if host is None else host, k, **kw)
    prof = None
    for mode in modes:
        km, _, p = _train(data, d, k, mode, **kw)
        _same_model(km, ref)
        prof = p if p is not None else prof
    if prof is not None:
        assert _count(prof, "kmeans_small_fused") == 0
        # at most one no-op iteration past convergence (several cases converge at iteration 5 or 9 well below
        # max_iters, where stopping only at a multiple of 4 would launch more)
        for name in ("kmeans_update_stats", "kmeans_epilogue"):
            assert ref[2] <= _count(prof, name) <= ref[2] + 1, (name, _count(prof, name), ref[2])
        sort = "member_sort_cluster" if k <= 1024 else "member_sort"
        other = "member_sort" if k <= 1024 else "member_sort_cluster"
        assert _count(prof, sort) >= ref[2] and _count(prof, other) == 0
    assert _runs_fused(data, d, k, **{a: b for a, b in kw.items() if a != "max_iters"}) == fused
    return ref


def _init(data, k, seed):
    return data[np.random.default_rng(seed).choice(len(data), k, replace=False)].copy()


def _granule(v):
    """per f32 value: the largest e such that v is an integer multiple of 2^e (zero: a huge number)"""
    b = np.ascontiguousarray(v, np.float32).view(np.uint32) & np.uint32(0x7FFFFFFF)
    ex = (b >> 23).astype(np.int64)
    mant = (b & 0x7FFFFF).astype(np.int64)
    mant = np.where(ex > 0, mant | 0x800000, mant)
    ex = np.maximum(ex, 1)
    tz = np.log2(mant & -mant, where=mant > 0, out=np.zeros(mant.shape)).astype(np.int64)
    return np.where(mant > 0, ex - 150 + tz, 1 << 30)


def _seq_f32(col):
    return np.cumsum(np.asarray(col, np.float32), dtype=np.float32)[-1]


def _pairwise_f32(col):
    return np.ascontiguousarray(col, np.float32).sum(dtype=np.float32)  # numpy: pairwise along a contiguous axis


# ---- 1. flat Lloyd: fused kernel --------------------------------------------------------------------------------
# d = 4 / 12: tail only (no 16-wide body); 20 / 100: body + tail; 24: d % 8 == 0 with a tail (warp update)
FUSED = [(4, 16, 4000), (12, 2, 3000), (20, 16, 2000), (24, 4, 3000), (100, 1, 2000), (100, 16, 600)]


@pytest.mark.parametrize("bf", [0.0, 1.0])
@pytest.mark.parametrize("metric", ["l2", "dot"])
@pytest.mark.parametrize("d,k,n", FUSED)
def test_fused_kernel_equals_oracle_and_multi_kernel(d, k, n, metric, bf):
    data = synth.gaussian_mixture(n, d, n_components=2 * k + 2, seed=d * 100 + k)
    if metric == "dot":
        data *= np.float32(1.5)  # not normalised: negative distances reach the loss and the radius
    _check_flat(data, d, k, fused=True, metric=metric, bf=bf, init=_init(data, k, n), max_iters=12)


# ---- multi-kernel loop at nearby shapes (K > 16, or n*K*d > 2^20) ------------------------------------------------
MULTI = [(12, 32, 6000, "l2", 1.0), (20, 16, 8000, "dot", 0.0), (20, 20, 4000, "dot", 1.0), (100, 24, 3000, "l2", 0.0),
         (4, 64, 20000, "l2", 1.0), (24, 17, 5000, "dot", 1.0)]


@pytest.mark.parametrize("d,k,n,metric,bf", MULTI)
def test_multi_kernel_graph_eager_and_profiled_equal_oracle(d, k, n, metric, bf):
    data = synth.gaussian_mixture(n, d, n_components=k + 5, seed=d * 7 + k)
    if metric == "dot":
        data *= np.float32(2.0)
    _check_flat(data, d, k, fused=False, metric=metric, bf=bf, init=_init(data, k, n + 1), max_iters=15)


# ---- per-thread update at d % 8 == 0: rows whose base is 4 bytes past a 16-byte boundary -------------------------
class _Offset(lb.DeviceArray):
    """a view of `base`'s memory starting `offset` bytes in (owns nothing)"""

    def __init__(self, base, offset, shape):
        self.base, self.ptr = base, base.ptr + offset
        self.shape, self.dtype = tuple(shape), np.dtype(np.float32)
        self.nbytes = int(np.prod(self.shape)) * 4

    def free(self):
        pass


@pytest.mark.parametrize("d,k,n,fused", [(24, 8, 3000, True), (32, 40, 6000, False), (16, 12, 2000, True)])
def test_unaligned_device_rows_take_the_per_thread_update(d, k, n, fused):
    data = synth.gaussian_mixture(n, d, n_components=k + 3, seed=d + k)
    buf = lb.DeviceArray.from_numpy(np.concatenate([np.zeros(1, np.float32), data.ravel()]))
    view = _Offset(buf, 4, (n, d))
    assert view.ptr % 16 == 4
    init = _init(data, k, 3)
    ref = _check_flat(view, d, k, fused=fused, host=data, init=init, bf=1.0, max_iters=10)
    # the same rows 16-byte aligned (warp-per-8-dims update) give the same model
    _same_model(_train(lb.DeviceArray.from_numpy(data), d, k, init=init, bf=1.0, max_iters=10)[0], ref)


# ---- data built for the exact-sum checks -------------------------------------------------------------------------
def test_update_fast_path_rejects_integer_sums_past_2_24():
    """integer columns, 512 members per cluster, column sums ~2.6e7: past 2^24 the f32 chain rounds, so the
    fast path (sum|term| < 2^23) must hand every cluster to the ordered chain"""
    rng = np.random.default_rng(31)
    n, d, k = 4096, 8, 8                    # n = 512 * k: every row is in the sample
    h = np.array([[1, 1], [1, -1]], np.float32)
    signs = np.kron(np.kron(h, h), h)       # 8 sign patterns: the clusters are far apart
    group = rng.permutation(np.repeat(np.arange(k), n // k))
    data = (rng.integers(45000, 55001, (n, d)).astype(np.float32) * signs[group]).astype(np.float32)
    init = signs * np.float32(50000)
    ids, _, _ = ob.compute_membership(init, data, nthreads=NT)
    assert np.array_equal(ids, group)
    differ = 0
    for c in range(k):
        m = data[ids == c]
        assert 2 ** 24 < np.abs(m).sum(0).min() and np.abs(m).sum(0).max() < 3.0e7
        differ += sum(_seq_f32(m[:, j]) != _pairwise_f32(m[:, j]) for j in range(d))
    assert differ > 0, "no column sum depends on the order: the case would not test the rejection"
    _check_flat(data, d, k, fused=True, init=init, max_iters=6, sample_rate=512)


def test_update_fast_path_with_one_late_fraction():
    """integer rows except one fractional value near the end: the fast path rejects that cluster and clears the
    problem's hint while other warps may already have used it"""
    rng = np.random.default_rng(32)
    n, d, k = 4000, 16, 8
    data = rng.integers(0, 4000, (n, d)).astype(np.float32)
    init = _init(data, k, 5)
    r = n - 40
    for frac in np.linspace(0.01, 0.99, 50):
        x = data.copy()
        x[r, 5] = np.float32(x[r, 5] + frac)
        ids, _, _ = ob.compute_membership(init, x, nthreads=NT)
        col = x[ids == ids[r], 5]
        if _seq_f32(col) != _pairwise_f32(col):
            break
    else:
        pytest.fail("no fraction makes the cluster's sum order dependent")
    assert len(col) >= 64
    _check_flat(x, d, k, fused=True, init=init, max_iters=8, sample_rate=512)


@pytest.mark.parametrize("max_iters", [1, 4])
def test_loss_fast_path_rejects_a_60_binade_span(max_iters):
    """one cluster whose first-iteration distances are ~2^-8 (granule ~2^-31) and ~2^19: the f64 loss needs ~58
    bits, so the order-independent sum (at most 53) must not be used"""
    rng = np.random.default_rng(33)
    n, d = 400, 4
    mag = np.where((np.arange(n) % 2 == 0)[:, None], rng.uniform(2.0 ** -5, 2.0 ** -4, (n, d)),
                   rng.uniform(256.0, 512.0, (n, d)))
    data = (mag * rng.choice([-1.0, 1.0], (n, d))).astype(np.float32)
    init = np.zeros((1, d), np.float32)
    _, dist, _ = ob.compute_membership(init, data, nthreads=NT)
    g = int(_granule(dist).min())
    ad = np.abs(dist.astype(np.float64)).sum()
    assert 2.0 ** (g + 53) <= ad < 2.0 ** (g + 61), (g, np.log2(ad))
    dd = dist.astype(np.float64)
    assert np.cumsum(dd)[-1] != dd.sum(), "the f64 sum does not depend on the order"
    _check_flat(data, d, 1, fused=True, init=init, max_iters=max_iters, sample_rate=512)


@pytest.mark.parametrize("kind", ["integer", "fraction"])
def test_clusters_of_63_64_65_members(kind):
    """the fast paths start at 64 members: 63 runs the chain, 64 and 65 try the fast path"""
    rng = np.random.default_rng(34 if kind == "integer" else 35)
    d, sizes = 8, (63, 64, 65)
    group = rng.permutation(np.repeat(np.arange(3), sizes))
    centers = np.arange(3, dtype=np.float32)[:, None] * np.float32(1000) + np.zeros((1, d), np.float32)
    if kind == "integer":
        noise = rng.integers(-20, 21, (len(group), d)).astype(np.float32)
    else:
        noise = (rng.standard_normal((len(group), d)) * 10).astype(np.float32)
    data = (centers[group] + noise).astype(np.float32)
    ids, _, _ = ob.compute_membership(centers, data, nthreads=NT)
    assert np.array_equal(np.bincount(ids, minlength=3), sizes)
    if kind == "fraction":
        for c in range(3):
            m = data[ids == c]
            assert any(_seq_f32(m[:, j]) != _pairwise_f32(m[:, j]) for j in range(d))
    _check_flat(data, d, 3, fused=True, init=centers, max_iters=6)


# ---- epilogue edges ---------------------------------------------------------------------------------------------
def _edge_case(name):
    rng = np.random.default_rng(len(name))
    d = 8
    if name == "donor_of_size_1":
        # 3 finite rows + 3 NaN rows, 4 centroids: sizes 1, 1, 1, 0 -> no donor passes the draw, the 64*K-tries
        # guard takes the largest (size 1) and the child gets 0 rows
        x = rng.standard_normal((6, d)).astype(np.float32)
        x[[1, 3, 5]] = np.nan
        init = np.concatenate([x[[0, 2, 4]], np.full((1, d), 1000, np.float32)])
        return x, 4, dict(init=init, max_iters=3)
    if name == "n_equals_k":
        # p = (size - 1) / (n - K) = x / 0: NaN for size 1, Inf for size 2
        x = (rng.standard_normal((8, d)) * 5).astype(np.float32)
        init = np.concatenate([x[:7], x[:1]])
        return x, 8, dict(init=init, max_iters=4)
    if name == "all_rows_equal":
        # centroid == every row exactly (512 copies of small integers): loss 0 never meets the tolerance
        x = np.tile(np.arange(1, d + 1, dtype=np.float32), (512, 1))
        return x, 1, dict(init=x[:1] + np.float32(0.5), max_iters=7)
    x = synth.gaussian_mixture(3000, 12, n_components=10, seed=36)
    if name == "max_iters_1":
        return x, 12, dict(init=_init(x, 12, 1), max_iters=1, bf=1.0)
    return x, 12, dict(init=_init(x, 12, 2), max_iters=9, tol=0.0, bf=1.0)  # tolerance_0


@pytest.mark.parametrize("name", ["donor_of_size_1", "n_equals_k", "all_rows_equal", "max_iters_1", "tolerance_0"])
def test_epilogue_edges(name):
    x, k, kw = _edge_case(name)
    ref = _check_flat(x, x.shape[1], k, fused=True, **kw)
    if name == "all_rows_equal":
        assert ref[1] == 0.0 and ref[2] == kw["max_iters"]
    if name == "tolerance_0":
        assert ref[2] == kw["max_iters"]


# ---- sample caps ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d,k,n,sample_rate,fused", [(16, 8, 5000, 256, True),     # sample_rate * k binds
                                                     (16, 8, 10000, 1024, True),   # lloyd_train's 512 * k binds
                                                     (12, 24, 20000, 1024, False)])
def test_sample_caps(d, k, n, sample_rate, fused):
    data = synth.gaussian_mixture(n, d, n_components=k + 4, seed=n + d)
    assert n > min(sample_rate, 512) * k
    _check_flat(data, d, k, fused=fused, init=_init(data[:512 * k], k, 4), sample_rate=sample_rate, max_iters=10,
                bf=1.0)


# ---- non-finite training rows: not members, but counted in n -----------------------------------------------------
@pytest.mark.parametrize("metric", ["l2", "dot"])
@pytest.mark.parametrize("d,k,n,fused", [(12, 8, 2000, True), (32, 40, 6000, False)])
def test_non_finite_training_rows(d, k, n, fused, metric):
    data = synth.gaussian_mixture(n, d, n_components=k + 2, seed=37 + d)
    data[[5, 900, n - 3]] = np.nan          # whole NaN rows
    data[17, 3] = np.nan                    # a single NaN
    data[400, 0] = np.inf
    data[401, d - 1] = -np.inf
    data[1200] = np.float32(1e20)           # finite, but every L2 distance overflows to Inf
    rows = np.setdiff1d(np.arange(n), [5, 900, n - 3, 17, 400, 401, 1200])
    init = _init(data[rows], k, 6)
    _check_flat(data, d, k, fused=fused, metric=metric, init=init, bf=1.0, max_iters=10)


# ---- K > 1024: four-kernel member sort, the epilogue's loss in 1024-cluster chunks ---------------------------------
@pytest.mark.parametrize("k,n,bf", [(1025, 16000, 0.0), (2000, 24000, 1.0)])
def test_more_than_1024_clusters(k, n, bf):
    d = 32
    data = synth.gaussian_mixture(n, d, n_components=k, seed=k)
    init = _init(data, k, 7)
    _check_flat(data, d, k, fused=False, modes=("graph", "profiled"), init=init, bf=bf, max_iters=3)


# ---- 2. batched (PQ) Lloyd --------------------------------------------------------------------------------------
def _pq_init(data, M, K, seed):
    ds = data.shape[1] // M
    rng = np.random.default_rng(seed)
    return np.stack([data[rng.choice(len(data), K, replace=False)][:, m * ds:(m + 1) * ds] for m in range(M)])


def _check_pq(data, M, nbits, metric, init=None, seed=0, max_iters=10):
    """codebooks and iteration counts equal the oracle's, the profiled run (exact assignment kernel, multi-kernel
    loop, no tensor-core filter) included"""
    cbo, iters_o = ob.pq_train(data, M, nbits=nbits, max_iters=max_iters, metric=metric, seed=seed,
                               init_codebook=init, nthreads=NT)
    for profiled in (False, True):
        if profiled:
            lb.profile.enable(True)
            lb.profile.reset()
        try:
            pq = lb.PQBuildParams(M, nbits, max_iters=max_iters, codebook=init, seed=seed).build(data, metric)
        finally:
            lb.profile.enable(False)
        assert np.array_equal(pq.train_iters.astype(np.int32), iters_o)
        assert np.array_equal(_bits(pq.codebook), _bits(cbo))
    prof = lb.profile.dump()
    assert _count(prof, "pq_assign_exact") > 0 and _count(prof, "tc_pq_filter") == 0
    last = int(iters_o.max())  # the loop runs until the last sub-space converges, plus at most one no-op iteration
    for name in ("kmeans_update_stats", "kmeans_epilogue"):
        assert last <= _count(prof, name) <= last + 1, (name, _count(prof, name), last)
    return iters_o


@pytest.mark.parametrize("ds,seeded", [(1, False), (2, True), (12, False)])
def test_pq_narrow_and_wide_subvectors(ds, seeded):
    M, n = 4, 3000
    data = synth.gaussian_mixture(n, M * ds, n_components=300, seed=40 + ds)
    _check_pq(data, M, 8, "l2", init=None if seeded else _pq_init(data, M, 256, ds), seed=ds)


@pytest.mark.parametrize("kind", ["mixture", "converging"])
def test_pq_more_than_256_sub_spaces(kind):
    """384 sub-spaces of width 2: more than 256 problems, and progress words, in one Lloyd loop.  mixture: every
    sub-space runs to max_iters; converging: 256 groups per sub-space around the initial codewords, the noise growing
    from sub-space to sub-space, so they converge at iterations 3 to 10 and the loop stops on the last of them"""
    M, ds, n, K = 384, 2, 3000, 256
    if kind == "mixture":
        data = synth.gaussian_mixture(n, M * ds, n_components=300, seed=47)
        iters = _check_pq(data, M, 8, "l2", seed=7)
        assert (iters == 10).all()
        return
    rng = np.random.default_rng(47)
    centers = (rng.standard_normal((M, K, ds)) * 50).astype(np.float32)
    sigma = np.geomspace(1e-3, 1.0, M).astype(np.float32)
    pick = rng.integers(0, K, (n, M))
    noise = rng.standard_normal((n, M, ds)).astype(np.float32) * sigma[None, :, None]
    data = np.ascontiguousarray((centers[np.arange(M)[None, :], pick] + noise).reshape(n, M * ds), np.float32)
    iters = _check_pq(data, M, 8, "l2", init=centers, max_iters=16)
    assert iters.min() < iters.max() < 15, iters


def test_pq_dot_8_wide():
    data = synth.gaussian_mixture(4000, 32, n_components=300, seed=41) * np.float32(2)
    _check_pq(data, 4, 8, "dot", init=_pq_init(data, 4, 256, 1))


def test_pq_4bit_dot_unnormalised():
    data = synth.gaussian_mixture(2000, 16, n_components=40, seed=42) * np.float32(3)
    _check_pq(data, 4, 4, "dot", init=_pq_init(data, 4, 16, 2))


def test_pq_per_problem_hints_and_early_convergence():
    """sub-space 0: small integers (the exact-sum fast path holds), 1: fractions (it fails and clears that problem's
    hint only), 2: 256 tight groups around the initial codewords (converges early, then idles in the replayed graph)"""
    rng = np.random.default_rng(43)
    n, K = 25600, 256
    s0 = rng.integers(0, 16, (n, 8)).astype(np.float32)
    s1 = (rng.standard_normal((n, 8)) * 3).astype(np.float32)
    centers = (rng.standard_normal((K, 8)) * 50).astype(np.float32)
    s2 = (centers[rng.integers(0, K, n)] + rng.standard_normal((n, 8)) * 1e-3).astype(np.float32)
    data = np.ascontiguousarray(np.concatenate([s0, s1, s2], axis=1))
    init = _pq_init(data, 3, K, 3)
    init[2] = centers
    iters = _check_pq(data, 3, 8, "l2", init=init, max_iters=12)
    assert iters[2] < iters.max() and iters[2] <= 4, iters


def test_pq_nan_in_one_subvector():
    rng = np.random.default_rng(44)
    n, M = 3000, 2
    data = synth.gaussian_mixture(n, 16, n_components=200, seed=44)
    bad1, bad0 = [10, 500, n - 1], [777]
    data[bad1, 11] = np.nan                 # sub-space 1 only
    data[bad0, 2] = np.inf                  # sub-space 0 only
    init = _pq_init(data[np.setdiff1d(np.arange(n), bad1 + bad0)], M, 256, int(rng.integers(1000)))
    # the oracle trains each sub-space on its own columns: a row is a non-member only where its sub-vector is bad
    _, _, v0 = ob.compute_membership(init[0], data[:, :8], nthreads=NT)
    _, _, v1 = ob.compute_membership(init[1], data[:, 8:], nthreads=NT)
    assert v0[bad1].all() and not v1[bad1].any() and not v0[bad0].any() and v1[bad0].all()
    _check_pq(data, M, 8, "l2", init=init)


# ---- 3. hierarchical training -----------------------------------------------------------------------------------
def _dominant(n, d, seed, metric):
    """70 % of the rows in one blob, the rest spread over 200 components"""
    rng = np.random.default_rng(seed)
    data = synth.gaussian_mixture(n, d, n_components=200, seed=seed)
    big = rng.choice(n, int(0.7 * n), replace=False)
    data[big] = (rng.standard_normal((len(big), d)) * 2 + 5).astype(np.float32)
    return data * np.float32(2) if metric == "dot" else data


HIER = [(2, "l2", 12, 257, 6000, 0.0), (4, "dot", 32, 257, 6000, 1.0), (16, "dot", 12, 400, 12000, 0.0),
        (4, "l2", 32, 1500, 24000, 1.0), (16, "l2", 32, 1500, 40000, 1.0), (16, "l2", 12, 700, 12000, 0.0)]


@pytest.mark.parametrize("hk,metric,d,k,n,bf", HIER)
def test_hierarchical_equals_oracle_and_is_repeatable(hk, metric, d, k, n, bf):
    data = _dominant(n, d, hk * 1000 + k, metric)
    seed = k + hk
    bfo = float(np.float32(bf) / np.float32(n)) if bf else 0.0
    co, got = ob.hierarchical_kmeans(data, k, max_iters=10, balance_factor=bfo, metric=metric, hk=hk, seed=seed,
                                     nthreads=NT)
    assert got == k
    if (hk, d, n) == (16, 32, 40000):
        # the first splits run the multi-kernel loop (n * ck * d > 2^20); the small late ones the fused kernel
        top, _, _ = ob.kmeans_train(data, hk, max_iters=10, balance_factor=bfo, metric=metric, seed=seed, nthreads=NT)
        ids, _, _ = ob.compute_membership(top, data, metric=metric, nthreads=NT)
        assert np.bincount(ids).max() * hk * d > 2 ** 20
    for _ in range(2):  # the bits do not depend on the worker threads' timing
        km = lb.train_kmeans(data, d, k, max_iters=10, distance_type=metric, balance_factor=bf, seed=seed,
                             hierarchical_k=hk)
        assert np.array_equal(_bits(km.centroids), _bits(co))


def test_hierarchical_with_fewer_distinct_rows_than_k():
    """clusters of copies of one row cannot be split: the product stops where the oracle stops"""
    rng = np.random.default_rng(45)
    base = (rng.standard_normal((200, 16)) * 4).astype(np.float32)
    data = base[rng.integers(0, 200, 3000)]
    k = 300
    co, got = ob.hierarchical_kmeans(data, k, max_iters=10, seed=1, nthreads=NT)
    if got == k:
        assert np.array_equal(_bits(lb.train_kmeans(data, 16, k, max_iters=10, seed=1).centroids), _bits(co))
    else:
        with pytest.raises(lb.LanceB200Error, match="(?i)no cluster can be further split"):
            lb.train_kmeans(data, 16, k, max_iters=10, seed=1)


# ---- 4. grouping past the one-launch sort's limits ----------------------------------------------------------------
def _skewed_ids(rng, n, k):
    ids = ((rng.zipf(1.4, n) - 1) % k).astype(np.uint32)
    ids[ids == k // 2] = 0                  # an empty partition in the middle
    ids[rng.choice(n, 64, replace=False)] = k - 1
    return ids


def _expected_layout(ids, k):
    order = np.argsort(ids, kind="stable")
    off = np.concatenate([[0], np.cumsum(np.bincount(ids, minlength=k))]).astype(np.uint64)
    return order, off


def _profiled(fn):
    lb.profile.enable(True)
    lb.profile.reset()
    try:
        out = fn()
    finally:
        lb.profile.enable(False)
    return out, lb.profile.dump()


def _check_grouping(ids, k, d=8, M=2, profile=True):
    rng = np.random.default_rng(int(ids.size) + k)
    n = ids.size
    order, off = _expected_layout(ids, k)
    rid = (rng.permutation(n).astype(np.uint64) * np.uint64(3) + np.uint64(7))
    cent = rng.standard_normal((k, d)).astype(np.float32)
    codes = rng.integers(0, 256, (n, M), dtype=np.uint8)
    cb = rng.standard_normal((M, 256, d // M)).astype(np.float32)
    ix, prof = _profiled(lambda: lb.IvfPqIndex.from_parts(cent, cb, ids, codes, rid))
    e = ix.export()
    assert np.array_equal(e["part_offsets"], off)
    assert np.array_equal(e["row_ids"], rid[order]) and np.array_equal(e["codes"], codes[order])
    ix.close()
    vec = rng.standard_normal((n, d)).astype(np.float32)
    fx = lb.IvfFlatIndex.from_parts(cent, ids, vec, rid)
    f = fx.export()
    assert np.array_equal(f["part_offsets"], off)
    assert np.array_equal(f["row_ids"], rid[order]) and np.array_equal(_bits(f["vectors"]), _bits(vec[order]))
    fx.close()
    return prof


@pytest.mark.parametrize("k", [1024, 1025, 3000])
def test_grouping_across_the_partition_limit(k):
    ids = _skewed_ids(np.random.default_rng(k), 60000, k)
    counts = np.bincount(ids, minlength=k)
    assert (counts == 0).any() and counts.max() > 60000 // 4
    prof = _check_grouping(ids, k)
    assert (_count(prof, "member_sort") > 0) == (k > 1024)
    assert (_count(prof, "member_sort_cluster") > 0) == (k <= 1024)


@pytest.mark.parametrize("n", [1 << 21, (1 << 21) + 1])
def test_grouping_across_the_row_limit(n):
    k = 256
    ids = _skewed_ids(np.random.default_rng(n), n, k)
    prof = _check_grouping(ids, k, d=4, M=1)
    assert (_count(prof, "member_sort") > 0) == (n > 1 << 21)
    assert (_count(prof, "member_sort_cluster") > 0) == (n <= 1 << 21)


def test_ivfpq_build_with_1100_partitions_equals_oracle_layout_and_search():
    """hierarchical IVF training, the four-kernel grouping and the skew code layout (d = 128, M = 16) at K > 1024;
    NaN rows stay out of the index"""
    n, d, K, M = 60000, 128, 1100, 16
    data = synth.sift_like(n, d, n_components=2048, seed=46)
    bad = [3, 30001, n - 2]
    data[bad, 7] = np.nan
    q = synth.sift_like_queries(24, d, n_components=2048, seed=46)
    ix = lb.IvfPqIndex.build(data, "l2", lb.IvfBuildParams(num_partitions=K, num_sub_vectors=M, max_iters=5,
                                                           pq_max_iters=5))
    e = ix.export()
    keep = np.isfinite(data).all(axis=1)
    rows = np.flatnonzero(keep)
    p_ref, _, _ = ob.compute_membership(e["centroids"], data[keep], nthreads=NT)
    codes_ref = ob.pq_encode(e["codebook"], ob.compute_residual(e["centroids"], data[keep], p_ref, nthreads=NT),
                             nthreads=NT)
    order, off = _expected_layout(p_ref, K)
    assert np.array_equal(e["part_offsets"], off)
    assert np.array_equal(e["row_ids"], rows[order].astype(np.uint64))
    assert np.array_equal(e["codes"], codes_ref[order])
    ids, dists = ix.search(q, k=10, nprobes=12)
    oi, od, _ = ob.ivfpq_search(e["centroids"], e["codebook"], e["part_offsets"], e["codes"], e["row_ids"], q, 10, 12,
                                nthreads=NT)
    for i in range(len(q)):  # the same (distance, row id) pairs: rows tied at the k-th distance may swap
        assert sorted(zip(dists[i].view(np.uint32).tolist(), ids[i].tolist())) == \
            sorted(zip(od[i].view(np.uint32).tolist(), oi[i].tolist()))
