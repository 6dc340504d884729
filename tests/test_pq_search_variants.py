"""The IVF_PQ query path against the oracle: probe selection, residual query, LUT (`build_lut_smem`: fixed-width code
for sub-vector widths 4, 8 and 16, a generic loop for every other width), the 8-bit row sum (`pq8_row_distance`: 16-byte
loads when M % 16 == 0, a byte loop otherwise), the selection routes and the merge.

Indexes are opened with `from_parts`, so every partition has exactly the size a case needs; centroids and codebooks
are random.  Which route a search takes follows from its numbers (SCAN_KFAST = 16, SCAN_CHUNK = 4096):
  * 8-bit, k + 1 <= 16: the skewed kernel (M = 16 x 8 dims, 2 or 4 teams) or the classic kernel, then the tie replay
    (`ivfpq_scan_radix_kernel` in list mode) for slots whose k-th and (k + 1)-th candidates tie;
  * 8-bit with k + 1 > 16, and every 4-bit search: the radix slot (`radix_slot`);
  * 4-bit: rows [0, flat_num) with flat_num = min(max(200, k), n_p) and the last n_p % 16 rows are exact sums, the
    others go through the table quantised to u8; with a prefilter every row is exact.
`LB2_SCAN=classic|skew` and `LB2_SCAN_TEAMS=2|4` force the fast 8-bit variant; `lb.profile` counts prove the route.

Every result is compared with the oracle BIT FOR BIT, ids and distances (NaN distances as NaN)."""
import numpy as np
import pytest

import lance_b200 as lb
from lance_b200._lib import UNSUPPORTED
from oracle import binding as ob

pytestmark = pytest.mark.gpu
NT = 16
NONE = np.uint64(2 ** 64 - 1)
SIZES = [0, 1, 31, 32, 33, 511, 512, 513, 4095, 4096, 4097, 12003]
# 4-bit: flat_num = 200 covers the whole partition, ends before the exact n_p % 16 tail, or inside / after it
SIZES4 = [15, 16, 17, 199, 200, 201, 215, 216, 217, 4111]


# ---- helpers -----------------------------------------------------------------------------------------------------
def _model(rng, sizes, M, ds, nbits=8, spread=3.0):
    """(centroids, codebook, part, data): data near its partition's centroid, in partition order"""
    K, d = len(sizes), M * ds
    cent = (rng.standard_normal((K, d)) * spread).astype(np.float32)
    cb = rng.standard_normal((M, 1 << nbits, ds)).astype(np.float32)
    part = np.repeat(np.arange(K, dtype=np.uint32), sizes)
    data = (cent[part] + rng.standard_normal((len(part), d))).astype(np.float32)
    return cent, cb, part, data


def _encode(cb, cent, part, data, metric, nbits=8):
    res = data if metric == "dot" else data - cent[part]
    return ob.pq_encode(cb, res, nbits=nbits, nthreads=NT)


def _open(rng, cent, cb, part, codes, metric, nbits=8, data=None):
    """IVF_PQ index over the given rows (shuffled, sparse row ids); checks every partition kept its size.  With
    `data`, also returns the column the row ids index (row id r -> col[r]; rows no id names are zero)."""
    n = len(part)
    perm = rng.permutation(n)
    rid = rng.permutation(n).astype(np.uint64) * 3 + 1
    ix = lb.IvfPqIndex.from_parts(cent, cb, part[perm], codes[perm], rid, metric, num_bits=nbits)
    parts = ix.export()
    assert np.array_equal(np.diff(parts["part_offsets"].astype(np.int64)), np.bincount(part, minlength=len(cent)))
    if data is None:
        return ix, parts
    col = np.zeros((3 * n + 1, data.shape[1]), np.float32)
    col[rid.astype(np.int64)] = data[perm]
    return ix, parts, col


def _oracle(parts, q, k, nprobes, metric, nbits=8, **kw):
    return ob.ivfpq_search(parts["centroids"], parts["codebook"], parts["part_offsets"], parts["codes"],
                           parts["row_ids"], q, k, nprobes, metric=metric, nbits=nbits, nthreads=NT, **kw)


def _assert_equal(got, want, what):
    ids, dists = got
    oi, od = want[0], want[1]
    for i in range(len(oi)):
        if not (np.array_equal(ids[i], oi[i]) and np.array_equal(dists[i], od[i], equal_nan=True)):
            r = next(j for j in range(len(oi[i])) if ids[i, j] != oi[i, j] or not
                     (dists[i, j] == od[i, j] or (np.isnan(dists[i, j]) and np.isnan(od[i, j]))))
            raise AssertionError(f"{what}: query {i}, rank {r}: got ({ids[i, r]}, {dists[i, r]!r}), "
                                 f"want ({oi[i, r]}, {od[i, r]!r}); count got {int(np.sum(ids[i] != NONE))}, "
                                 f"want {int(want[2][i])}")


def _profiled(fn):
    lb.profile.reset()
    lb.profile.enable(True)
    try:
        out = fn()
    finally:
        lb.profile.enable(False)
    return out, lb.profile.dump()


def _ran(prof, name):
    return prof.get(name, (0, 0))[0]


def _route(prof):
    """which 8-bit / 4-bit scan route a search took"""
    if _ran(prof, "search:pq_scan_skew"):
        assert _ran(prof, "search:pq_scan") == 0 and _ran(prof, "search:pq_scan_tie_replay") == 1, prof
        return "skew"
    assert _ran(prof, "search:pq_scan") == 1, prof
    return "classic" if _ran(prof, "search:pq_scan_tie_replay") == 1 else "radix"


def _queries(rng, cent, sizes, nq, noise=1.0):
    """half near the largest partitions (multi-chunk lists), half near random ones"""
    big = np.argsort(sizes)[-3:]
    c = np.concatenate([rng.choice(big, nq // 2), rng.integers(0, len(sizes), nq - nq // 2)])
    return (cent[c] + rng.standard_normal((nq, cent.shape[1])) * noise).astype(np.float32)


# ---- 1. 8-bit: sub-vector width x count -------------------------------------------------------------------------
# every width in {1, 2, 3, 4, 5, 8, 12, 16, 20, 32} and every count in {1, 2, 7, 8, 15, 16, 17, 32, 48, 96, 192}:
# ds = 4 / 8 / 16 take lut_entry_fixed, the others dist_exact_thread (ds = 20: one 16-lane chunk + a 4-element tail);
# M % 16 != 0 takes the byte loop of pq8_row_distance.  ds = 16 with M = 8 is a reference-built index at d = 128.
SHAPES8 = [(1, 192), (2, 96), (3, 17), (4, 48), (4, 7), (5, 7), (8, 32), (8, 17), (12, 15), (16, 8), (16, 2),
           (20, 1), (32, 16)]


@pytest.mark.parametrize("metric", ["l2", "dot", "cosine"])
@pytest.mark.parametrize("ds,M", SHAPES8, ids=[f"ds{ds}-M{M}" for ds, M in SHAPES8])
def test_pq8_subvector_widths_and_counts_match_oracle(ds, M, metric):
    rng = np.random.default_rng(6100 + 31 * ds + M + 7 * len(metric))
    sizes = [0, 1, 33, 700, 4097, 5000]
    cent, cb, part, data = _model(rng, sizes, M, ds)
    ix, parts = _open(rng, cent, cb, part, _encode(cb, cent, part, data, metric), metric)
    q = _queries(rng, cent, sizes, 12)
    for k, nprobes, route in ((10, 3, "classic"), (100, len(sizes), "radix"), (1, 1, "classic")):
        got, prof = _profiled(lambda: ix.search(q, k=k, nprobes=nprobes))
        _assert_equal(got, _oracle(parts, q, k, nprobes, metric), (ds, M, metric, k, nprobes))
        assert _route(prof) == route, (k, prof)


# ---- 2. 8-bit routes on both sides of their boundaries, partition sizes around the warp / slab / chunk edges -------
ROUTE_SHAPES = [("l2", 8, 16), ("dot", 8, 16), ("cosine", 8, 16), ("l2", 3, 17)]


@pytest.mark.parametrize("metric,ds,M", ROUTE_SHAPES, ids=[f"{m}-ds{ds}-M{M}" for m, ds, M in ROUTE_SHAPES])
def test_pq8_routes_and_partition_sizes_match_oracle(metric, ds, M, monkeypatch):
    """k = 1, 14, 15: the fast kernels (skewed with 2 and 4 teams where M = 16 x 8 dims, and classic); k = 16 .. 1024:
    the radix slot.  The 12003-row partition draws its codes from 48 distinct ones, so most of its lists tie at the
    k-th place and go through the replay."""
    rng = np.random.default_rng(6200 + M + 3 * len(metric))
    cent, cb, part, data = _model(rng, SIZES, M, ds)
    codes = _encode(cb, cent, part, data, metric)
    lo = int(np.sum(SIZES[:-1]))
    codes[lo:] = codes[lo + rng.integers(0, 48, SIZES[-1])]
    ix, parts = _open(rng, cent, cb, part, codes, metric)
    K = len(SIZES)
    q = _queries(rng, cent, SIZES, 16)
    skew = M == 16 and ds == 8
    fast = ["classic"] + (["skew2", "skew4"] if skew else [])
    for k, nprobes in ((1, K), (14, 3), (15, K), (16, 2), (17, K), (135, 4), (136, K), (1023, 2), (1024, K)):
        want = _oracle(parts, q, k, nprobes, metric)
        for mode in (fast if k + 1 <= 16 else ["radix"]):
            if mode != "radix":
                monkeypatch.setenv("LB2_SCAN", "classic" if mode == "classic" else "skew")
                monkeypatch.setenv("LB2_SCAN_TEAMS", "4" if mode == "skew4" else "2")
            got, prof = _profiled(lambda: ix.search(q, k=k, nprobes=nprobes))
            _assert_equal(got, want, (metric, M, mode, k, nprobes))
            assert _route(prof) == mode.rstrip("24"), (mode, k, prof)


@pytest.mark.parametrize("teams", ["2", "4"])
def test_skew_list_overflow_goes_to_the_replay(teams, monkeypatch):
    """6000 rows with one identical code: every row of a chunk ties at the threshold, more rows than a team list holds
    (1024 rows with 2 teams, 512 with 4), in every chunk (4096 / 2048 rows), so only the exact replay can settle the
    slot; the reference's heap decides which tied rows are returned."""
    rng = np.random.default_rng(6300 + int(teams))
    sizes = [6000, 900, 4097]
    cent, cb, part, data = _model(rng, sizes, 16, 8)
    codes = _encode(cb, cent, part, data, "l2")
    codes[:6000] = codes[rng.integers(0, 6000)]
    ix, parts = _open(rng, cent, cb, part, codes, "l2")
    q = (cent[[0, 0, 0, 1, 2, 0]] + rng.standard_normal((6, 128)) * 0.5).astype(np.float32)
    monkeypatch.setenv("LB2_SCAN", "skew")
    monkeypatch.setenv("LB2_SCAN_TEAMS", teams)
    for k in (1, 10, 15):
        for nprobes in (1, 3):
            got, prof = _profiled(lambda: ix.search(q, k=k, nprobes=nprobes))
            assert _route(prof) == "skew", prof
            _assert_equal(got, _oracle(parts, q, k, nprobes, "l2"), (teams, k, nprobes))


# ---- 3. the shared-memory limit ----------------------------------------------------------------------------------
def _limit_index(rng, M, nbits=8, ds=1):
    """one partition with 60 distinct codes over 4097 rows (ties at the k-th place: the replay), three others"""
    sizes = [300, 0, 4097, 50]
    cent, cb, part, _ = _model(rng, sizes, M, ds, nbits)
    cw = M // 2 if nbits == 4 else M
    codes = rng.integers(0, 256, (len(part), cw), dtype=np.uint8)
    codes[300:4397] = codes[300 + rng.integers(0, 60, 4097)]
    ix, parts = _open(rng, cent, cb, part, codes, "l2", nbits)
    q = (cent[[2, 2, 0, 3, 2, 0]] + rng.standard_normal((6, cent.shape[1])) * 0.5).astype(np.float32)
    return ix, parts, q


def _refused(fn):
    """True if fn raises LB2_UNSUPPORTED for lack of shared memory; any other error propagates"""
    try:
        fn()
    except lb.LanceB200Error as e:
        if e.status == UNSUPPORTED and "shared memory" in str(e):
            return True
        raise
    return False


@pytest.mark.parametrize("k", [10, 1024])
def test_pq8_largest_admitted_sub_vector_count_matches_oracle(k):
    """ds = 1: the LUT takes 1 KB per sub-vector.  The largest M the entry check admits must run every kernel its
    route launches (k = 10: the classic kernel and the tie replay; k = 1024: the radix slot) -- their static shared
    memory included -- and match the oracle; M + 1 must be refused with LB2_UNSUPPORTED."""
    rng = np.random.default_rng(6400 + k)
    lo, hi = 16, 256                       # 256 KB of LUT: more than any H100 block may hold
    while hi - lo > 1:
        mid = (lo + hi) // 2
        ix, parts, q = _limit_index(rng, mid)
        if _refused(lambda: ix.search(q, k=k, nprobes=2)):
            hi = mid
        else:
            lo = mid
    ix, parts, q = _limit_index(rng, lo)
    allow = parts["row_ids"][rng.choice(len(parts["row_ids"]), 3000, replace=False)]
    bm = ix.row_mask(allow, None)
    for nprobes in (1, 4):
        got, prof = _profiled(lambda: ix.search(q, k=k, nprobes=nprobes))
        _assert_equal(got, _oracle(parts, q, k, nprobes, "l2"), (lo, k, nprobes))
        assert _route(prof) == ("classic" if k < 16 else "radix"), prof
        got = ix.search_ex(q, k=k, nprobes=nprobes, allow_bitmap=bm)
        _assert_equal(got, _oracle(parts, q, k, nprobes, "l2", allow=allow), ("allow", lo, k, nprobes))
    ix, parts, q = _limit_index(rng, lo + 1)
    assert _refused(lambda: ix.search(q, k=k, nprobes=2)), lo + 1


@pytest.mark.parametrize("ds", [1, 2])
def test_pq4_sub_vector_count_256_matches_oracle(ds):
    """a 4-bit LUT holds M x 16 entries: M = 256, the largest count the entry point takes, fits at any k; M = 258 is
    refused by the count check."""
    rng = np.random.default_rng(6500 + ds)
    ix, parts, q = _limit_index(rng, 256, 4, ds)
    for k, nprobes in ((10, 2), (250, 4), (1024, 2)):
        got, prof = _profiled(lambda: ix.search(q, k=k, nprobes=nprobes))
        assert _route(prof) == "radix", prof
        _assert_equal(got, _oracle(parts, q, k, nprobes, "l2", nbits=4), (ds, k, nprobes))
    ix, parts, q = _limit_index(rng, 258, 4, ds)
    with pytest.raises(lb.LanceB200Error) as e:
        ix.search(q, k=10, nprobes=2)
    assert e.value.status == UNSUPPORTED


# ---- 4. 4-bit ------------------------------------------------------------------------------------------------------
SHAPES4 = [(2, 2), (4, 1), (16, 2), (34, 1), (128, 2), (210, 1), (256, 1)]


@pytest.mark.parametrize("metric", ["l2", "dot"])
@pytest.mark.parametrize("M,ds", SHAPES4, ids=[f"M{M}-ds{ds}" for M, ds in SHAPES4])
def test_pq4_counts_and_partition_sizes_match_oracle(M, ds, metric):
    """k below and above 200 moves flat_num; partitions around 200 and 216 and with n_p % 16 != 0 put the exact tail
    before, inside or after the quantised rows"""
    rng = np.random.default_rng(6600 + M + 7 * ds + len(metric))
    sizes = SIZES4 + ([0, 1, 512, 4097, 12003] if M <= 34 else [4097])
    cent, cb, part, data = _model(rng, sizes, M, ds, 4)
    ix, parts = _open(rng, cent, cb, part, _encode(cb, cent, part, data, metric, 4), metric, 4)
    q = _queries(rng, cent, sizes, 10)
    for k, nprobes in ((10, len(sizes)), (199, 3), (201, len(sizes)), (1024, 2)):
        got, prof = _profiled(lambda: ix.search(q, k=k, nprobes=nprobes))
        assert _route(prof) == "radix", prof
        _assert_equal(got, _oracle(parts, q, k, nprobes, metric, 4), (M, ds, metric, k, nprobes))


@pytest.mark.parametrize("metric", ["l2", "dot"])
def test_pq4_filters_refine_and_non_finite_queries_match_oracle(metric):
    """prefilter (every row exact), range bounds alone (the quantised distances are filtered), both, refine, and
    queries with an Inf, a 3e38 and a NaN component (the quantisation range is then Inf or NaN: q * range + qmin
    is NaN for q = 0)"""
    rng = np.random.default_rng(6700 + len(metric))
    M, ds = 34, 2
    sizes = [0, 17, 201, 216, 4111, 5003]
    K = len(sizes)
    cent, cb, part, data = _model(rng, sizes, M, ds, 4)
    ix, parts, col = _open(rng, cent, cb, part, _encode(cb, cent, part, data, metric, 4), metric, 4, data)
    q = _queries(rng, cent, sizes, 12)
    allow = rng.choice(parts["row_ids"], len(part) // 3, replace=False)
    bm = ix.row_mask(allow, None)
    for k, nprobes in ((10, 3), (300, K)):
        got = ix.search_ex(q, k=k, nprobes=nprobes, allow_bitmap=bm)
        _assert_equal(got, _oracle(parts, q, k, nprobes, metric, 4, allow=allow), ("allow", k, nprobes))
    _, d0 = ix.search(q, k=400, nprobes=K)
    lo, hi = float(np.median(d0[:, 5])), float(np.median(d0[:, 350]))
    for k, nprobes in ((10, K), (300, 3)):
        got = ix.search_ex(q, k=k, nprobes=nprobes, lower_bound=lo, upper_bound=hi)
        _assert_equal(got, _oracle(parts, q, k, nprobes, metric, 4, lower=lo, upper=hi), ("range", k, nprobes))
        got = ix.search_ex(q, k=k, nprobes=nprobes, allow_bitmap=bm, lower_bound=lo, upper_bound=hi)
        _assert_equal(got, _oracle(parts, q, k, nprobes, metric, 4, allow=allow, lower=lo, upper=hi),
                      ("allow+range", k, nprobes))
    # refine: the oracle's 4-bit candidates re-ranked with the exact distance, ascending (distance, id)
    for k, rf, nprobes in ((10, 20, 3), (100, 10, K)):
        ids, dists = ix.search_refine(col, q, k=k, nprobes=nprobes, refine_factor=rf)
        oi, _, oc = _oracle(parts, q, k * rf, nprobes, metric, 4)
        for i in range(len(q)):
            cand = oi[i, :oc[i]].astype(np.int64)
            ex = np.array([ob.l2(q[i], col[c]) if metric == "l2" else np.float32(1.0) - np.float32(ob.dot(q[i], col[c]))
                           for c in cand], np.float32)
            o = np.lexsort((cand, ex))[:k]
            c = len(o)
            assert np.array_equal(ids[i, :c].astype(np.int64), cand[o]) and np.array_equal(dists[i, :c], ex[o]), (k, i)
            assert np.all(ids[i, c:] == NONE)
    # non-finite query components
    qx = q[:6].copy()
    qx[0, 3] = np.inf
    qx[1, 40] = -np.inf
    qx[2, 7] = np.float32(3e38)
    qx[3, 0] = np.nan
    qx[4, 50] = np.float32(-3e38)
    for k, nprobes in ((10, 1), (10, K), (300, 2)):
        got = ix.search(qx, k=k, nprobes=nprobes)
        _assert_equal(got, _oracle(parts, qx, k, nprobes, metric, 4), ("non-finite", k, nprobes))


def test_pq4_constant_lut_and_the_primitive_on_a_non_finite_table():
    """a zero codebook and a query equal to the centroid give an all-zero L2 LUT: qmax == qmin, the factor is
    255 / 0 and every row ties; the library's 4-bit scan primitive (lb2_pq_scan_4bit) on a table with an Inf
    sub-space and with a NaN entry equals the oracle bit for bit"""
    rng = np.random.default_rng(6800)
    M, ds = 16, 2
    sizes = [250, 4111]
    cent = (rng.standard_normal((2, M * ds)) * 3).astype(np.float32)
    cb = np.zeros((M, 16, ds), np.float32)
    part = np.repeat(np.arange(2, dtype=np.uint32), sizes)
    codes = rng.integers(0, 256, (len(part), M // 2), dtype=np.uint8)
    ix, parts = _open(rng, cent, cb, part, codes, "l2", 4)
    q = cent[[0, 1, 1]].copy()
    for k, nprobes in ((10, 1), (300, 2)):
        got = ix.search(q, k=k, nprobes=nprobes)
        want = _oracle(parts, q, k, nprobes, "l2", 4)
        assert np.all(want[1][:, :min(k, 250)] == 0)
        _assert_equal(got, want, ("constant", k, nprobes))
    n = 4111
    ct = rng.integers(0, 256, (M // 2, n), dtype=np.uint8)
    for metric in ("l2", "dot"):
        for bad in (np.inf, -np.inf, np.nan):
            lut = rng.standard_normal(M * 16).astype(np.float32)
            if np.isnan(bad):
                lut[37] = bad
            else:
                lut[48:64] = bad
            for k_hint in (10, 300):
                got = lb.compute_pq_distance_4bit(lut, M, ct, k_hint, metric)
                want = ob.pq_scan_4bit(lut, ct, n, k_hint, metric)
                same = (got.view(np.uint32) == want.view(np.uint32)) | (np.isnan(got) & np.isnan(want) &
                                                                         (np.signbit(got) == np.signbit(want)))
                assert same.all(), (metric, bad, k_hint, np.flatnonzero(~same)[:5])


def test_pq4_quantisation_rounds_half_away_from_zero():
    """f32::round rounds x.5 away from zero.  Dot with a query of ones and sub-vectors of one dimension gives
    LUT[m][c] = 1 - cb[m][c] exactly; with entries 0, 0.5, 2.5, ..., 26.5 and 63.75, and a first row whose four codes
    all pick 63.75, qmin = 0 and qmax = 255, so the factor is 1 and every half-integer entry sits exactly half-way
    between two u8 levels (2.5 -> 3, where rounding half to even would give 2)."""
    rng = np.random.default_rng(6850)
    M, n = 4, 1000
    v = np.array([0.0, 0.5] + [2.5 + 2 * i for i in range(13)] + [63.75], np.float32)
    cb = np.tile((np.float32(1) - v)[None, :, None], (M, 1, 1)).astype(np.float32)
    codes = rng.integers(0, 15, (n, M // 2), dtype=np.uint8) * np.uint8(17)
    codes = (codes & 0x0F) | (rng.integers(0, 15, (n, M // 2), dtype=np.uint8) << 4)
    codes[0] = 0xFF
    ix, parts = _open(rng, np.zeros((1, M), np.float32), cb, np.zeros(n, np.uint32), codes, "dot", 4)
    q = np.ones((2, M), np.float32)
    lut = lb.build_distance_table_l2(cb, 4, M, q[0], "dot")
    assert np.array_equal(lut, np.tile(v, M))
    assert np.max(ob.pq_scan_4bit(lut, np.ascontiguousarray(codes.T), n, 10, "dot")) == 255 - (M - 1)   # qmax = 255
    for k in (10, 150):
        got = ix.search(q, k=k, nprobes=1)
        _assert_equal(got, _oracle(parts, q, k, 1, "dot", 4), ("half-way", k))


# ---- 5. filters and NaN keys on the exact slot -------------------------------------------------------------------
@pytest.mark.parametrize("metric", ["l2", "dot"])
def test_pq8_prefilter_and_range_on_the_radix_route_match_oracle(metric):
    rng = np.random.default_rng(6900 + len(metric))
    M, ds = 24, 4
    sizes = [0, 33, 513, 4097, 9000]
    K = len(sizes)
    cent, cb, part, data = _model(rng, sizes, M, ds)
    ix, parts = _open(rng, cent, cb, part, _encode(cb, cent, part, data, metric), metric)
    q = _queries(rng, cent, sizes, 12)
    allow = rng.choice(parts["row_ids"], len(part) // 4, replace=False)
    bm = ix.row_mask(allow, None)
    _, d0 = ix.search(q, k=300, nprobes=K)
    lo, hi = float(np.median(d0[:, 3])), float(np.median(d0[:, 250]))
    for k, nprobes in ((16, K), (40, 2), (200, K), (1024, 3)):
        (got, prof) = _profiled(lambda: ix.search_ex(q, k=k, nprobes=nprobes, allow_bitmap=bm, lower_bound=lo,
                                                     upper_bound=hi))
        assert _route(prof) == "radix", prof
        _assert_equal(got, _oracle(parts, q, k, nprobes, metric, allow=allow, lower=lo, upper=hi), (k, nprobes))
        got = ix.search_ex(q, k=k, nprobes=nprobes, allow_bitmap=bm)
        _assert_equal(got, _oracle(parts, q, k, nprobes, metric, allow=allow), ("allow", k, nprobes))


@pytest.mark.parametrize("n_p", [4200, 41])
@pytest.mark.parametrize("kind", ["pq8", "pq4", "flat"])
def test_nan_query_with_the_rows_behind_the_k_th_blocked_keeps_k_rows(kind, n_p):
    """A NaN query: every distance is NaN, whose order key is the one excluded rows carry.  With the rows at positions
    k - 5 .. k of the partition blocked, the k + 1 smallest (key, position) pairs of the slot end in six excluded rows;
    the reference's heap goes on to admitted NaN rows further on.  One partition and one probe, so the slot's list is
    the result: min(k, n_p - 6) rows."""
    rng = np.random.default_rng(7000 + len(kind) + n_p)
    k = 40
    sizes = [n_p]
    if kind == "flat":
        d = 24
        cent = (rng.standard_normal((1, d)) * 3).astype(np.float32)
        part = np.zeros(n_p, np.uint32)
        x = (cent[part] + rng.standard_normal((n_p, d))).astype(np.float32)
        ix = lb.IvfFlatIndex.from_parts(cent, part, x, rng.permutation(n_p).astype(np.uint64) * 2, "l2")
        parts = ix.export()

        def oracle(q, **kw):
            return ob.ivfflat_search(cent, parts["part_offsets"], parts["vectors"], parts["row_ids"], q, k, 1,
                                     nthreads=NT, **kw)
    else:
        nbits = 4 if kind == "pq4" else 8
        cent, cb, part, data = _model(rng, sizes, 12, 2, nbits)
        ix, parts = _open(rng, cent, cb, part, _encode(cb, cent, part, data, "l2", nbits), "l2", nbits)

        def oracle(q, **kw):
            return _oracle(parts, q, k, 1, "l2", nbits, **kw)
    block = parts["row_ids"][k - 5:k + 1]
    bm = ix.row_mask(None, block)
    q = (cent[[0, 0]] + rng.standard_normal((2, cent.shape[1]))).astype(np.float32)
    q[0, 0] = np.nan
    q[1, -1] = np.nan
    got, prof = _profiled(lambda: ix.search_ex(q, k=k, nprobes=1, allow_bitmap=bm))
    assert _ran(prof, "search:flat_scan" if kind == "flat" else "search:pq_scan") == 1, prof
    want = oracle(q, block=block)
    assert list(want[2]) == [min(k, n_p - 6)] * 2, want[2]
    assert [int(np.sum(got[0][i] != NONE)) for i in range(2)] == list(want[2])
    _assert_equal(got, want, kind)


# ---- 6. non-finite queries on the classic and radix routes at M != 16 -------------------------------------------------
@pytest.mark.parametrize("metric", ["l2", "dot"])
def test_pq8_non_finite_queries_on_classic_and_radix_match_oracle(metric):
    rng = np.random.default_rng(7100 + len(metric))
    M, ds = 24, 4
    sizes = [0, 17, 600, 4097, 5000]
    cent, cb, part, data = _model(rng, sizes, M, ds)
    ix, parts = _open(rng, cent, cb, part, _encode(cb, cent, part, data, metric), metric)
    q = _queries(rng, cent, sizes, 8)
    q[0, 5] = np.inf
    q[1, 60] = -np.inf
    q[2, 11] = np.float32(3e38)
    q[3, 90] = np.float32(-3e38)
    q[4, 0] = np.nan
    for k, nprobes, route in ((10, 2, "classic"), (15, len(sizes), "classic"), (100, 3, "radix"), (17, 1, "radix")):
        got, prof = _profiled(lambda: ix.search(q, k=k, nprobes=nprobes))
        assert _route(prof) == route, prof
        _assert_equal(got, _oracle(parts, q, k, nprobes, metric), (metric, k, nprobes))
