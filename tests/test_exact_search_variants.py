"""The exact-distance search kernels against the oracle: the IVF_FLAT scan (`ivfflat_scan_kernel<METRIC, T>`), the
exact re-rank (`refine_kernel<METRIC, T>`, on IVF_PQ and IVF_FLAT indexes) and the per-query merge of the partition
lists (`merge_rank_kernel` up to MERGE_RANK_MAX = 2048 candidates, `merge_kernel` above).

Indexes are opened with `from_parts`, so every partition has exactly the size a case needs.  Which path a case takes
follows from its numbers (SCAN_CHUNK = 4096 rows per scan chunk; k + 1 candidates are kept per list):
  * a probed partition of n_p > 4096 rows is scanned in ceil(n_p / 4096) chunks and carries its winners across them;
  * the k-th and (k + 1)-th candidates of a list tied -> the list is replayed through the reference's heap;
  * min(nprobes, K) * k <= 2048 -> merge_rank_kernel, otherwise merge_kernel;
  * d % 16 != 0 -> the sequential tail of the distance (all of it when d < 16).

L2 and dot are compared BIT FOR BIT with the oracle on the values the reference sees (16-bit rows converted to f32,
as FlatFloatStorage does, flat/storage.rs:352-365).  Cosine is compared with an f64 evaluation under a derived error
bound (`_cosine_bound`)."""
import math

import numpy as np
import pytest

import lance_b200 as lb
from oracle import binding as ob

pytestmark = pytest.mark.gpu
NT = 16
SCAN_CHUNK = 4096
MERGE_RANK_MAX = 2048


# ---- element types ---------------------------------------------------------------------------------------------
def _bf16_bits(x):
    """f32 -> bfloat16 bit patterns (uint16), round to nearest even; NaN stays a quiet NaN."""
    b = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    r = ((b + 0x7FFF + ((b >> 16) & 1)) >> 16).astype(np.uint16)
    return np.where(np.isnan(x), np.uint16(0x7FC0), r)


def _bf16_f32(bits):
    return (np.asarray(bits, dtype=np.uint32) << 16).view(np.float32)


def _native(x, dt):
    """f32 values -> the column's element type (bf16 as uint16 bit patterns)."""
    if dt == "f16":
        return x.astype(np.float16)
    if dt == "bf16":
        return _bf16_bits(x)
    return x.astype(np.float32)


def _f32(a, dt):
    """the exact f32 value of every element of a native array"""
    return _bf16_f32(a) if dt == "bf16" else np.asarray(a).astype(np.float32)


def _flat_index(rng, sizes, d, dt, metric, spread=4.0, noise=1.0, row_scale=None):
    """IVF_FLAT index whose partition p holds exactly sizes[p] rows, rows in partition order.  Row ids are the row
    numbers of the returned `data` (the native column), so the same array serves as refine vectors."""
    K = len(sizes)
    cent = (rng.standard_normal((K, d)) * spread).astype(np.float32)
    part = np.repeat(np.arange(K, dtype=np.uint32), sizes)
    n = len(part)
    x = cent[part] + rng.standard_normal((n, d)).astype(np.float32) * noise
    if row_scale is not None:  # rows of different norms (cosine divides them out)
        x *= rng.uniform(*row_scale, size=(n, 1)).astype(np.float32)
    data = _native(x, dt)
    cent_n = _native(cent, dt)
    ix = lb.IvfFlatIndex.from_parts(cent_n, part, data, np.arange(n, dtype=np.uint64), metric, bf16=(dt == "bf16"))
    parts = ix.export()
    assert np.array_equal(np.diff(parts["part_offsets"].astype(np.int64)), sizes)
    return ix, parts, data, _f32(cent_n, dt)


def _oracle_flat(parts, cent32, dt, q32, k, nprobes, metric, **kw):
    return ob.ivfflat_search(cent32, parts["part_offsets"], _f32(parts["vectors"], dt), parts["row_ids"], q32, k,
                             nprobes, metric=metric, nthreads=NT, **kw)


def _assert_equal(got, want, what):
    ids, dists = got
    oi, od = want[0], want[1]
    for i in range(len(oi)):
        if not (np.array_equal(ids[i], oi[i]) and np.array_equal(dists[i], od[i], equal_nan=True)):
            r = next(j for j in range(len(oi[i])) if ids[i, j] != oi[i, j] or not
                     (dists[i, j] == od[i, j] or (np.isnan(dists[i, j]) and np.isnan(od[i, j]))))
            raise AssertionError(f"{what}: query {i}, rank {r}: got ({ids[i, r]}, {dists[i, r]!r}), "
                                 f"want ({oi[i, r]}, {od[i, r]!r})")


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


# ---- 1. IVF_FLAT scan: element types x L2 / dot, dimension tails, chunk boundaries ------------------------------
SIZES = [0, 1, 15, 16, 17, 4095, 4096, 4097, 8193, 12003]   # K = 10
# IVF_FLAT takes d % 4 == 0 (lb2_index_load_flat); the tails: d % 16 = 4, 8, 12, and d < 16 (tail only)
FLAT_CASES = ([("f32", d) for d in (4, 8, 20, 100, 140)] + [("f16", d) for d in (8, 28, 132)]
              + [("bf16", d) for d in (4, 100, 1536)])


@pytest.mark.parametrize("metric", ["l2", "dot"])
@pytest.mark.parametrize("dt,d", FLAT_CASES, ids=[f"{t}-d{d}" for t, d in FLAT_CASES])
def test_ivf_flat_scan_matches_oracle_bit_for_bit(dt, d, metric):
    rng = np.random.default_rng(5100 + d + 7 * len(dt) + (metric == "dot"))
    sizes = SIZES if d < 1536 else [0, 17, 4097, 5000]
    K = len(sizes)
    ix, parts, data, cent32 = _flat_index(rng, sizes, d, dt, metric, noise=1.0 if metric == "l2" else 0.5)
    big = [p for p, s in enumerate(sizes) if s > SCAN_CHUNK]
    nq = 14
    q32 = cent32[rng.choice(big, nq)] + rng.standard_normal((nq, d)).astype(np.float32)   # near multi-chunk lists
    q32[nq // 2:] = cent32[rng.integers(0, K, nq - nq // 2)] + rng.standard_normal((nq - nq // 2, d)).astype(np.float32)
    q32[nq - 2, 0] = np.nan                        # every distance NaN: ties everywhere, the heap replay decides
    q32[nq - 1, d // 2] = np.inf                   # L2: +Inf everywhere; dot: +-Inf by the sign of the row element
    if metric == "l2":
        q32[nq - 1, 0] = -np.inf
    qn = _native(q32, dt)
    q32 = _f32(qn, dt)
    cases = [(1, 1), (15, 3), (16, K), (100, K + 5), (1024, 2)]   # (k, nprobes): k + 1 <= 16 and > 16; np*k vs 2048
    for k, nprobes in cases:
        got, prof = _profiled(lambda: ix.search(qn, k=k, nprobes=nprobes))
        _assert_equal(got, _oracle_flat(parts, cent32, dt, q32, k, nprobes, metric), (dt, d, metric, k, nprobes))
        assert _ran(prof, "search:flat_scan") == 1 and _ran(prof, "search:merge_topk") == 1, prof
    # prefilter and range over the multi-chunk lists; k larger than the allowed rows
    fin = q32[: nq - 2]
    fq = qn[: nq - 2]
    allow = rng.choice(parts["row_ids"][parts["part_offsets"][big[0]]:], 40, replace=False)
    bm = ix.row_mask(allow, None)
    for k, nprobes in ((10, K), (100, K)):
        got = ix.search_ex(fq, k=k, nprobes=nprobes, allow_bitmap=bm)
        _assert_equal(got, _oracle_flat(parts, cent32, dt, fin, k, nprobes, metric, allow=allow), ("allow", k))
    _, d0 = ix.search(fq, k=40, nprobes=K)
    lo, hi = float(np.median(d0[:, 3])), float(np.median(d0[:, 30]))
    for k in (5, 64):
        got = ix.search_ex(fq, k=k, nprobes=K, lower_bound=lo, upper_bound=hi)
        _assert_equal(got, _oracle_flat(parts, cent32, dt, fin, k, K, metric, lower=lo, upper=hi), ("range", k))
        got = ix.search_ex(fq, k=k, nprobes=K, allow_bitmap=bm, lower_bound=lo, upper_bound=hi)
        _assert_equal(got, _oracle_flat(parts, cent32, dt, fin, k, K, metric, allow=allow, lower=lo, upper=hi),
                      ("allow+range", k))


@pytest.mark.parametrize("metric", ["l2", "dot"])
def test_ivf_flat_ties_straddling_chunk_boundaries_go_through_the_replay(metric):
    """Copies of one row sit at storage positions 4090..4101 and 8188..8192 of a 8193-row partition (chunks
    [0, 4096), [4096, 8192), [8192, 8193)).  A query equal to that row ties all 17 copies at the best distance, so
    for k < 17 the k-th and (k + 1)-th candidates tie and the list is replayed through the reference's heap, whose
    result depends on rows of every chunk."""
    rng = np.random.default_rng(5200 + (metric == "dot"))
    d, sizes = 40, [3000, 8193, 5000]
    cent = (rng.standard_normal((3, d)) * 3).astype(np.float32)
    part = np.repeat(np.arange(3, dtype=np.uint32), sizes)
    x = (cent[part] + rng.standard_normal((len(part), d))).astype(np.float32)
    if metric == "dot":
        x /= np.linalg.norm(x, axis=1, keepdims=True)
    dup = x[3000 + 100].copy()
    pos = np.r_[4090:4102, 8188:8193]
    x[3000 + pos] = dup
    rid = rng.permutation(len(part)).astype(np.uint64) * 3 + 1
    ix = lb.IvfFlatIndex.from_parts(cent, part, x, rid, metric)
    parts = ix.export()
    stored = parts["vectors"][3000:3000 + 8193]
    assert np.array_equal(np.flatnonzero((stored == dup).all(1)), np.union1d(pos, [100]))
    q = np.stack([dup, dup, dup + np.float32(1e-3), cent[1]])
    for k, nprobes in ((1, 1), (5, 1), (12, 2), (16, 3), (17, 1), (40, 3)):
        got = ix.search(q, k=k, nprobes=nprobes)
        _assert_equal(got, _oracle_flat(parts, cent, "f32", q, k, nprobes, metric), (metric, k, nprobes))


# ---- 2. cosine against an f64 evaluation ------------------------------------------------------------------------
def _cosine_bound(q, y):
    """Error bound of the device's cosine distance 1 - <q, y> / |q| / sqrt(<y, y>) for f32 inputs q, y of length d.

    <q, y> and <y, y> are each a 16-lane FMA chain of ceil(d / 16) steps followed by a 4-level shuffle tree, and |q|
    is the same chain over q: every product term passes through at most n = ceil(d / 16) + log2(16) roundings, so
    (Higham, eq. 3.5) |<q, y>~ - <q, y>| <= g_n S |q||y| with S = sum|q_i y_i| / (|q||y|) <= 1 and g_n = n u / (1 - n u),
    u = 2^-24, and both squared norms carry a relative error <= g_n.  A square root halves a relative error and adds
    u; each of the two divisions adds u.  The ratio r = <q, y> / (|q||y|) therefore has
        |r~ - r| <= (g_n + g_n / 2 + g_n / 2 + 4u) S + O(u^2) <= 3 n u S   (n >= 4),
    and the final 1 - r~ (a value in [0, 2]) adds at most half an ulp of a number below 2, i.e. u.  Bound:
        B = 3 (ceil(d / 16) + 4) 2^-24 S + 2^-24,
    2.2e-6 at d = 128 even when S = 1, against the 1e-5 the old tolerance check allowed."""
    d = q.shape[-1]
    q64, y64 = q.astype(np.float64), y.astype(np.float64)
    s = (np.abs(q64 * y64).sum(-1)) / (np.linalg.norm(q64, axis=-1) * np.linalg.norm(y64, axis=-1))
    return 3.0 * (math.ceil(d / 16) + 4) * 2.0 ** -24 * s + 2.0 ** -24


def _cosine64(q, y):
    q64, y64 = q.astype(np.float64), y.astype(np.float64)
    return 1.0 - (q64 * y64).sum(-1) / (np.linalg.norm(q64, axis=-1) * np.linalg.norm(y64, axis=-1))


def _check_cosine(ids, dists, cand, q, rows_of, k, what):
    """ids / dists: the device's top-k of one query; cand: every row id it chose from; rows_of(ids) -> f32 rows."""
    c = int(np.sum(ids != np.uint64(~np.uint64(0))))
    assert c == min(k, len(cand)), (what, c)
    if c == 0:
        return
    ids, dists = ids[:c].astype(np.int64), dists[:c].astype(np.float64)
    ex = _cosine64(q, rows_of(ids))
    bnd = _cosine_bound(q, rows_of(ids))
    assert np.all(np.abs(dists - ex) <= bnd), (what, np.max(np.abs(dists - ex) / bnd))
    # ascending by (distance, id)
    assert all(dists[i] < dists[i + 1] or (dists[i] == dists[i + 1] and ids[i] < ids[i + 1]) for i in range(c - 1)), what
    # the ids are the f64 top-k except where the f64 distance is within twice the bound of the k-th
    cand = np.asarray(cand, np.int64)
    all_ex = _cosine64(q, rows_of(cand))
    order = np.lexsort((cand, all_ex))
    kth = all_ex[order[c - 1]]
    b2 = 2 * float(np.max(_cosine_bound(q, rows_of(cand))))
    must = set(cand[all_ex < kth - b2].tolist())
    assert must <= set(ids.tolist()), (what, sorted(must - set(ids.tolist()))[:5])
    assert np.all(ex <= kth + b2), what


def test_cosine_bound_is_tight():
    d = 128
    assert 3.0 * (math.ceil(d / 16) + 4) * 2.0 ** -24 + 2.0 ** -24 < 2.3e-6   # S <= 1 by Cauchy-Schwarz
    # the oracle's own f32 cosine (scalar form) stays inside the bound too
    rng = np.random.default_rng(5300)
    q, y = rng.standard_normal((2, 64, d)).astype(np.float32)
    got = np.array([ob.cosine(q[i], y[i]) for i in range(64)], np.float64)
    assert np.all(np.abs(got - _cosine64(q, y)) <= _cosine_bound(q, y))


@pytest.mark.parametrize("dt,d", [("f32", 128), ("f32", 140), ("f16", 128), ("f16", 36)])
def test_ivf_flat_cosine_within_bound_of_f64(dt, d):
    rng = np.random.default_rng(5400 + d)
    sizes = [700, 4097, 0, 9000, 31, 2500]
    K = len(sizes)
    ix, parts, data, cent32 = _flat_index(rng, sizes, d, dt, "cosine", row_scale=(0.25, 4.0))
    stored = _f32(parts["vectors"], dt)
    pos_of = np.empty(len(stored), np.int64)
    pos_of[parts["row_ids"].astype(np.int64)] = np.arange(len(stored))
    nq = 10
    qn = _native(cent32[rng.choice([1, 3], nq)] * 0.5 + rng.standard_normal((nq, d)).astype(np.float32), dt)
    q32 = _f32(qn, dt)
    qnorm = ob.normalize_rows(q32)                 # the device's normalise is bit-identical to this one
    off = parts["part_offsets"].astype(np.int64)
    for k, nprobes in ((10, 1), (100, 3), (1024, K)):
        (ids, dists), prof = _profiled(lambda: ix.search(qn, k=k, nprobes=nprobes))
        assert _ran(prof, "search:flat_scan") == 1
        for i in range(nq):
            pids, _ = ob.find_partitions(cent32, qnorm[i], nprobes)
            cand = np.concatenate([parts["row_ids"][off[p]:off[p + 1]] for p in pids]).astype(np.int64)
            _check_cosine(ids[i], dists[i], cand, qnorm[i], lambda r: stored[pos_of[r]], k, (dt, d, k, nprobes, i))


# ---- 3. refine ---------------------------------------------------------------------------------------------------
def _exact(metric, dt, q, v):
    """the distance the refine plan computes for key type dt (flat.rs:94-150); None for cosine (f64 bound)"""
    one = np.float32(1.0)
    if dt == "f32":
        return ob.l2(q, v) if metric == "l2" else one - np.float32(ob.dot(q, v))
    if dt == "f16":
        return ob.l2_f16(q, v) if metric == "l2" else one - np.float32(ob.dot_f16(q, v))
    if dt == "bf16":   # the reference has no bf16 arm; the product evaluates the f32 values (as its IVF_FLAT scan)
        return ob.l2_bf16(q, v) if metric == "l2" else one - np.float32(ob.dot(_bf16_f32(q), _bf16_f32(v)))
    return ob.l2_u8(q, v) if metric == "l2" else one - np.float32(ob.dot_u8(q, v))


def _rerank(metric, dt, q, vectors, cand, k, lower=None, upper=None):
    """exact re-rank of one query's candidates: ascending (distance, id), rows beyond `vectors` -> NaN, range after"""
    ex = np.array([_exact(metric, dt, q, vectors[c]) if c < len(vectors) else np.nan for c in cand], np.float32)
    keep = np.ones(len(cand), bool)
    if lower is not None:
        keep &= ex >= np.float32(lower)
    if upper is not None:
        keep &= ex < np.float32(upper)
    cand, ex = cand[keep], ex[keep]
    order = np.lexsort((cand, ex))[:k]
    return cand[order], ex[order]


def _check_refine(ids, dists, want, k, what):
    wi, wd = want
    c = len(wi)
    assert np.array_equal(ids[:c].astype(np.int64), wi) and np.array_equal(dists[:c], wd, equal_nan=True), (
        what, next((j, ids[j], dists[j], wi[j], wd[j]) for j in range(c) if ids[j] != wi[j] or
                   not (dists[j] == wd[j] or np.isnan(dists[j]) and np.isnan(wd[j]))))
    assert np.all(ids[c:] == np.uint64(~np.uint64(0))) and np.all(np.isinf(dists[c:])), what


def _pq_index(rng, data, metric, K=16):
    ix = lb.IvfPqIndex.build(data, metric, lb.IvfBuildParams(num_partitions=K, num_sub_vectors=16, max_iters=5,
                                                             pq_max_iters=4))
    return ix, ix.export()


def _pq_candidates(parts, q32, kc, nprobes, metric, **kw):
    oi, _, oc = ob.ivfpq_search(parts["centroids"], parts["codebook"], parts["part_offsets"], parts["codes"],
                                parts["row_ids"], q32, kc, nprobes, metric=metric, nthreads=NT, **kw)
    return [oi[i, :oc[i]].astype(np.int64) for i in range(len(q32))]


REFINE_SIZES = ((10, 1), (100, 10), (64, 16), (1024, 1))    # (k, refine_factor): k * rf = k, 1000, 1024, 1024


@pytest.mark.parametrize("metric", ["l2", "dot", "cosine"])
def test_refine_f32_on_ivf_pq(metric):
    rng = np.random.default_rng(5500 + len(metric))
    n, d = 24000, 128
    cent = (rng.standard_normal((24, d)) * 3).astype(np.float32)
    data = (cent[rng.integers(0, 24, n)] + rng.standard_normal((n, d))).astype(np.float32)
    data *= rng.uniform(0.5, 2.0, (n, 1)).astype(np.float32)
    ix, parts = _pq_index(rng, data, metric)
    q = (data[rng.choice(n, 12, replace=False)] + rng.standard_normal((12, d)) * 0.3).astype(np.float32)
    for k, rf in REFINE_SIZES:
        nprobes = 4
        (ids, dists), prof = _profiled(lambda: ix.search_refine(data, q, k=k, nprobes=nprobes, refine_factor=rf))
        assert _ran(prof, "search:refine") == 1, prof
        cands = _pq_candidates(parts, q, k * rf, nprobes, metric)
        for i in range(len(q)):
            if metric == "cosine":
                _check_cosine(ids[i], dists[i], cands[i], q[i], lambda r: data[r], k, (k, rf, i))
            else:
                _check_refine(ids[i], dists[i], _rerank(metric, "f32", q[i], data, cands[i], k), k, (metric, k, rf, i))
    # range bounds: the index search applies them to the PQ distances (flat/index.rs:100-115), and the plan filters
    # the exact distances again after the re-rank (scanner.rs:3342-3377)
    k, rf = 10, 20
    _, d0 = ix.search_refine(data, q, k=40, nprobes=4, refine_factor=5)
    lo, hi = float(np.median(d0[:, 2])), float(np.median(d0[:, 25]))
    ids, dists = ix.search_ex(q, k=k, nprobes=4, refine_factor=rf, vectors=data, lower_bound=lo, upper_bound=hi)
    cands = _pq_candidates(parts, q, k * rf, 4, metric, lower=lo, upper=hi)
    for i in range(len(q)):
        if metric != "cosine":
            _check_refine(ids[i], dists[i], _rerank(metric, "f32", q[i], data, cands[i], k, lo, hi), k, ("range", i))
            continue
        c = int(np.sum(np.isfinite(dists[i])))
        got, gd = ids[i][:c].astype(np.int64), dists[i][:c].astype(np.float64)
        assert set(got.tolist()) <= set(cands[i].tolist()) and np.all((gd >= np.float32(lo)) & (gd < np.float32(hi)))
        assert np.all(np.abs(gd - _cosine64(q[i], data[got])) <= _cosine_bound(q[i], data[got])), i
        assert all(gd[j] < gd[j + 1] or (gd[j] == gd[j + 1] and got[j] < got[j + 1]) for j in range(c - 1)), i
        if len(cands[i]) == 0:    # no candidate in range at all
            continue
        ex = _cosine64(q[i], data[cands[i]])
        b2 = 2 * float(np.max(_cosine_bound(q[i], data[cands[i]])))
        top = gd[-1] if c == k else hi
        sure = cands[i][(ex >= lo + b2) & (ex < min(hi, top) - b2)]
        assert set(sure.tolist()) <= set(got.tolist()), ("cosine range", i)


REFINE_FLAT = [("f32", "l2", 96), ("f32", "dot", 100), ("f16", "l2", 132), ("f16", "dot", 132), ("f16", "dot", 64),
               ("bf16", "l2", 100), ("bf16", "dot", 132), ("u8", "l2", 128), ("u8", "l2", 1536), ("u8", "dot", 128)]


@pytest.mark.parametrize("dt,metric,d", REFINE_FLAT, ids=[f"{t}-{m}-d{d}" for t, m, d in REFINE_FLAT])
def test_refine_element_types_on_ivf_flat(dt, metric, d):
    """f16 dot is the reference's 32-lane dot_scalar (dot.rs:133); u8 sums are exact integers (l2.rs:44-49,
    dot.rs:152-161): at d = 1536 with rows spread over 0..255 an f32 sum of the squares would round."""
    rng = np.random.default_rng(5600 + d + len(dt) + (metric == "dot"))
    sizes = [3, 1500, 0, 5000, 2, 2600] if d < 1536 else [3, 900, 1200]
    K = len(sizes)
    if dt == "u8":
        part = np.repeat(np.arange(K, dtype=np.uint32), sizes)
        lvl = rng.integers(0, 256, (K, d))
        data = np.clip(lvl[part] + rng.integers(-60, 61, (len(part), d)), 0, 255).astype(np.uint8)
        cent = lvl.astype(np.float32)
        ix = lb.IvfFlatIndex.from_parts(cent, part, data, np.arange(len(part), dtype=np.uint64), metric)
        parts = ix.export()
        qn = np.where(rng.random((8, d)) < 0.5, 0, 255).astype(np.uint8)   # far from every row: large sums
        qn[:4] = np.clip(lvl[rng.integers(0, K, 4)] + rng.integers(-20, 21, (4, d)), 0, 255)
        q32 = qn.astype(np.float32)
        vec32 = parts["vectors"]
    else:
        ix, parts, data, cent = _flat_index(rng, sizes, d, dt, metric, noise=1.0 if metric == "l2" else 0.5)
        qn = _native(cent[rng.integers(0, K, 8)] + rng.standard_normal((8, d)).astype(np.float32), dt)
        q32 = _f32(qn, dt)
        vec32 = _f32(parts["vectors"], dt)
    if dt == "u8" and metric == "l2" and d == 1536:   # the case is one where f32 accumulation is not exact
        v0 = data[:64].astype(np.float32)
        f32_sums = np.array([ob.l2(q32[5], r) for r in v0])
        assert np.any(f32_sums != np.array([ob.l2_u8(qn[5], r) for r in data[:64]], np.float32))
    for k, rf in ((10, 1), (10, 100), (1024, 1), (20, 3)):
        nprobes = 2
        (ids, dists), prof = _profiled(lambda: ix.search_refine(data, qn, k=k, nprobes=nprobes, refine_factor=rf))
        assert _ran(prof, "search:refine") == 1 and _ran(prof, "search:flat_scan") == 1, prof
        oi, _, oc = ob.ivfflat_search(cent, parts["part_offsets"], vec32, parts["row_ids"], q32, k * rf, nprobes,
                                      metric=metric, nthreads=NT)
        for i in range(len(qn)):
            cand = oi[i, :oc[i]].astype(np.int64)
            _check_refine(ids[i], dists[i], _rerank(metric, dt, qn[i], data, cand, k), k, (dt, metric, d, k, rf, i))
    if dt == "u8" and metric == "l2":   # the same numbers as the library's u8 L2 primitive (lb2_distance_batch)
        for i in (0, 5):
            ok = ids[i] != np.uint64(~np.uint64(0))
            assert np.array_equal(lb.l2_distance_batch(qn[i], data[ids[i][ok].astype(np.int64)], d), dists[i][ok]), i


def test_refine_cosine_on_ivf_flat_and_short_lists():
    """cosine re-rank of an IVF_FLAT index's own candidates under the f64 bound; queries whose single probed
    partition holds fewer than k rows return what there is, then (~0, +Inf) slots"""
    rng = np.random.default_rng(5700)
    d, sizes = 100, [3, 2000, 5, 4500]
    ix, parts, data, cent = _flat_index(rng, sizes, d, "f32", "cosine", row_scale=(0.3, 3.0))
    q = (cent[[1, 3, 1, 3, 0, 2]] + rng.standard_normal((6, d))).astype(np.float32)
    for k, rf in ((10, 1), (50, 20), (8, 128)):
        kc = k * rf
        ci, _ = ix.search(q, k=kc, nprobes=2)          # the scan's own candidates (what refine re-ranks)
        ids, dists = ix.search_refine(data, q, k=k, nprobes=2, refine_factor=rf)
        for i in range(len(q)):
            cand = ci[i][ci[i] != np.uint64(~np.uint64(0))].astype(np.int64)
            _check_cosine(ids[i], dists[i], cand, q[i], lambda r: data[r], k, (k, rf, i))
    # short lists: query 4 / 5 probe only the 3-row / 5-row partition
    for metric in ("l2", "dot"):
        ix2, parts2, data2, cent2 = _flat_index(rng, sizes, d, "f32", metric)
        qs = cent2[[0, 2]] + np.float32(0.01)
        ids, dists = ix2.search_refine(data2, qs, k=10, nprobes=1, refine_factor=3)
        oi, _, oc = ob.ivfflat_search(cent2, parts2["part_offsets"], parts2["vectors"], parts2["row_ids"], qs, 30, 1,
                                      metric=metric)
        assert list(oc) == [3, 5]
        for i in range(2):
            cand = oi[i, :oc[i]].astype(np.int64)
            _check_refine(ids[i], dists[i], _rerank(metric, "f32", qs[i], data2, cand, 10), 10, (metric, i))


@pytest.mark.parametrize("metric", ["l2", "dot"])
def test_refine_with_vectors_shorter_than_the_row_ids(metric):
    """A candidate id >= len(vectors) has no row to read: refine_kernel gives it a NaN distance (the quiet NaN
    0x7FC00000), which the (distance, id) order of the f32 total order puts after every number, so such ids are
    returned only when the list has nothing else, ascending by id among themselves."""
    rng = np.random.default_rng(5800 + (metric == "dot"))
    n, d = 20000, 64
    data = (rng.standard_normal((n, d)) + rng.integers(0, 4, (n, 1))).astype(np.float32)
    ix, parts = _pq_index(rng, data, metric, K=8)
    q = data[rng.choice(n, 8, replace=False)] + np.float32(0.05)
    short = data[: n // 40]
    for k, rf in ((10, 4), (100, 10)):
        ids, dists = ix.search_refine(short, q, k=k, nprobes=3, refine_factor=rf)
        cands = _pq_candidates(parts, q, k * rf, 3, metric)
        for i in range(len(q)):
            want = _rerank(metric, "f32", q[i], short, cands[i], k)
            _check_refine(ids[i], dists[i], want, k, (k, rf, i))
            nan = np.isnan(dists[i])
            assert np.all(ids[i][nan] >= len(short)) and np.all(dists[i][nan].view(np.uint32) == 0x7FC00000)
        assert np.isnan(dists).any() and not np.isnan(dists).all()


# ---- 4. merge: both sides of MERGE_RANK_MAX, ties across lists ----------------------------------------------------
def test_merge_both_sides_of_the_rank_limit_with_ties_across_lists():
    """K = 20 non-empty partitions; one row is copied into every partition (distinct ids), so a query equal to it
    sees equal distances in every list, ordered by row id alone.  min(nprobes, K) * k = 2040 and 2048 merge by rank
    counting, 2049 and 3072 by the k-round argmin."""
    rng = np.random.default_rng(5900)
    d, K, per = 24, 20, 1100
    cent = (rng.standard_normal((K, d)) * 0.6).astype(np.float32)
    part = np.repeat(np.arange(K, dtype=np.uint32), per)
    x = (cent[part] + rng.standard_normal((len(part), d))).astype(np.float32)
    x = np.round(x * 2) / 2                       # a half-integer grid: many more equal distances across lists
    dup = x[0].copy()
    x[np.arange(K) * per + 7] = dup
    rid = rng.permutation(len(part)).astype(np.uint64)
    ix = lb.IvfFlatIndex.from_parts(cent, part, x, rid, "l2")
    parts = ix.export()
    q = np.concatenate([dup[None], dup[None] + np.float32(0.5), np.round(cent[rng.integers(0, K, 6)] * 2) / 2])
    q = q.astype(np.float32)
    for k, nprobes, kernel in ((102, 20, "rank"), (128, 16, "rank"), (1024, 2, "rank"), (683, 3, "argmin"),
                               (1024, 3, "argmin"), (150, 25, "argmin")):
        assert (min(nprobes, K) * k > MERGE_RANK_MAX) == (kernel == "argmin")
        (ids, dists), prof = _profiled(lambda: ix.search(q, k=k, nprobes=nprobes))
        assert _ran(prof, "search:merge_topk") == 1
        _assert_equal((ids, dists), _oracle_flat(parts, cent, "f32", q, k, nprobes, "l2"), (k, nprobes))
        # the row copied into every probed partition: all copies at distance 0, ascending by id
        got0 = ids[0][dists[0] == 0]
        assert len(got0) >= min(nprobes, K) and np.all(np.diff(got0.astype(np.int64)) > 0)
