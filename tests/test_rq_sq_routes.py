"""Every route of the IVF_RQ scan, rotation and transform, and the slab and chunk paths of IVF_SQ and IVF_RQ, against
the restatements of the reference (tests/rq_reference.py, tests/sq_reference.py), bit for bit: ids, distance bits
and counts, ties at the k-th distance included.

The routes and how each case shows that it ran:
  - the scan's 16-bit table sums, which wrap mod 2^16 once a row's sum passes 65 535 (code_dim above 1028): the
    restatement counts the rows whose unwrapped sum exceeds 0xFFFF;
  - code widths from one sub-table to the shared-memory limit, and one step past it (LB2_UNSUPPORTED);
  - the rotation groups of ivfrq_search_f32 ((query, probe) residuals rotated ~256 MB at a time) and the
    32 768-query slabs of ivf_search: `rq_scan` / `sq_scan` launch counts;
  - row chunks (LB2_CHUNK_ROWS), host rows streamed through the staging slots (LB2_MAX_RESIDENT_MB) and the
    transform's code_dim-bounded sub-chunks: `rq_rotate` / `sq_encode` / `stage_rows` launch counts;
  - the Householder rotation past one 256-thread reduction, and the scan's numeric edges (flat tables, 2^+-40
    queries, factors that overflow to +-inf, -0.0 residual components)."""
import numpy as np
import pytest

import lance_b200 as lb
from oracle import binding as ob
from rq_reference import dist_table, dot16, ivfrq_search, pack_signs, quantize_table, rq_transform
from sq_reference import ivfsq_search, sq_bounds, sq_encode

pytestmark = pytest.mark.gpu

U64MAX = np.iinfo(np.uint64).max
SLAB = 32768                          # queries per scan launch (ivf_search, ivf_search.cu)
GROUP_BYTES = 256 << 20               # ivfrq_search_f32 rotates (query, probe) residuals ~256 MB at a time
SIZES = (0, 31, 32, 33, 4097)         # every probed partition: none, tail only, 32-row blocks, both, past 4096 rows


# ---- helpers -----------------------------------------------------------------------------------------------------
def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _same(got, want):
    """ids, distance bits and counts exactly; past the count, the empty marker (row id ~0, distance +inf)"""
    (gi, gd), (wi, wd, wc) = got, want
    assert gi.shape == wi.shape
    for i in range(wi.shape[0]):
        c = int(wc[i])
        assert np.array_equal(gi[i, :c], wi[i, :c]), i
        assert np.array_equal(_bits(gd[i, :c]), _bits(wd[i, :c])), i
        assert (gi[i, c:] == U64MAX).all() and np.isposinf(gd[i, c:]).all(), i


def _same_arrays(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    if a.dtype != b.dtype or a.shape != b.shape:
        return False
    if a.dtype.kind == "f":
        a, b = a.view(f"u{a.dtype.itemsize}"), b.view(f"u{b.dtype.itemsize}")
    return np.array_equal(a, b)


def _profiled(fn):
    lb.profile.enable(True)
    lb.profile.reset()
    try:
        fn()
    finally:
        lb.profile.enable(False)
    return lb.profile.dump()


def _launches(prof, name):
    """launches of `name` under any tag ("search:rq_scan", "transform:rq_rotate", ...)"""
    return sum(v[0] for key, v in prof.items() if key.split(":")[-1] == name)


def _knobs(monkeypatch, chunk=None, resident_mb=None):
    for name, v in (("LB2_CHUNK_ROWS", chunk), ("LB2_MAX_RESIDENT_MB", resident_mb)):
        if v is None:
            monkeypatch.delenv(name, raising=False)
        else:
            monkeypatch.setenv(name, str(v))


def _status(call):
    with pytest.raises(lb.LanceB200Error) as e:
        call()
    return e.value.status


def _rotation(cd, d, rng):
    """a full [code_dim][code_dim] matrix; the transform and the scan read its first d columns"""
    if cd == d:
        return rng.standard_normal((cd, cd), dtype=np.float32)
    r = np.zeros((cd, cd), np.float32)
    r[:, :d] = rng.standard_normal((cd, d), dtype=np.float32)
    return r


def _rq_index(d, nb, metric, sizes=SIZES, seed=0, rot=None, cent=None, codes=None, add=None, scale=None):
    """from_parts at exact partition sizes.  Codes, factors and rotation are random unless given: the scan's
    arithmetic is bit-exact for any inputs.  -> (index, the restatement's CSR arrays in storage order)"""
    rng = np.random.default_rng(seed)
    K, cd = len(sizes), d * nb
    n = int(sum(sizes))
    if cent is None:
        cent = rng.standard_normal((K, d), dtype=np.float32)
        if metric == "cosine":
            cent = ob.normalize_rows(cent)
    rot = _rotation(cd, d, rng) if rot is None else rot
    part = np.repeat(np.arange(K, dtype=np.uint32), sizes)
    codes = rng.integers(0, 256, (n, cd // 8), dtype=np.uint8) if codes is None else codes
    add = rng.uniform(0.5, 4.0, n).astype(np.float32) if add is None else add
    scale = rng.standard_normal(n, dtype=np.float32) if scale is None else scale
    perm = rng.permutation(n)                                    # rows arrive unsorted; the load groups them
    rid = rng.permutation(n).astype(np.uint64)
    ix = lb.IvfRqIndex.from_parts(cent, rot, part[perm], codes[perm], add[perm], scale[perm], rid[perm], metric,
                                  num_bits=nb)
    offs = np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint64)
    order = perm[np.argsort(part[perm], kind="stable")]         # the storage order the load produces
    return ix, (cent, rot, offs, codes[order], add[order], scale[order], rid[order])


def _wrapped_rows(m, queries, nprobes, metric):
    """(rows of the probed partitions whose unwrapped u8 table sum exceeds 0xFFFF, quantised rows scanned)"""
    cent, rot, offs, codes = m[:4]
    K, d = cent.shape
    R = np.ascontiguousarray(rot[:, :d])
    q = ob.normalize_rows(queries) if metric == "cosine" else np.ascontiguousarray(queries, np.float32)
    wrapped = total = 0
    for qi in q:
        pids, _ = ob.find_partitions(cent, qi, min(nprobes, K), metric="dot" if metric == "dot" else "l2")
        for p, rq in zip(pids, dot16(qi[None, :] - cent[pids], R)):
            a, b = int(offs[p]), int(offs[p + 1])
            nq = (b - a) - (b - a) % 32
            if nq == 0:
                continue
            qt = quantize_table(dist_table(rq))[2].astype(np.int64)
            c = codes[a:a + nq]
            i2 = np.arange(c.shape[1])
            s = (qt[2 * i2, c & 15] + qt[2 * i2 + 1, c >> 4]).sum(axis=1)
            wrapped += int((s > 0xFFFF).sum())
            total += nq
    return wrapped, total


# ---- 1. scan code widths -----------------------------------------------------------------------------------------
# code_dim -> (d, num_bits); the real embedding shapes d = 1536 / 3072 at one bit, the others from d = 8 or 16
WIDTHS = {8: (8, 1), 24: (24, 1), 40: (40, 1), 1024: (16, 64), 1032: (8, 129), 1536: (1536, 1), 2048: (16, 128),
          3072: (3072, 1), 4096: (16, 256), 8192: (16, 512)}
SEARCHES = ((1, 5), (10, 2), (100, 5), (1024, 5), (1024, 3))    # (k, nprobes); K = 5


@pytest.mark.parametrize("metric", ["l2", "cosine", "dot"])
@pytest.mark.parametrize("cd", list(WIDTHS))
def test_scan_code_widths(cd, metric):
    d, nb = WIDTHS[cd]
    ix, m = _rq_index(d, nb, metric, seed=cd)
    q = np.random.default_rng(cd + 1).standard_normal((2, d), dtype=np.float32)
    for k, nprobes in SEARCHES:
        _same(ix.search(q, k=k, nprobes=nprobes), ivfrq_search(*m, q, k, nprobes, metric=metric))
    wrapped, total = _wrapped_rows(m, q, 5, metric)
    assert total > 0
    if cd >= 2048:                                  # the wrapping 16-bit sums ran
        assert wrapped > 0, (wrapped, total)
    if cd <= 1024:                                  # at most 256 sub-tables of <= 255: no sum can wrap
        assert wrapped == 0


@pytest.mark.parametrize("metric", ["l2", "dot"])
def test_scan_wraps_with_sign_pattern_codes(metric):
    """code_dim 1536: every row's code is the sign pattern of the query's rotated residual for its partition (a few
    bits flipped), so every pair picks its sub-tables' maximum entries, close to 255: 384 sub-tables wrap."""
    d, nb, sizes = 8, 192, (33, 64, 4097, 100)
    cd, K = d * nb, len(sizes)
    rng = np.random.default_rng(15)
    q = rng.standard_normal((1, d), dtype=np.float32)
    # residuals q - c_p = (0.5 + 0.1 p) * (+-1, ..): every rotated component has nearly the same magnitude
    signs = rng.choice(np.array([-1.0, 1.0], np.float32), (K, d))
    cent = (q - (np.float32(0.5) + np.float32(0.1) * np.arange(K, dtype=np.float32))[:, None] * signs).astype(np.float32)
    rot = np.zeros((cd, cd), np.float32)
    rot[np.arange(cd), np.arange(cd) % d] = rng.choice(np.array([-1.0, 1.0], np.float32), cd)
    rot[:, :d] += np.float32(0.01) * rng.standard_normal((cd, d), dtype=np.float32)
    codes = []
    for p, n in enumerate(sizes):
        base = pack_signs(dot16(q - cent[p:p + 1], rot[:, :d]))
        flips = np.packbits(rng.random((n, cd)) < 0.03, axis=1, bitorder="little")
        codes.append(base ^ flips)
    ix, m = _rq_index(d, nb, metric, sizes=sizes, seed=16, rot=rot, cent=cent, codes=np.concatenate(codes))
    for k in (1, 10, 100, 1024):
        _same(ix.search(q, k=k, nprobes=K), ivfrq_search(*m, q, k, K, metric=metric))
    wrapped, total = _wrapped_rows(m, q, K, metric)
    assert wrapped == total == 32 + 64 + 4096 + 96, (wrapped, total)


@pytest.mark.parametrize("metric", ["l2", "dot"])
def test_wide_scan_ties_masks_and_range(metric):
    """code_dim 3072: rows drawn from 5 distinct rows (ties at the k-th distance), an allow list, a block list, both,
    a range, and a range with a list"""
    d, nb = 16, 192
    cd = d * nb
    n = int(sum(SIZES))
    rng = np.random.default_rng(21)
    pick = rng.integers(0, 5, n)
    codes = rng.integers(0, 256, (5, cd // 8), dtype=np.uint8)[pick]
    add = rng.uniform(0.5, 4.0, 5).astype(np.float32)[pick]
    scale = rng.standard_normal(5, dtype=np.float32)[pick]
    ix, m = _rq_index(d, nb, metric, seed=22, codes=codes, add=add, scale=scale)
    q = rng.standard_normal((3, d), dtype=np.float32)
    for k in (1, 10, 100, 1024):
        want = ivfrq_search(*m, q, k, 5, metric=metric)
        _same(ix.search(q, k=k, nprobes=5), want)
        if k in (10, 100):                         # the k-th distance is tied with the (k + 1)-th
            nxt = ivfrq_search(*m, q, k + 1, 5, metric=metric)[1]
            assert (_bits(nxt[:, k - 1]) == _bits(nxt[:, k])).all()
    rid = m[6]
    allow = rng.choice(rid, n // 2, replace=False)
    block = rng.choice(rid, n // 3, replace=False)
    _, d0 = ix.search(q, k=200, nprobes=5)
    lo, hi = float(d0[0, 20]), float(d0[0, 150])
    cases = [({"allow_bitmap": ix.row_mask(allow_row_ids=allow)}, {"allow": allow}),
             ({"allow_bitmap": ix.row_mask(block_row_ids=block)}, {"block": block}),
             ({"allow_bitmap": ix.row_mask(allow_row_ids=allow, block_row_ids=block)}, {"allow": allow, "block": block}),
             ({"lower_bound": lo, "upper_bound": hi}, {"lower": lo, "upper": hi}),
             ({"allow_bitmap": ix.row_mask(block_row_ids=block), "upper_bound": hi}, {"block": block, "upper": hi})]
    for kw, rkw in cases:
        for k in (10, 100, 1024):
            _same(ix.search_ex(q, k=k, nprobes=5, **kw), ivfrq_search(*m, q, k, 5, metric=metric, **rkw))


# ---- 2. the shared-memory boundary -------------------------------------------------------------------------------
def _smem_estimate(k):
    """rq_scan_smem_bytes = 20 code_dim + slot_smem_bytes(k) against the opt-in limit, rounded down to a multiple
    of 8 (the kernel's static shared memory lowers the true limit a little)"""
    import torch
    optin = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    slot = 4 * (4096 + 4 * (k + 1))
    return (optin - slot) // 20 // 8 * 8


def test_shared_memory_boundary():
    d, sizes = 8, (33, 4097)
    rng = np.random.default_rng(30)
    top = _smem_estimate(1) + 8                     # past the formula's limit: create must refuse it
    buf = rng.standard_normal(top * top, dtype=np.float32)   # every candidate's full code_dim^2 rotation

    def rot(cd):
        return buf[:cd * cd].reshape(cd, cd)

    def index(cd):
        return _rq_index(d, cd // d, "l2", sizes=sizes, seed=cd, rot=rot(cd))

    # C: the largest width that create accepts, walking down from past the estimate
    C, ix = top, None
    while ix is None:
        try:
            ix, m = index(C)
        except lb.LanceB200Error as e:
            assert e.status == lb._lib.UNSUPPORTED, e
            C -= 8
            assert C > top - 8 * 64
    assert C < top
    assert _status(lambda: index(C + 8)) == lb._lib.UNSUPPORTED
    q = rng.standard_normal((2, d), dtype=np.float32)
    _same(ix.search(q, k=1, nprobes=2), ivfrq_search(*m, q, 1, 2))
    assert _wrapped_rows(m, q, 2, "l2")[0] > 0
    # at C the k = 1024 selection does not fit: refused before anything is written
    ids, dists = np.full((2, 1024), 7, np.uint64), np.full((2, 1024), 3.0, np.float32)
    assert _status(lambda: ix.search(q, k=1024, nprobes=2, out=(ids, dists))) == lb._lib.UNSUPPORTED
    assert (ids == 7).all() and (dists == 3.0).all()
    del ix
    # the largest width at which k = 1024 fits, found the same way
    C2 = _smem_estimate(1024) + 8
    while True:
        ix, m = index(C2)
        try:
            got = ix.search(q, k=1024, nprobes=2)
            break
        except lb.LanceB200Error as e:
            assert e.status == lb._lib.UNSUPPORTED, e
            C2 -= 8
            assert C2 > _smem_estimate(1024) - 8 * 64
    assert C2 < C
    _same(got, ivfrq_search(*m, q, 1024, 2))
    assert _status(lambda: index(C2 + 8)[0].search(q, k=1024, nprobes=2)) == lb._lib.UNSUPPORTED
    print(f"IVF_RQ code_dim limit: {C} at k = 1, {C2} at k = 1024")


# ---- 3. rotation groups ------------------------------------------------------------------------------------------
def _group_queries(qc, nq, rng, extra=16):
    """the queries on either side of every group and slab boundary, plus a random few"""
    edges = [b for b in range(qc, nq, qc)] + [b for b in range(SLAB, nq, SLAB)]
    near = [i for b in edges for i in (b - 1, b) if 0 <= i < nq]
    return np.unique(np.concatenate([near, rng.choice(nq, extra, replace=False)]).astype(np.int64))


def _group_size(np_, d, cd, qn):
    return max(1, min(qn, GROUP_BYTES // (np_ * (d + cd) * 4)))


@pytest.mark.parametrize("shape", ["wide", "c1"])
def test_rotation_groups(shape):
    """wide: d = 16, code_dim 8192, 8 of 16 partitions probed -> groups of 1022 queries, 3 of them in 2100 queries;
    c1: d = 128, one bit, nprobes 10 -> groups of 26 214 queries: slab 1 is two groups, slab 2 (37 queries) one"""
    if shape == "wide":
        d, nb, K, nprobes, nq = 16, 512, 16, 8, 2100
        sizes = (0, 31, 32, 33, 40, 64, 65, 100, 1, 96, 97, 0, 31, 128, 200, 33)
    else:
        d, nb, K, nprobes, nq = 128, 1, 16, 10, SLAB + 37
        sizes = (31, 32, 33, 200, 0, 97, 64, 300, 65, 1, 33, 128, 129, 400, 70, 40)
    cd = d * nb
    ix, m = _rq_index(d, nb, "l2", sizes=sizes, seed=40 + d)
    rng = np.random.default_rng(41)
    q = rng.standard_normal((nq, d), dtype=np.float32)
    qc = _group_size(nprobes, d, cd, min(nq, SLAB))
    slabs = [(a, min(nq, a + SLAB)) for a in range(0, nq, SLAB)]
    groups = [(a + g, min(b, a + g + qc)) for a, b in slabs for g in range(0, b - a, qc)]
    assert len(groups) >= 3
    got = ix.search(q, k=10, nprobes=nprobes)
    # one call == the same queries searched one group at a time
    parts = [ix.search(q[a:b], k=10, nprobes=nprobes) for a, b in groups]
    for j in range(2):
        assert _same_arrays(got[j], np.concatenate([p[j] for p in parts])), j
    sel = _group_queries(qc, nq, rng)
    _same((got[0][sel], got[1][sel]), ivfrq_search(*m, q[sel], 10, nprobes))
    prof = _profiled(lambda: ix.search(q, k=10, nprobes=nprobes))
    assert _launches(prof, "rq_scan") == len(groups) and _launches(prof, "rq_rotate") == len(groups), prof


# ---- 4. query slabs for IVF_SQ and IVF_RQ ------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["sq", "rq"])
def test_search_across_query_slabs(kind):
    d, n, K, nprobes, rf, k = 128, 12000, 8, 2, 4, 10
    nq = SLAB + 37
    rng = np.random.default_rng(500 + len(kind))
    base = rng.integers(0, 6, (150, d)).astype(np.float32)
    data = base[rng.integers(0, 150, n)]          # integer rows, each ~80 times: ties at the k-th distance
    q = base[rng.integers(0, 150, nq)] + np.float32(0.25)
    build = lb.IvfSqIndex.build if kind == "sq" else lb.IvfRqIndex.build
    ix = build(data, "l2", num_partitions=K, max_iters=5)
    e = ix.export()
    allow = rng.choice(e["row_ids"], n // 2, replace=False)
    bm = ix.row_mask(allow, None)
    plain = ix.search_ex(q, k=k, nprobes=nprobes)
    lo, hi = float(np.median(plain[1][:, 1])), float(np.median(plain[1][:, k - 2]))
    variants = {"plain": {}, "mask": {"allow_bitmap": bm}, "range": {"lower_bound": lo, "upper_bound": hi},
                "refine": {"refine_factor": rf, "vectors": data}}
    sel = np.unique(np.concatenate([np.arange(SLAB - 32, SLAB + 32), rng.choice(nq, 64, replace=False)]))

    def restated(kk, **kw):
        if kind == "sq":
            return ivfsq_search(e["centroids"], e["bounds"], e["part_offsets"], e["codes"], e["row_ids"], q[sel], kk,
                                nprobes, **kw)
        return ivfrq_search(e["centroids"], e["rotation"], e["part_offsets"], e["codes"], e["add_factors"],
                            e["scale_factors"], e["row_ids"], q[sel], kk, nprobes, **kw)

    for var, kw in variants.items():
        got = ix.search_ex(q, k=k, nprobes=nprobes, **kw)
        a, b = ix.search_ex(q[:SLAB], k=k, nprobes=nprobes, **kw), ix.search_ex(q[SLAB:], k=k, nprobes=nprobes, **kw)
        for j in range(2):                          # one call == the same queries in two calls split at the slab
            assert _same_arrays(got[j], np.concatenate([a[j], b[j]])), (var, j)
        if var == "refine":                         # exact re-rank of the restatement's k * rf candidates
            oi, od, oc = restated(k * rf)
            for i, qi in enumerate(sel):
                cand = oi[i, :oc[i]].astype(np.int64)
                ex = np.array([ob.l2(q[qi], data[c]) for c in cand], np.float32)
                order = np.lexsort((cand, ex))[:k]
                assert _same_arrays(got[1][qi, :len(order)], ex[order]), (var, qi)
                assert np.array_equal(got[0][qi, :len(order)].astype(np.int64), cand[order]), (var, qi)
            continue
        extra = {"mask": {"allow": allow}, "range": {"lower": lo, "upper": hi}}.get(var, {})
        _same((got[0][sel], got[1][sel]), restated(k, **extra))
    # the second slab really has queries whose k-th distance is tied
    _, od, _ = restated(k + 1)
    second = sel >= SLAB
    assert np.any((od[second, k - 1] == od[second, k]) & np.isfinite(od[second, k]))
    prof = _profiled(lambda: ix.search_ex(q, k=k, nprobes=nprobes))
    assert _launches(prof, f"{kind}_scan") == 2, prof


# ---- 5. chunked and streamed builds and transforms ---------------------------------------------------------------
NC, DC, KC = 3000, 32, 8
CHUNKS = ((1, 300), (64, NC), (65, NC), (1000, NC))     # (LB2_CHUNK_ROWS, rows)
EDGES = (0, 1, 63, 64, 65, 129, 130, 299, 999, 1000, 1001, 1999, 2000, 2999)


@pytest.fixture
def make_src():
    """the same rows as pageable numpy, PinnedArray or DeviceArray; pinned buffers are freed at teardown"""
    pinned = []

    def make(x, kind):
        if kind == "numpy":
            return np.ascontiguousarray(x)
        if kind == "device":
            return lb.DeviceArray.from_numpy(x)
        p = lb.PinnedArray(x.shape, x.dtype)
        p.array[...] = x
        pinned.append(p)
        return p
    yield make
    for p in pinned:
        p.free()


def _chunk_data(seed):
    """rows around 8 centres; zero and non-finite rows on the first and last rows of chunks"""
    rng = np.random.default_rng(seed)
    cent = (rng.standard_normal((KC, DC)) * 2).astype(np.float32)
    x = cent[rng.integers(0, KC, NC)] + rng.standard_normal((NC, DC), dtype=np.float32)
    for i, r in enumerate(EDGES):
        if i % 5 == 0:
            x[r] = 0.0
        elif i % 5 == 1:
            x[r] = np.nan
        else:
            x[r, 3 * i % DC] = (np.inf, -np.inf, np.nan)[i % 5 - 2]
    return cent, x


def _sources(C):
    """(source kind, LB2_MAX_RESIDENT_MB): resident from every kind of memory; streamed from host memory"""
    out = [("device", None), ("pinned", None), ("numpy", None)]
    if C in (64, 1000):
        out += [("pinned", 0), ("numpy", 0)]
    return out


@pytest.mark.parametrize("metric", ["l2", "cosine", "dot"])
def test_rq_transform_over_chunks_and_streams(metric, make_src, monkeypatch):
    cent, x = _chunk_data(60)
    if metric == "cosine":
        cent = ob.normalize_rows(cent)
    rng = np.random.default_rng(61)
    rq = lb.RabitQuantizer(DC, 2, rotation=_rotation(2 * DC, DC, rng))
    part, codes, add, scale, valid = rq_transform(cent, rq.rotation, x, metric, 2)
    for C, n in CHUNKS:
        xn = np.ascontiguousarray(x[:n])
        _knobs(monkeypatch)
        ref = rq.transform(cent, make_src(xn, "device"), metric)
        assert np.array_equal(ref["valid"], valid[:n]) and np.array_equal(ref["part_ids"][valid[:n]], part[:n][valid[:n]])
        assert np.array_equal(ref["codes"], codes[:n])
        assert _same_arrays(ref["add_factors"], add[:n]) and _same_arrays(ref["scale_factors"], scale[:n])
        for kind, mb in _sources(C):
            _knobs(monkeypatch, chunk=C, resident_mb=mb)
            got = rq.transform(cent, make_src(xn, kind), metric)
            assert all(_same_arrays(got[key], ref[key]) for key in ref), (C, kind, mb)
    # chunks of 1000 rows: one rotation per chunk, one staged copy per chunk when streamed
    for kind, mb, staged in (("device", None, 0), ("pinned", 0, 3)):
        s = make_src(x, kind)
        _knobs(monkeypatch, chunk=1000, resident_mb=mb)
        p = _profiled(lambda: rq.transform(cent, s, metric))
        assert _launches(p, "rq_rotate") == 3 and _launches(p, "stage_rows") == staged, p
    _knobs(monkeypatch)


def test_sq_transform_under_chunks(make_src, monkeypatch):
    """ScalarQuantizer.transform encodes the whole matrix at once: the chunk and stream knobs leave it unchanged"""
    _, x = _chunk_data(62)
    sq = lb.ScalarQuantizer(DC)
    _knobs(monkeypatch)
    assert sq.build(x) == sq_bounds(x)
    want = sq_encode(x, *sq.bounds)
    assert np.array_equal(sq.transform(x), want)
    for C, n in CHUNKS:
        for kind, mb in _sources(C):
            _knobs(monkeypatch, chunk=C, resident_mb=mb)
            assert np.array_equal(sq.transform(make_src(np.ascontiguousarray(x[:n]), kind)), want[:n]), (C, kind, mb)
    _knobs(monkeypatch)


@pytest.mark.parametrize("kind", ["rq", "sq"])
@pytest.mark.parametrize("metric", ["l2", "dot"])
def test_build_over_chunks_and_streams(kind, metric, make_src, monkeypatch):
    _, x = _chunk_data(63 + len(metric))
    cls = lb.IvfRqIndex if kind == "rq" else lb.IvfSqIndex
    build = lambda s: cls.build(s, metric, num_partitions=KC, max_iters=5, seed=3)
    finite = np.isfinite(x).all(axis=1)
    for C, n in CHUNKS:
        xn = np.ascontiguousarray(x[:n])
        _knobs(monkeypatch)
        ref = build(make_src(xn, "device")).export()
        # the restatement: every finite row is stored; the codes of the stored rows
        rows = ref["row_ids"].astype(np.int64)
        assert np.array_equal(np.sort(rows), np.flatnonzero(finite[:n]))
        if kind == "rq":
            _, codes, add, scale, valid = rq_transform(ref["centroids"], ref["rotation"], xn[rows], metric)
            assert valid.all() and np.array_equal(ref["codes"], codes)
            assert _same_arrays(ref["add_factors"], add) and _same_arrays(ref["scale_factors"], scale)
        else:
            assert ref["bounds"] == sq_bounds(xn[finite[:n]])          # n <= 65 536: the sample is every row
            assert np.array_equal(ref["codes"], sq_encode(xn[rows], *ref["bounds"]))
        for src_kind, mb in _sources(C):
            _knobs(monkeypatch, chunk=C, resident_mb=mb)
            e = build(make_src(xn, src_kind)).export()
            for key in ref:
                assert _same_arrays(e[key], ref[key]) if key != "bounds" else e[key] == ref[key], (C, src_kind, mb, key)
    # chunks of 1000 rows, streamed: one staged copy and one encode per chunk
    s = make_src(x, "pinned")
    _knobs(monkeypatch, chunk=1000, resident_mb=0)
    p = _profiled(lambda: build(s))
    _knobs(monkeypatch)
    assert _launches(p, "stage_rows") == 3, p
    assert _launches(p, "rq_rotate" if kind == "rq" else "sq_encode") == 3, p


def test_rq_transform_sub_chunks(monkeypatch):
    """d = 8, num_bits = 1024: a row chunk of 70 000 rows is rotated in sub-chunks of 2^28 / 8192 = 32 768 rows"""
    d, nb, n = 8, 1024, 70000
    cd = d * nb
    rng = np.random.default_rng(70)
    cent = rng.standard_normal((4, d), dtype=np.float32)
    x = cent[rng.integers(0, 4, n)] + rng.standard_normal((n, d), dtype=np.float32)
    rq = lb.RabitQuantizer(d, nb, rotation=_rotation(cd, d, rng))
    _knobs(monkeypatch, chunk=n)
    got = rq.transform(cent, x, "l2")
    res = []
    p = _profiled(lambda: res.append(rq.transform(cent, x, "l2")))
    _knobs(monkeypatch)
    assert all(_same_arrays(res[0][key], got[key]) for key in got)
    sub = (1 << 28) // cd
    assert _launches(p, "rq_rotate") == 3 and _launches(p, "rq_encode") == 3, p    # 32 768 + 32 768 + 4 464 rows
    rows = np.unique(np.concatenate([np.arange(b - 8, b + 8) for b in (sub, 2 * sub)] + [rng.choice(n, 48)]))
    part, codes, add, scale, valid = rq_transform(cent, rq.rotation, x[rows], "l2", nb)
    assert valid.all() and np.array_equal(got["part_ids"][rows], part) and np.array_equal(got["codes"][rows], codes)
    assert _same_arrays(got["add_factors"][rows], add) and _same_arrays(got["scale_factors"][rows], scale)


# ---- 6. the rotation ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 2, 8, 255, 256, 257, 1032, 3072])
def test_rotation_householder_properties(n):
    """|Q^T Q - I|_max <= n 2^-24: the f64 factor is orthogonal to ~n 2^-52, and rounding each entry to f32 moves
    an entry of Q^T Q by at most 2 * 2^-24 * sum_k |q_ki q_kj| <= 2^-23 (Cauchy-Schwarz)"""
    r1 = lb.RabitQuantizer(n, 1).build(seed=5)
    assert np.isfinite(r1).all()
    assert np.array_equal(r1, lb.RabitQuantizer(n, 1).build(seed=5))
    if n > 1:
        assert not np.array_equal(r1, lb.RabitQuantizer(n, 1).build(seed=6))
    r = r1.astype(np.float64)
    err = np.abs(r.T @ r - np.eye(n)).max()
    assert err <= max(n, 2) * 2.0 ** -24, err
    sign, _ = np.linalg.slogdet(r)
    assert sign == (-1) ** (n - 1)                  # all n - 1 reflections were applied


@pytest.mark.parametrize("d,nb,n", [(1536, 1, 200), (3072, 1, 100), (16, 512, 300)])
def test_transform_at_wide_code_widths(d, nb, n):
    rng = np.random.default_rng(d + nb)
    cent = rng.standard_normal((4, d), dtype=np.float32)
    x = cent[rng.integers(0, 4, n)] + rng.standard_normal((n, d), dtype=np.float32)
    x[7] = cent[2]
    rq = lb.RabitQuantizer(d, nb, rotation=_rotation(d * nb, d, rng))
    for metric in ("l2", "dot"):
        got = rq.transform(cent, x, metric)
        part, codes, add, scale, valid = rq_transform(cent, rq.rotation, x, metric, nb)
        assert valid.all() and np.array_equal(got["part_ids"], part) and np.array_equal(got["codes"], codes)
        assert _same_arrays(got["add_factors"], add) and _same_arrays(got["scale_factors"], scale)


# ---- 7. numeric edges of the scan --------------------------------------------------------------------------------
@pytest.mark.parametrize("metric", ["l2", "dot"])
def test_query_on_a_probed_centroid_gives_a_flat_table(metric):
    ix, m = _rq_index(16, 4, metric, seed=80)
    q = m[0][[1, 3, 4]].copy()                      # the residual query of that probe is zero: qmin == qmax
    assert (quantize_table(dist_table(np.zeros(64, np.float32)))[2] == 0).all()
    for k in (1, 10, 100, 1024):
        _same(ix.search(q, k=k, nprobes=5), ivfrq_search(*m, q, k, 5, metric=metric))


@pytest.mark.parametrize("metric", ["l2", "cosine", "dot"])
@pytest.mark.parametrize("e", [40, -40])
def test_queries_scaled_by_large_and_small_powers_of_two(metric, e):
    ix, m = _rq_index(16, 2, metric, seed=81)
    q = np.random.default_rng(82).standard_normal((3, 16), dtype=np.float32) * np.float32(2.0 ** e)
    for k in (1, 10, 1024):
        _same(ix.search(q, k=k, nprobes=5), ivfrq_search(*m, q, k, 5, metric=metric))


@pytest.mark.parametrize("metric", ["l2", "dot"])
def test_factors_that_overflow_give_nans_that_sort_first(metric):
    """rows near 2^64: |x - c|^2 overflows and the row is dropped, or -2 |r|^2 / ip (L2) or |r|^2 (dot) does and
    the scale becomes -inf.  A query on a centroid has the flat table there (dvq = 0): 0 * inf = NaN, which the scan
    writes as x86's NaN 0xFFC00000, ordered before every number; other queries give +-inf"""
    d, sizes = 16, (33, 64, 4097)
    rng = np.random.default_rng(83)
    cent = rng.standard_normal((3, d), dtype=np.float32)
    n = int(sum(sizes))
    x = cent[np.repeat(np.arange(3), sizes)] + rng.standard_normal((n, d), dtype=np.float32)
    big = rng.choice(n, 300, replace=False)
    x[big] *= np.float32(2.0 ** 62)
    rot = _rotation(d, d, rng)
    t = lb.RabitQuantizer(d, 1, rotation=rot).transform(cent, x, metric)
    part, codes, add, scale, valid = rq_transform(cent, rot, x, metric)
    assert np.array_equal(t["valid"], valid) and np.array_equal(t["codes"], codes)
    assert _same_arrays(t["add_factors"], add) and _same_arrays(t["scale_factors"], scale)
    assert np.isneginf(scale[valid]).any() and (valid.all() if metric == "dot" else not valid.all())
    sizes = np.bincount(part[valid], minlength=3)
    order = np.argsort(part[valid], kind="stable")
    ix, m = _rq_index(d, 1, metric, sizes=tuple(sizes), seed=84, rot=rot, cent=cent, codes=codes[valid][order],
                      add=add[valid][order], scale=scale[valid][order])
    q = np.concatenate([cent, rng.standard_normal((2, d), dtype=np.float32)])
    for k in (1, 10, 100, 1024):
        want = ivfrq_search(*m, q, k, 3, metric=metric)
        _same(ix.search(q, k=k, nprobes=3), want)
        assert np.isnan(want[1][:3, 0]).any() and np.isinf(want[1][3:]).any()


@pytest.mark.parametrize("metric", ["l2", "dot"])
def test_negative_zero_residual_components(metric):
    """-0.0 - +0.0 = -0.0: rows and queries with -0.0 where the centroids hold +0.0, against rotations with -0.0 and
    +0.0 entries"""
    d, sizes = 16, (33, 64, 100)
    rng = np.random.default_rng(85)
    cent = rng.standard_normal((3, d), dtype=np.float32)
    cent[:, :6] = 0.0
    n = int(sum(sizes))
    x = cent[np.repeat(np.arange(3), sizes)] + rng.standard_normal((n, d), dtype=np.float32)
    x[:, :6] = -0.0
    x[::7] = cent[np.repeat(np.arange(3), sizes)][::7]
    x[::7, :6] = -0.0
    rot = _rotation(d, d, rng)
    rot[::3, :6] = -0.0
    rot[1::3, :6] = 0.0
    t = lb.RabitQuantizer(d, 1, rotation=rot).transform(cent, x, metric)
    part, codes, add, scale, valid = rq_transform(cent, rot, x, metric)
    res = x - cent[part]
    assert (np.signbit(res) & (res == 0)).any()
    assert np.array_equal(t["valid"], valid) and np.array_equal(t["part_ids"], part)
    assert np.array_equal(t["codes"], codes)
    assert _same_arrays(t["add_factors"], add) and _same_arrays(t["scale_factors"], scale)
    order = np.argsort(part, kind="stable")
    ix, m = _rq_index(d, 1, metric, sizes=tuple(np.bincount(part, minlength=3)), seed=86, rot=rot, cent=cent,
                      codes=codes[order], add=add[order], scale=scale[order])
    q = np.concatenate([x[[0, 7, 50]], cent[[0, 2]]])
    q[3:, :6] = -0.0
    for k in (1, 10, 100):
        _same(ix.search(q, k=k, nprobes=3), ivfrq_search(*m, q, k, 3, metric=metric))
