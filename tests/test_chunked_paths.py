"""The paths that split the work into pieces: row chunks of the per-row pass (`Source::rows_per_chunk`,
`for_each_chunk`, the chunked output loop of `index_load_flat_src`), host rows streamed through the two staging
slots, and searches longer than one 32 768-query slab.

At their natural sizes these paths need inputs of tens of GB.  Two knobs reach them at test sizes:
LB2_CHUNK_ROWS (rows per chunk, without the 64 Ki floor) and LB2_MAX_RESIDENT_MB (a host matrix above it is
streamed).  Every case is compared two ways: (a) bit for bit with the same call without the knobs on
device-resident rows, and (b) with the oracle on the converted values.  Separate profiled calls show that each
path ran; parity runs are not profiled, because profiling turns the asynchronous sample gather off."""
import numpy as np
import pytest

import lance_b200 as lb
from oracle import binding as ob

pytestmark = pytest.mark.gpu
NT = 16
SLAB = 32768          # queries per scan launch (grid.y limit, ivf_search.cuh)
TYPES = ("f32", "f16", "bf16", "u8")


def _knobs(monkeypatch, chunk=None, resident_mb=None):
    for name, v in (("LB2_CHUNK_ROWS", chunk), ("LB2_MAX_RESIDENT_MB", resident_mb)):
        if v is None:
            monkeypatch.delenv(name, raising=False)
        else:
            monkeypatch.setenv(name, str(v))


def _typed(a, t):
    """f32 values -> (array of column type t, the exact f32 values it holds); bf16 = uint16 bit patterns"""
    a = np.ascontiguousarray(a, np.float32)
    if t == "bf16":
        x = (a.view(np.uint32) >> 16).astype(np.uint16)
        return x, (x.astype(np.uint32) << 16).view(np.float32)
    x = {"f32": lambda: a.copy(), "f16": lambda: a.astype(np.float16),
         "u8": lambda: np.clip(np.rint(a), 0, 255).astype(np.uint8)}[t]()
    return x, x.astype(np.float32)


def _model(a, t):
    """a model of a column of type t: f32 for f32 / u8 columns, the column's own type otherwise"""
    return _typed(a, "f32" if t in ("f32", "u8") else t)


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


def _profiled(fn):
    lb.profile.enable(True)
    lb.profile.reset()
    try:
        fn()
    finally:
        lb.profile.enable(False)
    return lb.profile.dump()


def _launches(prof, name):
    return prof.get(name, (0, 0.0))[0]


def _tight_groups(rng, k, d):
    """centroids in groups of 8 that differ by ~1e-3 (far below the TF32 resolution) and exact duplicates"""
    base = (rng.standard_normal(((k + 7) // 8, d)) * 20).astype(np.float32)
    cent = np.repeat(base, 8, axis=0)[:k] + (rng.standard_normal((k, d)) * 1e-3).astype(np.float32)
    cent[17] = cent[16]
    cent[40:44] = cent[40]
    cent[k - 40:k - 20] = cent[k - 40]      # 20 identical: more candidates than slots -> full exact scan
    return cent


def _same(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    if a.dtype != b.dtype or a.shape != b.shape:
        return False
    if a.dtype.kind == "f":                # bit for bit (the NaN distance of an invalid row included)
        a, b = a.view(f"u{a.dtype.itemsize}"), b.view(f"u{b.dtype.itemsize}")
    return np.array_equal(a, b)


def _check_topk(ids, dists, oi, od):
    """the SET of (distance, row id) pairs equals the oracle's (rows tied at the k-th distance included)"""
    got = sorted(zip(np.asarray(dists).view(np.uint32).tolist(), np.asarray(ids).tolist()))
    exp = sorted(zip(np.asarray(od).view(np.uint32).tolist(), np.asarray(oi).tolist()))
    assert got == exp


# ---- 1. + 2. compute_partitions and ivfpq_transform over row chunks, resident and streamed ---------------------
SHAPES = {"resident": (128, 200, 16), "general": (192, 300, 24)}     # d, K, M: resident / general filter
N1 = 3000
# chunk rows -> row counts: an exact multiple, a ragged tail (< 256 rows: the PQ encoder's exact path for that
# chunk), n = 1.5 C (one call, the 1.5-chunk rule) and n = 1.5 C + 1 (two chunks)
CHUNK_CASES = ((1, (1, 2, 300)), (64, (320, 273, 96, 97)), (65, (260, 205, 97, 98)), (1000, (3000, 2100, 1500, 1501)))
BOUNDS = (64, 65, 96, 97, 128, 130, 192, 195, 205, 256, 260, 273, 320, 1000, 1500, 2000, 2100, 3000)


def _case1_data(t, d, K, M, seed):
    rng = np.random.default_rng(seed)
    s = {"f32": 1.0, "bf16": 1.0, "f16": 0.05, "u8": 2.0}[t]
    cent_m, cent = _model(_tight_groups(rng, K, d) * np.float32(s) + np.float32(128.0 if t == "u8" else 0.0), t)
    idx = rng.integers(0, K, N1)
    x = cent[idx] + (rng.standard_normal((N1, d)) * (0.3 * s)).astype(np.float32)
    cb_m, cb = _model((rng.standard_normal((M, 256, d // M)) * (0.3 * s)).astype(np.float32), t)
    cb[0, 7] = cb[0, 3]                  # duplicate codeword: index 3 must win
    cb[1, 100:104] = cb[1, 100]          # 4-way tie
    cb_m, cb = _model(cb, t)
    ds = d // M
    # near-ties on both sides of every chunk boundary, so that the fallback lists of later chunks are not empty
    for b in BOUNDS:
        for r in range(b - 3, min(b + 3, N1)):
            kind = r % 4
            if kind == 0:
                x[r] = (cent[0] + cent[9]) * np.float32(0.5)     # half-way between two centroids
            elif kind == 1:
                x[r] = cent[K - 30]                              # on the 20-fold duplicate
            elif kind == 2:
                x[r] = cent[16]                                  # on an exact duplicate pair
            else:
                x[r, :ds] = cent[idx[r], :ds] + cb[0, 3]         # residual on a duplicated codeword
    if t != "u8":                        # non-finite rows on the first and last row of chunks
        x[64] = np.nan
        x[1000] = np.nan
        x[63, 5] = np.nan
        x[1999, 0] = np.nan
        x[65, 3] = np.inf
        x[2000, 7] = np.inf
        x[129, 1] = -np.inf
        x[999, d - 1] = -np.inf
    xt, x32 = _typed(x, t)
    po, do, vo = ob.compute_membership(cent, x32, nthreads=NT)
    res = ob.compute_residual(cent, np.where(np.isfinite(x32), x32, 0), po, nthreads=NT)
    co = ob.pq_encode(cb, res, nthreads=NT)
    return cent_m, cb_m, xt, (po, do, vo, co)


@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("t", TYPES)
def test_partitions_and_transform_over_chunks_and_streams(t, shape, make_src, monkeypatch):
    d, K, M = SHAPES[shape]
    bf = t == "bf16"
    cent_m, cb_m, xt, (po, do, vo, co) = _case1_data(t, d, K, M, seed=100 + d + len(t))
    part = lambda x: lb.compute_partitions(cent_m, x, bf16=bf)
    trans = lambda x: lb.ivfpq_transform(cent_m, cb_m, x, bf16=bf)

    def same_as(got, ref, what):
        assert all(_same(g, r) for g, r in zip(got, ref)), what

    for C, ns in CHUNK_CASES:
        for n in ns:
            xn = np.ascontiguousarray(xt[:n])
            _knobs(monkeypatch)
            dev = make_src(xn, "device")
            ref_p, ref_t = part(dev), trans(dev)
            # (b) the unchunked device run is the oracle's
            v = ref_p[2]
            assert np.array_equal(v, vo[:n]) and np.array_equal(ref_t[2], vo[:n])
            assert np.array_equal(ref_p[0][v], po[:n][v]) and np.array_equal(ref_p[1][v], do[:n][v])
            assert np.array_equal(ref_t[0][v], po[:n][v]) and np.array_equal(ref_t[1][v], co[:n][v])
            # (a) chunked, from every kind of source, is the unchunked run bit for bit
            for kind in ("device", "pinned", "numpy"):
                s = dev if kind == "device" else make_src(xn, kind)
                _knobs(monkeypatch, chunk=C)
                same_as(part(s), ref_p, (C, n, kind, "partitions"))
                same_as(trans(s), ref_t, (C, n, kind, "transform"))
                if kind == "device" or C not in (64, 1000):
                    continue
                # streamed through the staging slots, right after the resident runs above warmed the cache
                _knobs(monkeypatch, chunk=C, resident_mb=0)
                same_as(part(s), ref_p, (C, n, kind, "partitions, streamed"))
                same_as(trans(s), ref_t, (C, n, kind, "transform, streamed"))
    _knobs(monkeypatch)


def test_chunk_and_stream_paths_ran(make_src, monkeypatch):
    """Profiled calls, separate from the parity runs.  Launches that run exactly once per chunk:
    `tc_filter` / `tc_filter_general(16)` once per tensor-core assignment, and the per-row pass calls the
    assignment once per chunk (its own sub-chunks are >= 64 Ki rows); `tc_pq_filter` once per PQ encode of a
    chunk of >= 256 rows, `pq_assign_exact` for a shorter one; `stage_rows` once per staged host chunk."""
    # f32, resident filter, C = 1000, n = 2100: chunks of 1000, 1000 and a 100-row tail
    d, K, M = SHAPES["resident"]
    cent_m, cb_m, xt, _ = _case1_data("f32", d, K, M, seed=7)
    dev = make_src(np.ascontiguousarray(xt[:2100]), "device")
    _knobs(monkeypatch, chunk=1000)
    p = _profiled(lambda: lb.compute_partitions(cent_m, dev))
    assert _launches(p, "tc_filter") == 2 and _launches(p, "assign_exact") == 1, p
    p = _profiled(lambda: lb.ivfpq_transform(cent_m, cb_m, dev))
    assert _launches(p, "tc_pq_filter") == 2 and _launches(p, "pq_assign_exact") == 1, p   # one call, both paths
    assert _launches(p, "stage_rows") == 0
    # f16 / bf16, general filter, C = 1000, n = 3000: the native 16-bit operands serve every chunk, the first and
    # the later ones, whether the rows are device-resident or streamed through the staging slots
    d, K, M = SHAPES["general"]
    for t in ("f16", "bf16"):
        cent_m, cb_m, xt, _ = _case1_data(t, d, K, M, seed=8)
        for kind, mb in (("device", None), ("numpy", 0), ("pinned", 0)):
            s = make_src(xt, kind)
            _knobs(monkeypatch, chunk=1000)
            lb.compute_partitions(cent_m, s, bf16=t == "bf16")       # (resident copy first: a warm staging cache)
            _knobs(monkeypatch, chunk=1000, resident_mb=mb)
            p = _profiled(lambda: lb.compute_partitions(cent_m, s, bf16=t == "bf16"))
            assert _launches(p, "tc_filter_general16") == 3 and _launches(p, "tc_filter_general") == 0, (t, kind, p)
            assert _launches(p, "stage_rows") == (0 if mb is None else 3), (t, kind, p)
    # u8 from pinned memory, C = 64, n = 320: five staged chunks; without the knob the same call stages nothing
    d, K, M = SHAPES["resident"]
    cent_m, cb_m, xt, _ = _case1_data("u8", d, K, M, seed=9)
    s = make_src(np.ascontiguousarray(xt[:320]), "pinned")
    _knobs(monkeypatch, chunk=64)
    assert _launches(_profiled(lambda: lb.ivfpq_transform(cent_m, cb_m, s)), "stage_rows") == 0
    _knobs(monkeypatch, chunk=64, resident_mb=0)
    p = _profiled(lambda: lb.ivfpq_transform(cent_m, cb_m, s))
    assert _launches(p, "stage_rows") == 5 and _launches(p, "pq_assign_exact") == 5, p
    _knobs(monkeypatch)


def test_native_16bit_rows_across_assignment_sub_chunks(monkeypatch):
    """A row chunk longer than 1.5 times the assignment's own chunk (2^20 rows at d = 64) is split again inside
    assign_f32_ex; the second part then reads its native f16 / bf16 rows at an offset from the chunk's native rows."""
    n, d, K = 1_600_000, 64, 300                 # K > 256: the general filter, which takes the native rows
    for t, s, seed in (("f16", 0.05, 700), ("bf16", 1.0, 701)):
        rng = np.random.default_rng(seed)
        cent_m, cent = _model(_tight_groups(rng, K, d) * np.float32(s), t)
        pool, pool32 = _typed(cent[rng.integers(0, K, 8192)] + (rng.standard_normal((8192, d)) * (0.3 * s)).astype(np.float32), t)
        pick = rng.integers(0, len(pool), n)
        dev = lb.DeviceArray.from_numpy(pool[pick])
        rows = np.unique(np.concatenate([np.arange((1 << 20) - 64, (1 << 20) + 64), rng.choice(n, 2000, replace=False)]))
        po, do, vo = ob.compute_membership(cent, pool32[pick[rows]], nthreads=NT)
        part = lambda: lb.compute_partitions(cent_m, dev, bf16=t == "bf16")
        _knobs(monkeypatch)                      # default: two row chunks, split at 2^20
        ref = part()
        _knobs(monkeypatch, chunk=1 << 21)       # one row chunk, split at 2^20 by the assignment
        got = part()
        assert all(_same(g, r) for g, r in zip(got, ref)), t
        assert np.array_equal(got[2][rows], vo) and np.array_equal(got[0][rows], po) and np.array_equal(got[1][rows], do), t
        # one conversion to f32 for the centroids and one for the single row chunk; two native-operand filters
        p = _profiled(part)
        _knobs(monkeypatch)
        assert _launches(p, "convert_to_f32") == 2 and _launches(p, "tc_filter_general16") == 2, (t, p)
        dev.free()


# ---- 3. IvfPqIndex.build: unchunked from the device == chunked == chunked and streamed from host memory ---------
BUILDS = [("l2", "f32", 8), ("l2", "f16", 8), ("l2", "bf16", 8), ("l2", "u8", 8), ("dot", "f16", 8),
          ("cosine", "f32", 8), ("cosine", "f16", 8), ("l2", "f32", 4)]
NB, DB, KB, MB = 4200, 192, 16, 24       # 4 chunks of 1000 rows and a 200-row tail


def _build_data(metric, t, seed):
    rng = np.random.default_rng(seed)
    if t == "u8":
        cent = rng.uniform(30, 220, (KB, DB)).astype(np.float32)
        x = cent[rng.integers(0, KB, NB)] + (rng.standard_normal((NB, DB)) * 12).astype(np.float32)
    else:
        cent = (rng.standard_normal((KB, DB)) * 2).astype(np.float32)
        x = cent[rng.integers(0, KB, NB)] + rng.standard_normal((NB, DB)).astype(np.float32)
        if metric == "dot":
            x /= np.linalg.norm(x, axis=1, keepdims=True)
        x[999, 4] = np.nan               # dropped rows on the last / first row of a chunk
        x[2000] = np.inf
    return _typed(x, t)


@pytest.mark.parametrize("metric,t,nbits", BUILDS)
def test_ivfpq_build_chunked_and_streamed_equals_resident(metric, t, nbits, make_src, monkeypatch):
    xt, x32 = _build_data(metric, t, seed=200 + nbits + len(metric) + len(t))
    prm = lb.IvfBuildParams(num_partitions=KB, num_sub_vectors=MB, num_bits=nbits, max_iters=5, pq_max_iters=4, seed=7)
    build = lambda s: lb.IvfPqIndex.build(s, metric, prm, bf16=t == "bf16")
    _knobs(monkeypatch)
    ix = build(make_src(xt, "device"))
    ref = ix.export()
    for kind, mb in (("device", None), ("pinned", 0), ("numpy", 0)):
        _knobs(monkeypatch, chunk=1000, resident_mb=mb)
        e = build(make_src(xt, kind)).export()
        for key in ref:
            assert _same(e[key], ref[key]), (kind, key)
    _knobs(monkeypatch)
    # the oracle's assignment and codes for the stored model; non-finite rows never enter the index
    src = ob.normalize_rows(x32, nthreads=NT) if metric == "cosine" else x32
    keep = np.isfinite(src).all(axis=1)
    assert np.array_equal(np.sort(ref["row_ids"]), np.flatnonzero(keep).astype(np.uint64))
    order = np.argsort(ref["row_ids"])
    p_ref, _, _ = ob.compute_membership(ref["centroids"], src[keep], metric="dot" if metric == "dot" else "l2", nthreads=NT)
    sizes = np.diff(ref["part_offsets"]).astype(np.int64)
    assert np.array_equal(np.repeat(np.arange(KB, dtype=np.uint32), sizes)[order], p_ref)
    res = src[keep] if metric == "dot" else ob.compute_residual(ref["centroids"], src[keep], p_ref, nthreads=NT)
    assert np.array_equal(ref["codes"][order], ob.pq_encode(ref["codebook"], res, nbits=nbits, nthreads=NT))
    # searches with queries in the column type (a bf16 IVF_PQ search included)
    rows = np.flatnonzero(keep)[np.random.default_rng(3).choice(int(keep.sum()), 24, replace=False)]
    ids, dists = ix.search(xt[rows], k=10, nprobes=4)
    oi, od, oc = ob.ivfpq_search(ref["centroids"], ref["codebook"], ref["part_offsets"], ref["codes"], ref["row_ids"],
                                 x32[rows], 10, 4, metric=metric, nbits=nbits, nthreads=NT)
    for i in range(len(rows)):
        c = int(oc[i])
        _check_topk(ids[i, :c], dists[i, :c], oi[i, :c], od[i, :c])
        assert np.isinf(dists[i, c:]).all()


def test_ivfpq_build_stream_path_ran(make_src, monkeypatch):
    """`transform:stage_rows` once per staged chunk (5); `tc_pq_filter` once per chunk of >= 256 rows (4) and the
    exact encoder once for the 200-row tail"""
    xt, _ = _build_data("l2", "f32", seed=5)
    prm = lb.IvfBuildParams(num_partitions=KB, num_sub_vectors=MB, max_iters=5, pq_max_iters=4, seed=7)
    s = make_src(xt, "pinned")
    _knobs(monkeypatch, chunk=1000, resident_mb=0)
    p = _profiled(lambda: lb.IvfPqIndex.build(s, "l2", prm))
    _knobs(monkeypatch)
    assert _launches(p, "transform:stage_rows") == 5, p
    assert _launches(p, "transform:tc_pq_filter") == 4 and _launches(p, "transform:pq_assign_exact") == 1, p


# ---- 4. IVF_FLAT: the chunked output loop, and the refusal of streamed input -----------------------------------
FLATS = [("l2", "u8"), ("cosine", "f16"), ("cosine", "f32"), ("l2", "bf16")]
NF, DF, KF = 4200, 64, 16


def _flat_data(t, seed):
    rng = np.random.default_rng(seed)
    if t == "u8":
        cent = rng.uniform(30, 220, (KF, DF)).astype(np.float32)
        x = cent[rng.integers(0, KF, NF)] + (rng.standard_normal((NF, DF)) * 12).astype(np.float32)
    else:
        cent = (rng.standard_normal((KF, DF)) * 2).astype(np.float32)
        x = cent[rng.integers(0, KF, NF)] + rng.standard_normal((NF, DF)).astype(np.float32)
        x[1000] = 0.0                    # a zero row: dropped under cosine
    return _typed(x, t)


@pytest.mark.parametrize("metric,t", FLATS)
def test_ivfflat_build_and_load_chunked_equal_unchunked(metric, t, make_src, monkeypatch):
    xt, x32 = _flat_data(t, seed=300 + len(metric) + len(t))
    bf = t == "bf16"
    build = lambda s: lb.IvfFlatIndex.build(s, metric, num_partitions=KF, max_iters=5, seed=3, bf16=bf)
    _knobs(monkeypatch)
    ref = build(make_src(xt, "device")).export()
    for kind in ("device", "pinned", "numpy"):
        _knobs(monkeypatch, chunk=1000)
        e = build(make_src(xt, kind)).export()
        for key in ref:
            assert _same(e[key], ref[key]), (kind, key)
    _knobs(monkeypatch)
    # (b) the stored rows are the oracle's (normalised for cosine, in the index's element type), grouped by the
    # oracle's partition of every kept row
    src = ob.normalize_rows(x32, nthreads=NT) if metric == "cosine" else x32
    keep = np.isfinite(src).all(axis=1)
    assert np.array_equal(np.sort(ref["row_ids"]), np.flatnonzero(keep).astype(np.uint64))
    order = np.argsort(ref["row_ids"])
    stored = {"f32": src, "u8": src, "f16": src.astype(np.float16), "bf16": xt}[t]
    assert _same(ref["vectors"][order], stored[keep])
    p_ref, _, _ = ob.compute_membership(ref["centroids"], src[keep], nthreads=NT)
    sizes = np.diff(ref["part_offsets"]).astype(np.int64)
    assert np.array_equal(np.repeat(np.arange(KF, dtype=np.uint32), sizes)[order], p_ref)
    # from_parts: the rows as given, grouped stably by the given partition ids
    cent_m, _ = _model(ref["centroids"], t)
    part = np.random.default_rng(4).integers(0, KF, NF).astype(np.uint32)
    _knobs(monkeypatch)
    want = lb.IvfFlatIndex.from_parts(cent_m, part, xt, distance_type=metric, bf16=bf).export()
    grouped = np.argsort(part, kind="stable")
    assert np.array_equal(want["row_ids"], grouped.astype(np.uint64))
    assert _same(want["vectors"], (xt if t in ("f16", "bf16") else x32)[grouped])
    _knobs(monkeypatch, chunk=1000)
    for kind in ("device", "pinned", "numpy"):
        e = lb.IvfFlatIndex.from_parts(cent_m, part, make_src(xt, kind), distance_type=metric, bf16=bf).export()
        for key in want:
            assert _same(e[key], want[key]), ("from_parts", kind, key)
    _knobs(monkeypatch)


def test_ivfflat_streamed_input_is_refused_and_releases_the_staging_cache(make_src, monkeypatch):
    xt, _ = _flat_data("u8", seed=31)
    build = lambda s: lb.IvfFlatIndex.build(s, "l2", num_partitions=KF, max_iters=5, seed=3)
    _knobs(monkeypatch)
    ref = build(make_src(xt, "device")).export()
    pin = make_src(xt, "pinned")
    # the chunked output loop ran once per chunk: `group_vectors` is two launches per chunk of 1000 rows
    _knobs(monkeypatch, chunk=1000)
    p = _profiled(lambda: build(pin))
    assert _launches(p, "group:group_vectors") == 2 * 5, p
    # device-resident rows are never streamed
    _knobs(monkeypatch, chunk=1000, resident_mb=0)
    e = build(make_src(xt, "device")).export()
    assert all(_same(e[k], ref[k]) for k in ref)
    for kind in ("pinned", "numpy"):
        _knobs(monkeypatch, chunk=1000, resident_mb=0)
        with pytest.raises(lb.LanceB200Error, match="must fit in device memory") as err:
            build(pin if kind == "pinned" else make_src(xt, "numpy"))
        assert err.value.status == 5
        # the next build on this thread gets the staging cache back and equals a fresh build
        _knobs(monkeypatch)
        e = build(pin).export()
        assert all(_same(e[k], ref[k]) for k in ref), kind
    _knobs(monkeypatch)


# ---- 5. searches of more than one query slab ---------------------------------------------------------------
NQ = SLAB + 37
SLAB_KINDS = {  # name: (index kind, d, M, nbits, k, environment)
    "skew2": ("pq", 128, 16, 8, 10, {"LB2_SCAN": "skew", "LB2_SCAN_TEAMS": "2"}),
    "skew4": ("pq", 128, 16, 8, 10, {"LB2_SCAN": "skew", "LB2_SCAN_TEAMS": "4"}),
    "classic": ("pq", 128, 16, 8, 10, {"LB2_SCAN": "classic"}),
    "m8": ("pq", 64, 8, 8, 10, {}),              # no skewed layout: the classic kernel
    "radix": ("pq", 128, 16, 8, 20, {}),         # k + 1 > 16: radix selection
    "pq4": ("pq", 128, 16, 4, 10, {}),
    "flat": ("flat", 128, 0, 0, 10, {}),
}
SCAN_LAUNCH = {"skew2": "search:pq_scan_skew", "skew4": "search:pq_scan_skew", "flat": "search:flat_scan"}


@pytest.mark.parametrize("name", list(SLAB_KINDS))
def test_search_across_query_slabs(name, monkeypatch):
    kind, d, M, nbits, k, env = SLAB_KINDS[name]
    for key, v in env.items():
        monkeypatch.setenv(key, v)
    rng = np.random.default_rng(400 + len(name))
    n, K, nprobes, rf = 12000, 8, 2, 4
    base = rng.integers(0, 6, (150, d)).astype(np.float32)
    data = base[rng.integers(0, 150, n)]          # integer rows, each ~80 times: ties at the k-th distance
    q = base[rng.integers(0, 150, NQ)] + np.float32(0.25)
    if kind == "pq":
        ix = lb.IvfPqIndex.build(data, "l2", lb.IvfBuildParams(num_partitions=K, num_sub_vectors=M, num_bits=nbits,
                                                               max_iters=5, pq_max_iters=4))
    else:
        ix = lb.IvfFlatIndex.build(data, "l2", num_partitions=K, max_iters=5)
    e = ix.export()
    allow = rng.choice(e["row_ids"], n // 2, replace=False)
    bm = ix.row_mask(allow, None)
    plain = ix.search_ex(q, k=k, nprobes=nprobes)
    lo, hi = float(np.median(plain[1][:, 1])), float(np.median(plain[1][:, k - 2]))
    variants = {"plain": {}, "mask": {"allow_bitmap": bm}, "range": {"lower_bound": lo, "upper_bound": hi},
                "refine": {"refine_factor": rf, "vectors": data}}
    sel = np.unique(np.concatenate([np.arange(SLAB - 32, SLAB + 32), rng.choice(NQ, 256, replace=False)]))

    def oracle(kk, **kw):
        if kind == "pq":
            return ob.ivfpq_search(e["centroids"], e["codebook"], e["part_offsets"], e["codes"], e["row_ids"], q[sel], kk,
                                   nprobes, nbits=nbits, nthreads=NT, **kw)
        return ob.ivfflat_search(e["centroids"], e["part_offsets"], e["vectors"], e["row_ids"], q[sel], kk, nprobes,
                                 nthreads=NT, **kw)

    for var, kw in variants.items():
        got = ix.search_ex(q, k=k, nprobes=nprobes, **kw)
        a, b = ix.search_ex(q[:SLAB], k=k, nprobes=nprobes, **kw), ix.search_ex(q[SLAB:], k=k, nprobes=nprobes, **kw)
        for j in range(2):                          # one call == the same queries in two calls split at the slab
            assert _same(got[j], np.concatenate([a[j], b[j]])), (var, j)
        if var == "refine":                         # exact re-rank of the oracle's k * rf candidates
            oi, od, oc = oracle(k * rf)
            for i, qi in enumerate(sel):
                cand = oi[i, :oc[i]].astype(np.int64)
                ex = np.array([ob.l2(q[qi], data[c]) for c in cand], np.float32)
                order = np.lexsort((cand, ex))[:k]
                assert _same(got[1][qi, :len(order)], ex[order]), (var, qi)
                assert np.array_equal(got[0][qi, :len(order)].astype(np.int64), cand[order]), (var, qi)
            continue
        extra = {"mask": {"allow": allow}, "range": {"lower": lo, "upper": hi}}.get(var, {})
        oi, od, oc = oracle(k, **extra)
        for i, qi in enumerate(sel):
            c = int(oc[i])
            _check_topk(got[0][qi, :c], got[1][qi, :c], oi[i, :c], od[i, :c])
            assert np.isinf(got[1][qi, c:]).all(), (var, qi)
    # the second slab really has queries whose k-th distance is tied (the device replays those slots)
    oi, od, oc = oracle(k + 1)
    second = sel >= SLAB
    assert np.any((od[second, k - 1] == od[second, k]) & np.isfinite(od[second, k]))
    # one scan launch per slab
    prof = _profiled(lambda: ix.search_ex(q, k=k, nprobes=nprobes))
    assert _launches(prof, SCAN_LAUNCH.get(name, "search:pq_scan")) == 2, prof


# ---- 6. one natural-size case: no knobs, the default chunk rule gives three chunks ----------------------------
def test_natural_row_chunks_u8_1536(make_src):
    n, d, K, M = 400_000, 1536, 32, 192
    chunk = (1 << 28) // d                          # rows_per_chunk(): 174 762 rows -> chunks of 174 762, 174 762, 50 476
    rng = np.random.default_rng(600)
    cent = rng.uniform(40, 215, (K, d)).astype(np.float32)
    pool = np.clip(np.rint(cent[rng.integers(0, K, 8192)] + rng.standard_normal((8192, d)).astype(np.float32) * 12),
                   0, 255).astype(np.uint8)
    cb = (rng.standard_normal((M, 256, d // M)) * 6).astype(np.float32)
    pin = lb.PinnedArray((n, d), np.uint8)
    pick = rng.integers(0, len(pool), n)
    for s in range(0, n, 1 << 16):
        pin.array[s:s + (1 << 16)] = pool[pick[s:s + (1 << 16)]]
    try:
        rows = np.unique(np.concatenate([np.arange(b - 64, b + 64) for b in (chunk, 2 * chunk)] +
                                        [rng.choice(n, 2000, replace=False)]))
        x32 = pin.array[rows].astype(np.float32)
        po, do, vo = ob.compute_membership(cent, x32, nthreads=NT)
        co = ob.pq_encode(cb, ob.compute_residual(cent, x32, po, nthreads=NT), nthreads=NT)
        dev = lb.DeviceArray.from_numpy(pin.array)
        for s in (dev, pin):
            p, dist, v = lb.compute_partitions(cent, s)
            assert v[rows].all() and np.array_equal(p[rows], po) and np.array_equal(dist[rows], do)
            tp, tc, tv = lb.ivfpq_transform(cent, cb, s)
            assert tv[rows].all() and np.array_equal(tp[rows], po) and np.array_equal(tc[rows], co)
        # three chunks: one u8 -> f32 conversion and one tensor-core assignment per chunk
        prof = _profiled(lambda: lb.compute_partitions(cent, dev))
        assert _launches(prof, "convert_to_f32") == 3 and _launches(prof, "tc_filter_general") == 3, prof
        dev.free()
    finally:
        pin.free()
