"""The stand-alone lance-linalg entry points of the C ABI at every element type, against the oracle:
`lb2_distance_batch`, `lb2_normalize`, `lb2_find_partitions` and `lb2_compute_residual`.

Every call passes the caller's own element type (bf16 as uint16 bit patterns) straight to the C ABI, and every
expectation is computed on the values the reference sees:
  * distances (`l2_distance_batch` / `dot_distance_batch`, l2.rs:194-203, dot.rs:164-172) BIT FOR BIT with the
    oracle's function for that type: f32 and 16-bit L2 and f32 dot take 16 f32 lanes (l2.rs:57-91,100-106,
    dot.rs:30-58), 16-bit dot takes 32 lanes with the d % 32 tail first (dot.rs:78-83,133), u8 sums are exact u32
    sums converted to f32 once (l2.rs:44-49, dot.rs:152-161);
  * cosine within a derived bound of an f64 evaluation (the reference's own order depends on the ISA);
  * normalisation and residuals as one f32 operation per element, rounded once to the model type;
  * probe selection as the oracle's `find_partitions` on the f32 values (16 lanes for every type: k-means and the
    IVF probes use the same rule, a documented divergence for 16-bit dot).

Routes of `lb2_distance_batch` (f32 L2 / dot and 16-bit L2 reuse the assignment kernels with `from` as the one row
and `to` as n centroids): the tile kernel for d % 16 == 0, d <= 256 and a 16-byte aligned `from`; the generic kernel
with 16 rows per CTA up to 96 KB of rows (d <= 1536), with 8 rows above that.  u8 and 16-bit dot take the typed
half-warp-per-row kernel (`distance_batch`)."""
import ctypes as C
import math
import os

import numpy as np
import pytest

import lance_b200 as lb
from lance_b200 import _lib
from oracle import binding as ob

gpu = pytest.mark.gpu
REF_SO = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "libref_simd.so")
DT = {"f32": _lib.F32, "f16": _lib.F16, "bf16": _lib.BF16, "u8": _lib.U8}
METRIC = {"l2": _lib.L2, "cosine": _lib.COSINE, "dot": _lib.DOT}
DTYPES = ["f32", "f16", "bf16", "u8"]
# An H100 block may opt in to 227 KB (232,448 bytes) of shared memory.  The 8-row generic kernel keeps 8 rows of d f32
# there: as lb2_distance_batch runs it (every distance written out, no static shared memory) 32 d <= 232,448 ->
# d <= 7264; as the assignment runs it, its per-half-warp argmin scratch (3 x 16 x 8 x 4 = 1,536 bytes of static shared
# memory) counts against the same limit: 32 d + 1,536 <= 232,448 -> d <= 7216
D_MAX_GENERIC = 7264
D_MAX_ASSIGN = 7216


# ---- element types ---------------------------------------------------------------------------------------------
def _bf16_bits(x):
    """f32 -> bfloat16 bit patterns (uint16), round to nearest even; NaN stays a quiet NaN."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    b = x.view(np.uint32).astype(np.uint64)
    r = ((b + 0x7FFF + ((b >> 16) & 1)) >> 16).astype(np.uint16)
    return np.where(np.isnan(x), np.uint16(0x7FC0), r)


def _bf16_f32(bits):
    return (np.asarray(bits, dtype=np.uint32) << 16).view(np.float32)


def _native(x, dt):
    """f32 values -> the caller's element type (bf16 as uint16 bit patterns; u8 values are taken as they are)."""
    if dt == "f16":
        return x.astype(np.float16)
    if dt == "bf16":
        return _bf16_bits(x)
    if dt == "u8":
        return x.astype(np.uint8)
    return x.astype(np.float32)


def _f32(a, dt):
    """the exact f32 value of every element of a native array"""
    return _bf16_f32(a) if dt == "bf16" else np.asarray(a).astype(np.float32)


def _model(x32, dt):
    """f32 results -> the model type, rounded once to nearest even (f16 / bf16 keep their type, u8's model is f32)"""
    return _native(x32, dt) if dt in ("f16", "bf16") else x32.astype(np.float32)


def _model_np(dt):
    return {"f32": np.float32, "f16": np.float16, "bf16": np.uint16, "u8": np.float32}[dt]


def _rows(rng, n, d, dt):
    if dt == "u8":
        return rng.integers(0, 256, (n, d), dtype=np.uint8)
    return _native(rng.standard_normal((n, d)).astype(np.float32), dt)


def _assert_bits(got, want, what):
    """same bits everywhere, NaN where the expectation is NaN (any NaN)"""
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape and got.dtype == want.dtype, (what, got.shape, want.shape, got.dtype, want.dtype)
    g32, w32 = got.astype(np.float32), want.astype(np.float32)
    gn, wn = np.isnan(g32), np.isnan(w32)
    ub = np.uint16 if got.itemsize == 2 else np.uint32
    bad = (gn != wn) | (~wn & (np.ascontiguousarray(got).view(ub) != np.ascontiguousarray(want).view(ub)))
    if bad.any():
        i = np.unravel_index(int(np.argmax(bad)), bad.shape)
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.size} values differ; first at {i}: "
                             f"got {g32[i]!r}, want {w32[i]!r}")


# ---- the C ABI, called with raw buffers ----------------------------------------------------------------------------
def _ptr(a):
    """numpy array (pageable), PinnedArray, DeviceArray, or (DeviceArray, byte offset) -> (c_void_p, keepalive)"""
    if isinstance(a, tuple):
        return C.c_void_p(a[0].ptr + a[1]), a
    if isinstance(a, (lb.DeviceArray, lb.PinnedArray)):
        return C.c_void_p(a.ptr), a
    a = np.ascontiguousarray(a)
    return C.c_void_p(a.ctypes.data), a


def _status(st):
    if st == _lib.OK:
        return
    _lib.check(st)


def _distance_batch(frm, to, n, d, dt, metric, check=True):
    out = np.full(n, np.float32(-7.0), np.float32)
    fp, _k1 = _ptr(frm)
    tp, _k2 = _ptr(to)
    st = _lib.lib().lb2_distance_batch(fp, tp, C.c_uint64(n), C.c_uint32(d), C.c_int(DT[dt]), C.c_int(METRIC[metric]),
                                       C.c_void_p(out.ctypes.data))
    if check:
        _status(st)
        return out
    return st, out


def _profiled(fn):
    lb.profile.reset()
    lb.profile.enable(True)
    try:
        out = fn()
    finally:
        lb.profile.enable(False)
    return out, lb.profile.dump()


# ---- expectations --------------------------------------------------------------------------------------------------
_ORACLE = {("f32", "l2"): ob.l2, ("f16", "l2"): ob.l2_f16, ("bf16", "l2"): ob.l2_bf16, ("u8", "l2"): ob.l2_u8,
           ("f32", "dot"): ob.dot, ("f16", "dot"): ob.dot_f16, ("bf16", "dot"): ob.dot_bf16, ("u8", "dot"): ob.dot_u8}


def _oracle_rows(frm, rows, dt, metric):
    """the oracle's distance of `frm` to every row, in the caller's element type; dot distance = 1 - dot in f32"""
    f = _ORACLE[dt, metric]
    v = np.array([f(frm, r) for r in rows], np.float32).reshape(len(rows))
    return v if metric == "l2" else (np.float32(1.0) - v).astype(np.float32)


def _lanes_np(x, Y, lanes, metric):
    """dot_scalar / l2_scalar::<_, f32, LANES> (dot.rs:30-58, l2.rs:57-91) for every row of Y at once: x [d], Y [n, d]
    f32; the d % LANES tail summed first, lane accumulators over the full chunks, folded 0..LANES-1.  numpy rounds every
    f32 operation on its own (no contraction)."""
    x, Y = np.asarray(x, np.float32), np.asarray(Y, np.float32)
    n, d = Y.shape
    full = d // lanes * lanes

    def term(a, b):
        return (a - b) * (a - b) if metric == "l2" else a * b

    s = np.zeros(n, np.float32)
    for i in range(full, d):
        s = s + term(x[i], Y[:, i])
    acc = np.zeros((n, lanes), np.float32)
    for c in range(0, full, lanes):
        acc = acc + term(x[c:c + lanes], Y[:, c:c + lanes])
    t = np.zeros(n, np.float32)
    for q in range(lanes):
        t = t + acc[:, q]
    v = s + t
    return v if metric == "l2" else (np.float32(1.0) - v).astype(np.float32)


def _u8_np(x, Y, metric, chunk=8192):
    """l2_distance_uint_scalar / the u8 dot (l2.rs:44-49, dot.rs:152-161): the u32 sum (wrapping) converted to f32
    once; the int64 sum mod 2^32 is exact, and it goes through f64 (exact) to one f32 rounding."""
    x = np.asarray(x, np.int64)
    out = np.empty(len(Y), np.float32)
    for r0 in range(0, len(Y), chunk):
        Z = np.asarray(Y[r0:r0 + chunk], np.int64)
        s = ((x - Z) ** 2).sum(1) if metric == "l2" else (x * Z).sum(1)
        out[r0:r0 + chunk] = (s & 0xFFFFFFFF).astype(np.float64).astype(np.float32)
    return out if metric == "l2" else (np.float32(1.0) - out).astype(np.float32)


def _restated(frm, rows, dt, metric):
    """the per-type rule of the reference, vectorised over rows"""
    if dt == "u8":
        return _u8_np(frm, rows, metric)
    lanes = 32 if (metric == "dot" and dt in ("f16", "bf16")) else 16
    return _lanes_np(_f32(frm, dt), _f32(rows, dt), lanes, metric)


# ---- 1. lb2_distance_batch: L2 / dot bit for bit ---------------------------------------------------------------------
DIMS = [1, 5, 15, 16, 17, 31, 32, 33, 100, 128, 256, 272, 768, 1536, 1552, 2048]
NS = [0, 1, 63, 64, 65, 4097]


@gpu
@pytest.mark.parametrize("d", DIMS)
@pytest.mark.parametrize("metric", ["l2", "dot"])
@pytest.mark.parametrize("dt", DTYPES)
def test_distance_batch_matches_oracle_bit_for_bit(dt, metric, d):
    rng = np.random.default_rng(9100 + d + 131 * DTYPES.index(dt) + 17 * (metric == "dot"))
    frm = _rows(rng, 1, d, dt)[0]
    to = _rows(rng, max(NS), d, dt)
    want = _oracle_rows(frm, to, dt, metric)
    for n in NS:
        got = _distance_batch(frm, to[:n], n, d, dt, metric)
        _assert_bits(got, want[:n], (dt, metric, d, n))


def test_restatement_equals_oracle_per_row():
    """The vectorised restatement that checks the 10^5-row case is the oracle's per-row rule (CPU only)."""
    rng = np.random.default_rng(9200)
    for dt in DTYPES:
        for metric in ("l2", "dot"):
            for d in (1, 5, 16, 17, 31, 32, 33, 100, 1040):
                frm = _rows(rng, 1, d, dt)[0]
                to = _rows(rng, 40, d, dt)
                _assert_bits(_restated(frm, to, dt, metric), _oracle_rows(frm, to, dt, metric), (dt, metric, d))
    # the restatement tells the rules apart: 32 vs 16 lanes on bf16 dot, integer vs f32 sums on u8 at d = 2048
    frm, to = _rows(rng, 1, 128, "bf16")[0], _rows(rng, 200, 128, "bf16")
    assert np.sum(_restated(frm, to, "bf16", "dot") != _lanes_np(_f32(frm, "bf16"), _f32(to, "bf16"), 16, "dot")) > 20
    frm, to = _rows(rng, 1, 2048, "u8")[0], _rows(rng, 200, 2048, "u8")
    assert np.sum(_restated(frm, to, "u8", "dot") != _lanes_np(_f32(frm, "u8"), _f32(to, "u8"), 16, "dot")) > 20


@gpu
@pytest.mark.parametrize("dt", DTYPES)
def test_distance_batch_100k_rows(dt):
    """About 10^5 rows against the vectorised restatement of each lane rule (checked against the oracle above)."""
    rng = np.random.default_rng(9300 + DTYPES.index(dt))
    n, d = 100_003, (1040 if dt == "u8" else 100)   # u8: sums past 2^24, where an f32 sum would round
    frm, to = _rows(rng, 1, d, dt)[0], _rows(rng, n, d, dt)
    for metric in ("l2", "dot"):
        _assert_bits(_distance_batch(frm, to, n, d, dt, metric), _restated(frm, to, dt, metric), (dt, metric, n))


# ---- 2. cosine: within a derived bound of f64 ----------------------------------------------------------------------
def _cosine_bound(x, Y):
    """Error bound of the device's cosine 1 - <x, y> / sqrt(<x, x>) / sqrt(<y, y>) on f32 values.  Each of the three
    sums is a 32-lane FMA chain of ceil(d / 32) steps followed by a 5-level shuffle tree, so every product term passes
    through at most n = ceil(d / 32) + 5 roundings: |<x, y>~ - <x, y>| <= g_n S |x||y| with S = sum|x_i y_i| / (|x||y|)
    <= 1 and g_n = n u / (1 - n u), u = 2^-24 (Higham, eq. 3.5), and both squared norms carry a relative error <= g_n.
    The two square roots halve those and add u each; the two divisions add u each, so the ratio is off by at most
    (g_n + g_n / 2 + g_n / 2 + 4u) S <= 3 n u S for n >= 4, and 1 - r (a value in [0, 2]) adds at most u:
        B = 3 (ceil(d / 32) + 5) 2^-24 S + 2^-24."""
    d = Y.shape[-1]
    x64, Y64 = np.asarray(x, np.float64), np.asarray(Y, np.float64)
    with np.errstate(invalid="ignore", divide="ignore"):   # zero vectors: NaN, checked apart
        s = np.abs(x64 * Y64).sum(-1) / (np.linalg.norm(x64) * np.linalg.norm(Y64, axis=-1))
    return 3.0 * (math.ceil(d / 32) + 5) * 2.0 ** -24 * s + 2.0 ** -24


def _cosine64(x, Y):
    x64, Y64 = np.asarray(x, np.float64), np.asarray(Y, np.float64)
    with np.errstate(invalid="ignore", divide="ignore"):
        return 1.0 - (Y64 @ x64) / (np.linalg.norm(x64) * np.linalg.norm(Y64, axis=-1))


@gpu
@pytest.mark.parametrize("d", [1, 5, 16, 33, 100, 768, 1552, 2048])
@pytest.mark.parametrize("dt", DTYPES)
def test_distance_batch_cosine_within_bound_of_f64(dt, d):
    rng = np.random.default_rng(9400 + d + 7 * DTYPES.index(dt))
    frm, to = _rows(rng, 1, d, dt)[0], _rows(rng, 4097, d, dt)
    to[3] = 0                                      # a zero row: 1 - 0 / 0 is NaN in the reference too
    x32, Y32 = _f32(frm, dt), _f32(to, dt)
    ok = np.any(Y32 != 0, axis=1) & np.any(x32 != 0)
    ex, bnd = _cosine64(x32, Y32), _cosine_bound(x32, Y32)
    for n in (0, 1, 65, 4097):
        got = _distance_batch(frm, to[:n], n, d, dt, "cosine")
        assert np.array_equal(np.isnan(got), ~ok[:n]), (dt, d, n)
        err = np.abs(got[ok[:n]].astype(np.float64) - ex[:n][ok[:n]])
        assert np.all(err <= bnd[:n][ok[:n]]), (dt, d, n, float(np.max(err / bnd[:n][ok[:n]])))
    zero = np.zeros_like(frm)
    assert np.all(np.isnan(_distance_batch(zero, to[:65], 65, d, dt, "cosine"))), (dt, d)


def test_cosine_bound_holds_for_the_oracle():
    """The bound is not loose by construction: the oracle's f32 cosine (16 lanes, fewer roundings) stays inside it."""
    rng = np.random.default_rng(9450)
    for d in (5, 100, 768):
        x, Y = rng.standard_normal(d).astype(np.float32), rng.standard_normal((64, d)).astype(np.float32)
        got = np.array([ob.cosine(x, y) for y in Y], np.float64)
        assert np.all(np.abs(got - _cosine64(x, Y)) <= _cosine_bound(x, Y)), d
    assert 3.0 * (math.ceil(128 / 32) + 5) * 2.0 ** -24 + 2.0 ** -24 < 1.7e-6


# ---- 3. routes, residency and refusals ------------------------------------------------------------------------------
def _ran(prof, name):
    return prof.get(name, (0, 0))[0]


@gpu
@pytest.mark.parametrize("metric", ["l2", "dot"])
@pytest.mark.parametrize("d", [128, 256])
def test_distance_batch_unaligned_from_takes_generic_kernel_with_same_bits(d, metric):
    """A `from` one f32 past a 16-byte boundary cannot feed the tile kernel's float4 loads: it takes the generic
    kernel, which must return the aligned call's bits."""
    rng = np.random.default_rng(9500 + d)
    frm, to = _rows(rng, 1, d, "f32")[0], _rows(rng, 4097, d, "f32")
    buf = lb.DeviceArray.from_numpy(np.concatenate([np.zeros(1, np.float32), frm]))
    try:
        al, pa = _profiled(lambda: _distance_batch(frm, to, 4097, d, "f32", metric))
        un, pu = _profiled(lambda: _distance_batch((buf, 4), to, 4097, d, "f32", metric))
    finally:
        buf.free()
    assert _ran(pa, "assign_exact") == 1 and _ran(pa, "assign_exact_generic") == 0, pa
    assert _ran(pu, "assign_exact_generic") == 1 and _ran(pu, "assign_exact") == 0, pu
    _assert_bits(un, al, ("unaligned vs aligned", d, metric))
    _assert_bits(al, _oracle_rows(frm, to, "f32", metric), ("aligned vs oracle", d, metric))


@gpu
def test_distance_batch_routes_by_element_type():
    rng = np.random.default_rng(9550)
    d = 128
    for dt, metric, kern in (("f32", "l2", "assign_exact"), ("f32", "dot", "assign_exact"),
                             ("f16", "l2", "assign_exact"), ("bf16", "l2", "assign_exact"),
                             ("f16", "dot", "distance_batch"), ("bf16", "dot", "distance_batch"),
                             ("u8", "l2", "distance_batch"), ("u8", "dot", "distance_batch")):
        frm, to = _rows(rng, 1, d, dt)[0], _rows(rng, 65, d, dt)
        got, prof = _profiled(lambda: _distance_batch(frm, to, 65, d, dt, metric))
        assert _ran(prof, kern) == 1, (dt, metric, prof)
        _assert_bits(got, _oracle_rows(frm, to, dt, metric), (dt, metric))


@gpu
@pytest.mark.parametrize("metric", ["l2", "dot"])
def test_distance_batch_generic_kernel_shared_memory_limit(metric):
    """Up to D_MAX_GENERIC the 8-row generic kernel serves f32 and 16-bit L2 (and f32 dot); one more dimension is
    refused with LB2_UNSUPPORTED before anything is launched.  The typed kernel (u8, 16-bit dot) has no such limit."""
    rng = np.random.default_rng(9600 + (metric == "dot"))
    dts = ["f32", "bf16"] if metric == "l2" else ["f32"]
    for dt in dts:
        for d in (D_MAX_GENERIC, D_MAX_GENERIC + 1):
            frm, to = _rows(rng, 1, d, dt)[0], _rows(rng, 65, d, dt)
            if d == D_MAX_GENERIC:
                _assert_bits(_distance_batch(frm, to, 65, d, dt, metric), _oracle_rows(frm, to, dt, metric), (dt, d))
                continue
            st, _ = _distance_batch(frm, to, 65, d, dt, metric, check=False)
            assert st == _lib.UNSUPPORTED, (dt, metric, d, st)
    for dt in (["u8"] if metric == "l2" else ["u8", "f16", "bf16"]):
        d = D_MAX_GENERIC + 1
        frm, to = _rows(rng, 1, d, dt)[0], _rows(rng, 65, d, dt)
        _assert_bits(_distance_batch(frm, to, 65, d, dt, metric), _oracle_rows(frm, to, dt, metric), (dt, d))


@gpu
def test_assignment_generic_kernel_limit_counts_static_shared_memory():
    """lb2_compute_partitions on fewer than 256 rows takes the exact kernels; above d = 256 the generic one, 8 rows per
    CTA past 96 KB.  Its static argmin scratch leaves room for d <= D_MAX_ASSIGN; one more is refused before any
    launch instead of failing in cudaFuncSetAttribute."""
    rng = np.random.default_rng(9650)
    for d in (D_MAX_ASSIGN, D_MAX_ASSIGN + 1):
        cent, x = rng.standard_normal((5, d)).astype(np.float32), rng.standard_normal((9, d)).astype(np.float32)
        part, dist, valid = np.empty(9, np.uint32), np.empty(9, np.float32), np.empty(9, np.uint8)
        st = _lib.lib().lb2_compute_partitions(_ptr(cent)[0], C.c_uint32(5), C.c_uint32(d), C.c_int(_lib.F32),
                                               C.c_int(_lib.L2), _ptr(x)[0], C.c_uint64(9),
                                               C.c_void_p(part.ctypes.data), C.c_void_p(dist.ctypes.data),
                                               C.c_void_p(valid.ctypes.data))
        if d == D_MAX_ASSIGN:
            _status(st)
            ids, dists, _ = ob.compute_membership(cent, x)
            assert np.array_equal(part, ids) and np.array_equal(dist, dists) and valid.all()
        else:
            assert st == _lib.UNSUPPORTED, st


@gpu
@pytest.mark.parametrize("where", ["device", "pinned", "pageable"])
def test_distance_batch_to_buffer_residency(where):
    rng = np.random.default_rng(9700)
    for dt, metric, d in (("f32", "l2", 128), ("f16", "l2", 100), ("bf16", "dot", 100), ("u8", "dot", 300)):
        frm, to = _rows(rng, 1, d, dt)[0], _rows(rng, 4097, d, dt)
        if where == "device":
            buf = lb.DeviceArray.from_numpy(to)
        elif where == "pinned":
            buf = lb.PinnedArray(to.shape, to.dtype)
            buf.array[...] = to
        else:
            buf = to
        try:
            got = _distance_batch(frm, buf, len(to), d, dt, metric)
        finally:
            if where != "pageable":
                buf.free()
        _assert_bits(got, _oracle_rows(frm, to, dt, metric), (where, dt, metric, d))


# ---- 4. u8 edges and non-finite values ------------------------------------------------------------------------------
@gpu
def test_u8_reference_literal_and_u32_wrap():
    # l2.rs:433-438: 2048 zeros against 2048 x 255 is (255^2 * 2048) as f32, both ways round
    z, f = np.zeros(2048, np.uint8), np.full(2048, 255, np.uint8)
    want = np.float32(255 ** 2 * 2048)
    assert _distance_batch(z, f, 1, 2048, "u8", "l2")[0] == want
    assert _distance_batch(f, z, 1, 2048, "u8", "l2")[0] == want
    assert _distance_batch(z, z, 1, 2048, "u8", "l2")[0] == 0.0
    # d = 66,052: 66,052 * 255^2 = 4,295,031,300 passes 2^32 and wraps to 64,004, as the reference's release build's
    # u32 sum (and the oracle) does; L2 of 255 against 0, dot of 255 against 255
    d = 66_052
    wrapped = 66_052 * 255 ** 2 - 2 ** 32
    assert wrapped == 64_004
    z, f = np.zeros(d, np.uint8), np.full(d, 255, np.uint8)
    assert _distance_batch(f, z, 1, d, "u8", "l2")[0] == np.float32(wrapped) == np.float32(ob.l2_u8(f, z))
    assert _distance_batch(f, f, 1, d, "u8", "dot")[0] == np.float32(1 - wrapped) == np.float32(1) - np.float32(ob.dot_u8(f, f))
    rows = np.stack([z, f, np.full(d, 17, np.uint8)])
    for metric in ("l2", "dot"):
        _assert_bits(_distance_batch(f, rows, 3, d, "u8", metric), _oracle_rows(f, rows, "u8", metric), metric)


@gpu
@pytest.mark.parametrize("metric", ["l2", "dot"])
@pytest.mark.parametrize("dt", ["f32", "f16", "bf16"])
def test_distance_batch_non_finite_values(dt, metric):
    rng = np.random.default_rng(9800 + DTYPES.index(dt))
    for d in (17, 33, 128):
        x = rng.standard_normal((130, d)).astype(np.float32)
        specials = np.array([np.nan, np.inf, -np.inf], np.float32)
        for r in range(1, 130, 3):
            x[r, rng.integers(0, d)] = specials[(r // 3) % 3]
        frm = x[0].copy()
        frm[rng.integers(0, d)] = np.inf          # +inf in `from`: inf - inf and 0 * inf on some rows
        nat_f, nat_t = _native(frm, dt), _native(x[1:], dt)
        want = _oracle_rows(nat_f, nat_t, dt, metric)
        assert np.isnan(want).any() and np.isinf(want).any()
        _assert_bits(_distance_batch(nat_f, nat_t, len(nat_t), d, dt, metric), want, (dt, metric, d))


@gpu
@pytest.mark.skipif(not os.path.exists(REF_SO), reason="the reference's C kernels were not built (oracle/_ref)")
def test_f16_distances_against_reference_c_kernels():
    """l2_f16_avx2 / dot_f16_avx2 (built -ffast-math like lance-linalg/build.rs) reassociate freely: the device's f16
    L2 and dot agree with them within d * 2^-23 * sum|terms|, the bound test_oracle_dot_lanes uses."""
    ref = C.CDLL(REF_SO)
    for name in ("l2_f16_avx2", "dot_f16_avx2"):
        getattr(ref, name).restype = C.c_float
        getattr(ref, name).argtypes = [C.c_void_p, C.c_void_p, C.c_uint32]
    rng = np.random.default_rng(9850)
    for d in (8, 16, 100, 128, 130, 768):
        frm, to = _rows(rng, 1, d, "f16")[0], _rows(rng, 33, d, "f16")
        x64, Y64 = frm.astype(np.float64), to.astype(np.float64)
        l2 = _distance_batch(frm, to, 33, d, "f16", "l2")
        dd = _distance_batch(frm, to, 33, d, "f16", "dot")
        for i in range(len(to)):
            y = np.ascontiguousarray(to[i])
            r_l2 = float(ref.l2_f16_avx2(frm.ctypes.data, y.ctypes.data, d))
            r_dot = float(ref.dot_f16_avx2(frm.ctypes.data, y.ctypes.data, d))
            assert abs(r_l2 - float(l2[i])) <= d * 2.0 ** -23 * float(((x64 - Y64[i]) ** 2).sum()), (d, i)
            # the distance is 1 - dot rounded once more: half an ulp of a value below 1 + |dot|
            bound = d * 2.0 ** -23 * float(np.abs(x64 * Y64[i]).sum()) + 2.0 ** -24 * (1 + abs(r_dot))
            assert abs((1.0 - r_dot) - float(dd[i])) <= bound, (d, i)


# ---- 5. lb2_normalize ------------------------------------------------------------------------------------------------
def _normalize(x, n, d, dt):
    out = np.empty((n, d), _model_np(dt))
    xp, _k = _ptr(x)
    _status(_lib.lib().lb2_normalize(xp, C.c_uint64(n), C.c_uint32(d), C.c_int(DT[dt]), C.c_void_p(out.ctypes.data)))
    return out


@gpu
@pytest.mark.parametrize("d", [1, 3, 16, 100, 768, 1537])
@pytest.mark.parametrize("dt", DTYPES)
def test_normalize_every_element_type(dt, d):
    """kernels.rs:141-146 on the exact f32 values (the oracle's normalize_rows), the result rounded once to the model
    type; zero rows divide 0 by 0."""
    rng = np.random.default_rng(9900 + d + DTYPES.index(dt))
    x = _rows(rng, 70, d, dt)
    x[5] = 0
    x[69] = 0
    got = _normalize(x, 70, d, dt)
    want = _model(ob.normalize_rows(_f32(x, dt)), dt)
    assert got.dtype == want.dtype == _model_np(dt)
    if dt == "bf16":
        _assert_bf16(got, want, (dt, d))
    else:
        _assert_bits(got, want, (dt, d))
    assert np.all(np.isnan(_f32(got[[5, 69]], dt)))
    assert _normalize(x[:0], 0, d, dt).shape == (0, d)


def _assert_bf16(got, want, what):
    """bf16 bit patterns: equal, or both NaN"""
    gn, wn = np.isnan(_bf16_f32(got)), np.isnan(_bf16_f32(want))
    bad = (gn != wn) | (~wn & (got != want))
    assert not bad.any(), (what, int(bad.sum()), _bf16_f32(got[bad])[:4], _bf16_f32(want[bad])[:4])


# ---- 6. lb2_find_partitions ------------------------------------------------------------------------------------------
def _find_partitions(cent, K, d, dt, metric, q, nq, nprobes, check=True):
    ids = np.full((nq, nprobes), 0xDEADBEEF, np.uint32)
    dists = np.full((nq, nprobes), np.float32(-7.0), np.float32)
    cp, _k1 = _ptr(cent)
    qp, _k2 = _ptr(q)
    st = _lib.lib().lb2_find_partitions(cp, C.c_uint32(K), C.c_uint32(d), C.c_int(DT[dt]), C.c_int(METRIC[metric]),
                                        qp, C.c_uint64(nq), C.c_uint32(nprobes), C.c_void_p(ids.ctypes.data),
                                        C.c_void_p(dists.ctypes.data))
    if check:
        _status(st)
        return ids, dists
    return st, ids, dists


KS = [1, 2, 63, 64, 65, 300, 1024, 1025, 4096]


@gpu
@pytest.mark.parametrize("d", [100, 128, 272])      # 128: the tile kernel; 100 and 272: the generic kernel
@pytest.mark.parametrize("metric", ["l2", "dot"])
@pytest.mark.parametrize("dt", ["f32", "f16", "bf16"])
def test_find_partitions_matches_oracle(dt, metric, d):
    """Ids and distance bits of the oracle's find_partitions on the f32 values: ascending (distance, id), so
    duplicated centroids come out in ascending id order.  16-bit dot takes 16 lanes here, like k-means and the IVF
    probes (DESIGN.md records the divergence from the reference's 32)."""
    rng = np.random.default_rng(10000 + d + 3 * (metric == "dot") + 11 * len(dt))
    nq = 257
    q = _rows(rng, nq, d, dt)
    for K in KS:
        c32 = rng.standard_normal((K, d)).astype(np.float32)
        c32[1::7] = c32[0::7][:len(c32[1::7])]      # every 7th pair of centroids is one point twice: exact ties
        cent = _native(c32, dt)
        cf, qf = _f32(cent, dt), _f32(q, dt)
        full = [ob.find_partitions(cf, qf[i], K, metric) for i in range(nq)]
        for nprobes in sorted({1, (K + 1) // 2, K}):
            ids, dists = _find_partitions(cent, K, d, dt, metric, q, nq, nprobes)
            ids1, dists1 = _find_partitions(cent, K, d, dt, metric, q[:1], 1, nprobes)
            want_i = np.stack([f[0][:nprobes] for f in full])
            want_d = np.stack([f[1][:nprobes] for f in full])
            assert np.array_equal(ids, want_i), (dt, metric, d, K, nprobes)
            _assert_bits(dists, want_d, (dt, metric, d, K, nprobes))
            assert np.array_equal(ids1, want_i[:1]) and np.array_equal(dists1, dists[:1]), (dt, metric, d, K, nprobes)
        if K >= 2:   # the tie itself: centroid 1 is centroid 0, so wherever 0 is chosen 1 follows right after it
            for i in range(nq):
                r = int(np.flatnonzero(full[i][0] == 0)[0])
                assert full[i][0][r + 1] == 1 and full[i][1][r] == full[i][1][r + 1]


@gpu
def test_find_partitions_refusals_and_empty_batch():
    rng = np.random.default_rng(10100)
    cent, q = rng.standard_normal((10, 16)).astype(np.float32), rng.standard_normal((3, 16)).astype(np.float32)
    st, _, _ = _find_partitions(cent, 10, 16, "f32", "l2", q, 3, 11, check=False)
    assert st == _lib.INVALID_ARG
    for dt in ("f32", "f16", "bf16"):
        st, _, _ = _find_partitions(_native(cent, dt), 10, 16, dt, "cosine", _native(q, dt), 3, 4, check=False)
        assert st == _lib.INVALID_ARG, dt
    ids, dists = _find_partitions(cent, 10, 16, "f32", "l2", q[:0], 0, 4)
    assert ids.shape == (0, 4) and dists.shape == (0, 4)


# ---- 7. lb2_compute_residual ----------------------------------------------------------------------------------------
def _residual(cent, K, d, dt, x, n, part):
    out = np.empty((n, d), _model_np(dt))
    cp, _k1 = _ptr(cent)
    xp, _k2 = _ptr(x)
    pp, _k3 = _ptr(np.ascontiguousarray(part, np.uint32))
    _status(_lib.lib().lb2_compute_residual(cp, C.c_uint32(K), C.c_uint32(d), C.c_int(DT[dt]), xp, C.c_uint64(n), pp,
                                            C.c_void_p(out.ctypes.data)))
    return out


@gpu
@pytest.mark.parametrize("d", [1, 5, 16, 17, 100, 1537])
@pytest.mark.parametrize("dt", DTYPES)
def test_compute_residual_every_element_type(dt, d):
    """residual.rs:86-95,111-154: `*v - *cent` in the element type.  For f16 that is half's Sub, f32(x) - f32(c)
    rounded once to f16; f32 and u8 rows (converted to floating point, centroids f32) subtract in f32.  The reference
    has no bf16 residual (its match refuses the type); the product applies the f16 rule to bf16."""
    rng = np.random.default_rng(10200 + d + DTYPES.index(dt))
    K, n = 7, 300
    x = _rows(rng, n, d, dt)
    c32 = (rng.uniform(0, 255, (K, d)) if dt == "u8" else rng.standard_normal((K, d)) * 1.5).astype(np.float32)
    cent = _model(c32, dt)
    part = rng.integers(0, K, n).astype(np.uint32)
    want = _model(_f32(x, dt) - _f32(cent, dt)[part], dt)
    got = _residual(cent, K, d, dt, x, n, part)
    assert got.dtype == want.dtype == _model_np(dt)
    assert np.array_equal(got.view(np.uint16 if got.itemsize == 2 else np.uint32),
                          want.view(np.uint16 if want.itemsize == 2 else np.uint32)), (dt, d)
    assert _residual(cent, K, d, dt, x[:0], 0, part[:0]).shape == (0, d)


# ---- 8. the Python mirror keeps the element type -------------------------------------------------------------------
@gpu
def test_python_mirror_keeps_element_types():
    rng = np.random.default_rng(10300)
    d = 40
    for dt in DTYPES:
        bf = dt == "bf16"
        x = _rows(rng, 20, d, dt)
        cent = _model(rng.standard_normal((5, d)).astype(np.float32) * (100 if dt == "u8" else 1), dt)
        assert np.array_equal(lb.dot_distance_batch(x[0], x, d, bf16=bf), _oracle_rows(x[0], x, dt, "dot")), dt
        assert lb.normalize_fsl(x, bf16=bf).dtype == _model_np(dt)
        part = rng.integers(0, 5, 20).astype(np.uint32)
        r = lb.compute_residual(cent, x, part, bf16=bf)
        assert r.dtype == _model_np(dt) and np.array_equal(r, _residual(cent, 5, d, dt, x, 20, part)), dt
        if dt != "u8":
            ids, dists = lb.kmeans_find_partitions(cent, x, 3, "dot", bf16=bf)
            wi, wd = _find_partitions(cent, 5, d, dt, "dot", x, 20, 3)
            assert np.array_equal(ids, wi) and np.array_equal(dists, wd), dt
