"""CPU checks of the IVF_RQ restatement (tests/rq_reference.py): the reference's own literals, the 16-bit table sums
against the reference's AVX-512 kernel, the Householder QR the device rotation implements, and the bound that
separates our exactly ordered data-side rotation from the reference's GEMM."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import binding as ob
from rq_reference import dist_table, dot16, pack_codes_block, pack_signs, quantize_table, rq_distances, seq_sum

REF_SO = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "libref_simd.so")


def test_dist_table_reference_literal():
    # test_build_dist_table_not_optimized (bq/storage.rs:779-787): the lowbit chain equals the subset sums
    sub = np.array([1.0, 2.0, 3.0, 4.0], np.float32)
    want = np.array([sum(sub[b] for b in range(4) if j >> b & 1) for j in range(16)], np.float32)
    assert np.array_equal(dist_table(sub)[0], want)


def test_sign_packing_reference_literal():
    # test_binary_quantization (bq.rs:112-128): bit j of byte j / 8 is the sign of element j, LSB first
    data = np.array([1.0, -1.0, 1.0, -5.0, -7.0, -1.0, 1.0, -1.0, -0.2, 1.2, 3.2], np.float32)
    assert pack_signs(data).tolist() == [0b01000101, 0b00000110]
    # is_sign_positive: +0.0 -> 1, -0.0 -> 0
    assert pack_signs(np.array([0.0, -0.0, 0, 0, 0, 0, 0, 0], np.float32)).tolist() == [0b11111101]


@pytest.mark.parametrize("d", [1, 8, 15, 16, 17, 120, 128, 1032])
def test_rotation_is_the_oracle_dot(d):
    rng = np.random.default_rng(d)
    X = rng.standard_normal((5, d)).astype(np.float32)
    R = rng.standard_normal((7, d)).astype(np.float32)
    got = dot16(X, R)
    want = np.array([[ob.dot(R[j], X[m]) for j in range(7)] for m in range(5)], np.float32)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def test_quantised_sums_wrap_like_the_avx512_kernel():
    """the model of distance_all's u8 table sums -- a u32 sum & 0xffff -- against dist_table.c, past code_dim = 1024
    where the 16-bit lanes wrap (the scalar fallback would saturate instead)"""
    if not os.path.exists(REF_SO):
        pytest.skip("oracle/_ref/libref_simd.so was not built (the reference's sources are not present)")
    if "avx512bw" not in open("/proc/cpuinfo").read():
        pytest.skip("the CPU has no AVX-512")
    L = C.CDLL(REF_SO)
    fn = L.sum_4bit_dist_table_32bytes_batch_avx512
    fn.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
    rng = np.random.default_rng(0)
    wrapped = 0
    for code_dim in (64, 1024, 2048, 4096):
        cb = code_dim // 8
        for trial in range(3):
            codes = rng.integers(0, 256, size=(32, cb), dtype=np.uint8)
            table = rng.integers(200 if trial else 0, 256, size=(code_dim // 4, 16), dtype=np.uint8)
            packed = pack_codes_block(codes)
            out = np.zeros(32, np.uint16)
            fn(packed.ctypes.data, packed.size, table.ctypes.data, out.ctypes.data)
            i2 = np.arange(cb)
            full = (table[2 * i2, codes & 15].astype(np.int64) + table[2 * i2 + 1, codes >> 4]).sum(axis=1)
            assert np.array_equal(out, (full & 0xFFFF).astype(np.uint16)), (code_dim, trial)
            wrapped += int((full > 0xFFFF).sum())
            if code_dim <= 1024:   # below the wrap the scalar fallback agrees
                sat = ob.sum_4bit_dist_table(32, cb, packed, table.ravel())
                assert np.array_equal(sat, out)
    assert wrapped > 0


def test_distance_all_rows_and_tail():
    """the first n - n % 32 rows go through the u8 table, the rest are exact; every row is exact with a mask"""
    rng = np.random.default_rng(3)
    rq = rng.standard_normal(128).astype(np.float32)
    codes = rng.integers(0, 256, size=(70, 16), dtype=np.uint8)
    add, scale = rng.random(70, dtype=np.float32), rng.random(70, dtype=np.float32)
    a = rq_distances(rq, codes, add, scale, 0.25)
    e = rq_distances(rq, codes, add, scale, 0.25, exact_all=True)
    assert np.array_equal(a[64:], e[64:]) and not np.array_equal(a[:64], e[:64])
    assert np.allclose(a, e, rtol=0.05, atol=0.5)
    t = dist_table(rq)
    qmin, qmax, qt = quantize_table(t)
    assert qt.min() == 0 and qt.max() == 255 and qmin == t.min() and qmax == t.max()
    assert not quantize_table(np.zeros((4, 16), np.float32))[2].any()


def _householder(a):
    """householder_qr (bq/builder.rs:314-357) with each reflection applied as a rank-1 update, as the device does"""
    r = a.copy()
    n = r.shape[0]
    q = np.eye(n)
    for k in range(n - 1):
        x = r[k:, k].copy()
        xn = np.sqrt(x @ x)
        if xn < np.finfo(np.float64).eps:
            continue
        x[0] += (1.0 if x[0] >= 0 else -1.0) * xn
        u = x / np.sqrt(x @ x)
        r[k:, k:] -= 2.0 * np.outer(u, u @ r[k:, k:])
        q[:, k:] -= 2.0 * np.outer(q[:, k:] @ u, u)
    return q, r


@pytest.mark.parametrize("n", [8, 16, 32])
def test_householder_properties(n):
    # test_householder_qr (bq/builder.rs:375-412)
    a = np.random.default_rng(n).standard_normal((n, n))
    q, r = _householder(a)
    assert np.allclose(q.T @ q, np.eye(n), atol=1e-5, rtol=0)
    assert np.allclose(q @ r, a, atol=1e-5, rtol=0)
    assert np.allclose(np.tril(r, -1), 0, atol=1e-5, rtol=0)


@pytest.mark.parametrize("d", [16, 128, 1024])
def test_code_bits_differ_from_any_summation_order_only_below_the_rounding_bound(d):
    """Any f32 evaluation of dot(R[j], r) -- the restatement's 16 lanes, or the reference's GEMM in whatever order --
    lies within gamma_d * sum_k |R_jk r_k| of the exact value (gamma_d = d u / (1 - d u), u = 2^-24).  So a code bit
    can only differ between two orders where the exact |rot[j]| is below that bound."""
    rng = np.random.default_rng(d)
    q, _ = _householder(rng.standard_normal((d, d)))
    R = q.astype(np.float32)
    r = rng.standard_normal((64, d)).astype(np.float32)
    r[:8] *= np.float32(1e-3)
    r[8, :] = R[3] * np.float32(1e-2)                   # orthogonal to every other row: tiny components
    rot = dot16(r, R)
    exact = r.astype(np.float64) @ R.astype(np.float64).T
    mag = np.abs(r.astype(np.float64)) @ np.abs(R.astype(np.float64)).T
    u = 2.0 ** -24
    gamma = d * u / (1 - d * u)
    assert (np.abs(rot - exact) <= gamma * mag).all()
    flips = np.signbit(rot) != np.signbit(exact)
    assert (np.abs(exact[flips]) <= gamma * mag[flips]).all()
    # the packed codes: f32 order against the f64 rotation, bit for bit outside the bound
    sure = np.abs(exact) > gamma * mag
    assert np.array_equal(pack_signs(np.where(sure, rot, 1.0)), pack_signs(np.where(sure, exact, 1.0).astype(np.float32)))


def test_sequential_sums_start():
    # Rust's float Sum starts from -0.0: only an all -0.0 sum keeps the sign
    assert np.signbit(seq_sum(np.array([-0.0, -0.0], np.float32), start=-0.0))
    assert not np.signbit(seq_sum(np.array([-0.0, -0.0], np.float32), start=0.0))
