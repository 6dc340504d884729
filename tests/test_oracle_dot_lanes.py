"""The oracle's dot products for f16 / bf16 / u8 keys (oracle/lance_oracle.cc: lo_dot_f16, lo_dot_bf16, lo_dot_u8)
and its bf16 L2 binding, pinned to the reference's lane structure (lance-linalg/src/distance/dot.rs)."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import binding as ob

REF_SO = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "libref_simd.so")


def _bf16(x):
    b = np.asarray(x, np.float32).view(np.uint32)
    return ((b + 0x7FFF + ((b >> 16) & 1)) >> 16).astype(np.uint16)


def _bf16_f32(bits):
    return (np.asarray(bits, np.uint32) << 16).view(np.float32)


def _dot_lanes(x, y, lanes):
    """dot_scalar::<_, f32, LANES> (dot.rs:30-58) restated in numpy f32: tail first, then the lanes folded 0..L-1"""
    x, y = np.asarray(x, np.float32), np.asarray(y, np.float32)
    n = len(x) // lanes * lanes
    s = np.float32(0)
    for a, b in zip(x[n:], y[n:]):
        s = np.float32(s + np.float32(a * b))
    acc = np.zeros(lanes, np.float32)
    for c in range(0, n, lanes):
        acc = (acc + (x[c:c + lanes] * y[c:c + lanes]).astype(np.float32)).astype(np.float32)
    t = np.float32(0)
    for v in acc:
        t = np.float32(t + v)
    return np.float32(s + t)


def test_dot_known_answers():
    # dot.rs `test_dot`: (0..20) . (100..120) for f32 and f16; every partial sum is an exact integer
    x, y = np.arange(20), np.arange(100, 120)
    want = float(np.dot(x, y))
    assert want == 21470.0
    assert ob.dot(x, y) == want
    assert ob.dot_f16(x.astype(np.float16), y.astype(np.float16)) == want
    assert ob.dot_bf16(_bf16(x), _bf16(y)) == want
    assert ob.dot_u8(x.astype(np.uint8), y.astype(np.uint8)) == want
    # (0..512) . (100..612) in f32 is the test's second pair: within the reference's own bound of the f64 value
    x, y = np.arange(512, dtype=np.float32), np.arange(100, 612, dtype=np.float32)
    exact = float(np.dot(x.astype(np.float64), y.astype(np.float64)))
    assert abs(ob.dot(x, y) - exact) <= 2 * 2.0 ** -24 * 1023 * exact


def test_32_lanes_are_pinned():
    """x = y = [1, 2^-12, 0 ..., 2^-12 at 17, 0 ...]: with 16 lanes the two 2^-24 products share lane 1 and add up to
    2^-23, which survives the fold with 1; with 32 lanes each meets the 1 alone and rounds away (ties to even)."""
    x = np.zeros(32, np.float32)
    x[0], x[1], x[17] = 1.0, 2.0 ** -12, 2.0 ** -12
    assert ob.dot_f16(x.astype(np.float16), x.astype(np.float16)) == 1.0
    assert ob.dot_bf16(_bf16(x), _bf16(x)) == 1.0
    assert ob.dot(x, x) == np.float32(1.0 + 2.0 ** -23)        # the f32 dot: 16 lanes
    # random inputs: equal to the numpy restatement with 32 lanes, and often different from 16 lanes
    rng = np.random.default_rng(11)
    differ = 0
    for d in (1, 5, 31, 32, 33, 64, 100, 128, 130, 768):
        for _ in range(6):
            a = rng.standard_normal(d).astype(np.float16)
            b = rng.standard_normal(d).astype(np.float16)
            a32, b32 = a.astype(np.float32), b.astype(np.float32)
            got = ob.dot_f16(a, b)
            assert got == _dot_lanes(a32, b32, 32), d
            differ += got != _dot_lanes(a32, b32, 16)
            ab, bb = _bf16(a32), _bf16(b32)
            assert ob.dot_bf16(ab, bb) == _dot_lanes(_bf16_f32(ab), _bf16_f32(bb), 32), d
    assert differ >= 10, differ


def test_u8_dot_and_l2_are_exact_integer_sums():
    rng = np.random.default_rng(12)
    for d in (3, 128, 1536):
        x = rng.integers(0, 256, d, dtype=np.uint8)
        y = np.where(rng.random(d) < 0.5, 0, 255).astype(np.uint8)
        assert ob.dot_u8(x, y) == np.float32(int(np.dot(x.astype(np.int64), y.astype(np.int64))))
        assert ob.l2_u8(x, y) == np.float32(int(((x.astype(np.int64) - y) ** 2).sum()))
    # d = 1536, values spread over 0..255: the 16-lane f32 sum of the same squares rounds, the integer sum does not
    x = rng.integers(0, 256, (32, 1536), dtype=np.uint8)
    y = np.where(rng.random(1536) < 0.5, 0, 255).astype(np.uint8)
    assert any(ob.l2(r.astype(np.float32), y.astype(np.float32)) != ob.l2_u8(r, y) for r in x)


def test_l2_bf16_binding():
    rng = np.random.default_rng(13)
    for d in (7, 16, 130):
        a, b = _bf16(rng.standard_normal(d)), _bf16(rng.standard_normal(d))
        assert ob.l2_bf16(a, b) == ob.l2(_bf16_f32(a), _bf16_f32(b))   # each element converted, 16 lanes


@pytest.mark.skipif(not os.path.exists(REF_SO), reason="the reference's C kernels were not built (oracle/_ref)")
def test_dot_f16_against_reference_c_kernel():
    """dot_f16_avx2 (simd/f16.c, built -ffast-math like lance-linalg/build.rs) reassociates freely: it agrees with the
    32-lane restatement within the accumulation bound d * 2^-23 * sum|x_i y_i|."""
    ref = C.CDLL(REF_SO)
    ref.dot_f16_avx2.restype = C.c_float
    ref.dot_f16_avx2.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32]
    rng = np.random.default_rng(14)
    for d in (8, 16, 100, 128, 130, 768):
        a = rng.standard_normal(d).astype(np.float16)
        b = rng.standard_normal(d).astype(np.float16)
        r = float(ref.dot_f16_avx2(a.ctypes.data, b.ctypes.data, d))
        bound = d * 2.0 ** -23 * float(np.abs(a.astype(np.float64) * b).sum())
        assert abs(r - ob.dot_f16(a, b)) <= bound, d
