"""PQ code assignment on rows the tensor-core filter must not decide: non-finite rows, and rows a few ulps
from the midpoint of two codewords (their TF32 scores tie within the error bound).  The filter path must give
the same codes as the exact path and the CPU oracle."""
import os

import numpy as np
import pytest

import lance_b200 as lb
from oracle import binding as ob

pytestmark = pytest.mark.gpu
NT = 16


def _both_paths(fn):
    os.environ.pop("LB2_DISABLE_TC", None)
    a = fn()
    os.environ["LB2_DISABLE_TC"] = "1"
    try:
        b = fn()
    finally:
        os.environ.pop("LB2_DISABLE_TC", None)
    return a, b


@pytest.mark.parametrize("n,d,M", [(4097, 128, 16), (3000, 384, 48)])
def test_tc_pq_encode_non_finite_and_midpoint_rows(n, d, M):
    rng = np.random.default_rng(n + d + 1)
    cb = (rng.standard_normal((M, 256, 8)) * 2).astype(np.float32)
    vec = (rng.standard_normal((n, d)) * 2).astype(np.float32)
    vec[10, 3] = np.nan
    vec[11, :] = np.nan
    vec[12, 9] = np.inf
    vec[13, d - 1] = -np.inf
    vec[14, :8] = np.float32(3e38)          # finite, but |r|^2 overflows
    # rows 100.. : every sub-vector within a few ulps of the midpoint of two codewords
    for i in range(64):
        row = 100 + i
        for m in range(M):
            a, b = rng.choice(256, 2, replace=False)
            mid = (cb[m, a] + cb[m, b]) / np.float32(2)
            steps = int(rng.integers(-3, 4))
            t = int(rng.integers(0, 8))
            for _ in range(abs(steps)):
                mid[t] = np.nextafter(mid[t], np.float32(np.inf if steps > 0 else -np.inf))
            vec[row, m * 8:(m + 1) * 8] = mid
    pq = lb.ProductQuantizer(M, 8, d, cb)
    c1, c2 = _both_paths(lambda: pq.quantize(vec))
    assert np.array_equal(c1, c2)
    assert np.array_equal(c1, ob.pq_encode(cb, vec, nthreads=NT))
