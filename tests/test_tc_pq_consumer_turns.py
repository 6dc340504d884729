"""PQ training through the tensor-core filter when the consumer warpgroups of a CTA get uneven shares of the
work.  The warpgroups take the (64-row tile, 4-sub-space chunk) items in turns, and chunks whose sub-spaces have
all converged are skipped.  Small row counts leave each CTA one to five items, so the last turn of a CTA leaves
zero to three warpgroups idle, and the skipped chunks shift the turns between iterations.  Codebooks and
iteration counts must equal the exact path and the CPU oracle."""
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


def _inputs(n, d=128, M=16):
    rng = np.random.default_rng(n)
    res = (rng.standard_normal((n, d)) * np.linspace(0.5, 4.0, d)).astype(np.float32)
    init = np.stack([res[rng.choice(n, 256, replace=False)][:, m * 8:(m + 1) * 8] for m in range(M)])
    # sub-spaces 0-3 (the whole first chunk) and 5: every row is one of the initial codewords, and each codeword
    # is used, so these converge within a few iterations while the others go on
    for m in (0, 1, 2, 3, 5):
        pick = np.concatenate([np.arange(256), rng.integers(0, 256, n - 256)])
        res[:, m * 8:(m + 1) * 8] = init[m][pick]
    return res, init


@pytest.mark.parametrize("n", [700, 4000, 6000, 9001])
def test_tc_pq_training_with_uneven_turns_and_converged_chunks(n):
    M, iters = 16, 10
    res, init = _inputs(n, M=M)
    (p1, p2) = _both_paths(lambda: lb.PQBuildParams(M, 8, max_iters=iters, codebook=init).build(res))
    assert p1.train_iters[:4].max() < p1.train_iters.max(), "the first chunk must converge before the others"
    assert np.array_equal(p1.train_iters, p2.train_iters) and np.array_equal(p1.codebook, p2.codebook)
    cbo, iters_o = ob.pq_train(res, M, max_iters=iters, init_codebook=init, nthreads=NT)
    assert np.array_equal(p1.codebook, cbo) and np.array_equal(p1.train_iters.astype(np.int32), iters_o)
