"""The PQ filter's decision pass: the top 3 of every (row, sub-space) are parked in shared memory, and once an item's
tournaments are done one converged pass per warp (all 32 lanes) decides its 16 rows x 4 sub-spaces.  Cases put the
four sub-spaces of a row, and the rows of one 16-row warp slice, on different flags (a codeword: flag 0; the midpoint
of two codewords: flag 1; a duplicated codeword or a NaN sub-vector: undecided), end the row count inside an item and
inside a warp slice, give CTAs one item or many, and run PQ training with sub-spaces that converge early (inactive
sub-spaces inside an item).  Codes and codebooks must equal the exact path and the CPU oracle.  The CPU test checks
that the shared-memory layout of both variants fits the 227 KB of one block."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import lance_b200 as lb
from oracle import binding as ob

NT = 16
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _both_paths(fn):
    os.environ.pop("LB2_DISABLE_TC", None)
    a = fn()
    os.environ["LB2_DISABLE_TC"] = "1"
    try:
        b = fn()
    finally:
        os.environ.pop("LB2_DISABLE_TC", None)
    return a, b


def _mixed_flags(n, M, seed):
    """codebook and rows whose (row, sub-space) kind is (row + 3 m) % 4: every 16-row slice of every sub-space and
    the four sub-spaces of every row hold all four kinds"""
    rng = np.random.default_rng(seed)
    cb = (rng.standard_normal((M, 256, 8)) * 2).astype(np.float32)
    cb[:, 200] = cb[:, 77]  # a duplicated codeword (pairs 38 and 100): equal score bits keep rows undecided
    vec = np.empty((n, M * 8), np.float32)
    for m in range(M):
        kind = (np.arange(n) + 3 * m) % 4
        a = rng.integers(0, 256, n)
        b = (a + 2 + 2 * rng.integers(0, 100, n)) % 256  # another pair than a's
        sub = cb[m, a].copy()                                                   # 0: a codeword
        sub[kind == 1] = ((cb[m, a] + cb[m, b]) / np.float32(2))[kind == 1]     # 1: two codewords tie
        sub[kind == 2] = cb[m, 77] + np.float32(1e-3) * rng.standard_normal((n, 8)).astype(np.float32)[kind == 2]
        sub[kind == 3] = np.nan                                                 # 3: no finite score
        vec[:, m * 8:(m + 1) * 8] = sub
    return cb, vec


def _fallback_share(capfd, fn):
    os.environ["LB2_TC_STATS"] = "1"
    try:
        capfd.readouterr()
        fn()
        err = capfd.readouterr().err
    finally:
        os.environ.pop("LB2_TC_STATS", None)
    return [float(v) for v in re.findall(r"exact-fallback pairs ([\d.]+)%", err)]


# n: one item per CTA at most (300 rows: 20 items), rows ending inside a warp slice (1000 = 15 x 64 + 40), many items
# per CTA; M = 16 keeps the codebook resident, M = 48 streams it
@pytest.mark.gpu
@pytest.mark.parametrize("n,M", [(300, 16), (1000, 16), (70001, 16), (1000, 48), (20007, 48)])
def test_decision_pass_encode_mixed_flags(n, M, capfd):
    cb, vec = _mixed_flags(n, M, seed=n + M)
    pq = lb.ProductQuantizer(M, 8, M * 8, cb)
    share = _fallback_share(capfd, lambda: pq.quantize(vec))
    # about half the pairs (the duplicated and NaN kinds) are undecided, the others are decided in the pass
    assert share and all(40.0 < s < 75.0 for s in share), share
    c1, c2 = _both_paths(lambda: pq.quantize(vec))
    assert np.array_equal(c1, c2)
    assert np.array_equal(c1, ob.pq_encode(cb, vec, nthreads=NT))


def _converging(n, M, seed):
    """residuals whose sub-spaces 0-3 and 5 are exact copies of the initial codewords (they converge first), with a
    duplicated initial codeword and midpoint rows in the other sub-spaces"""
    rng = np.random.default_rng(seed)
    d = M * 8
    res = (rng.standard_normal((n, d)) * np.linspace(0.5, 4.0, d)).astype(np.float32)
    init = np.stack([res[rng.choice(n, 256, replace=False)][:, m * 8:(m + 1) * 8] for m in range(M)])
    for m in range(M):
        if m in (0, 1, 2, 3, 5):
            pick = np.concatenate([np.arange(256), rng.integers(0, 256, n - 256)])
            res[:, m * 8:(m + 1) * 8] = init[m][pick]
        else:
            init[m, 201] = init[m, 14]
            mid = (np.arange(n) % 16) < 5  # five rows of every warp slice on a midpoint
            a, b = rng.integers(0, 128, n) * 2, rng.integers(0, 128, n) * 2 + 1
            res[mid, m * 8:(m + 1) * 8] = ((init[m][a] + init[m][b]) / np.float32(2))[mid]
    return res, init


@pytest.mark.gpu
@pytest.mark.parametrize("n,M", [(1000, 16), (9040, 16), (3001, 48)])
def test_decision_pass_training_with_inactive_sub_spaces(n, M):
    iters = 10
    res, init = _converging(n, M, seed=n + M)
    p1, p2 = _both_paths(lambda: lb.PQBuildParams(M, 8, max_iters=iters, codebook=init).build(res))
    assert p1.train_iters[:4].max() < p1.train_iters.max(), "the first chunk must converge before the others"
    assert np.array_equal(p1.train_iters, p2.train_iters) and np.array_equal(p1.codebook, p2.codebook)
    cbo, iters_o = ob.pq_train(res, M, max_iters=iters, init_codebook=init, nthreads=NT)
    assert np.array_equal(p1.codebook, cbo) and np.array_equal(p1.train_iters.astype(np.int32), iters_o)


def test_shared_memory_layout_fits_one_block():
    """tc_pq.cu asserts at compile time that the resident (M = 16) and streamed (M = 256) layouts, parking slots and
    alignment slack included, fit 227 KB; the front end alone evaluates those assertions"""
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc is not installed")
    src = os.path.join(ROOT, "lance_b200", "csrc", "tc_pq.cu")
    text = open(src).read()
    assert "layout(MAX_M_RESIDENT / 4, MAX_M_RESIDENT, false).total + 1024 <= SMEM_OPTIN" in text
    assert "layout(MAX_M / 4, MAX_M, true).total + 1024 <= SMEM_OPTIN" in text
    assert re.search(r"SMEM_OPTIN = 227 \* 1024", text)
    out = subprocess.run([nvcc, "-std=c++17", "--expt-relaxed-constexpr", "-gencode", "arch=compute_90a,code=sm_90a",
                          "--cuda", src, "-o", os.devnull], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr[-2000:]
