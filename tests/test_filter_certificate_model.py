"""CPU model of the tensor-core FILTER's certificate (DESIGN.md section 5; lance_b200/csrc/tc_assign.cu, tc_common.cuh).

The product decides most rows from a reduced-precision GEMM: score_j = x.c_j - (|c_j|^2 + bias_j)/2 with the column
index packed into the low mantissa byte, top-3 per row, and a row is *unique* when top1 - top2 > tau, *two-candidate*
when top1 - top3 > tau, else *undecided* -- with tau = tau_scale max(|x|^2 + max|c|^2, 2^-90) (tau_of).  The claim
the bit-exactness of the whole build rests on: for a unique row the reference's argmin (exact f32 arithmetic in
reference order, strict `<`, lowest index; lance-linalg/src/kernels.rs:79-111 over l2.rs:57-91) IS top1's column,
for a two-candidate row it is one of top1 / top2.  The GPU tests check that end to end on an H100; this file checks the ARGUMENT on the CPU, against the
oracle, under every rounding behaviour the hardware could have inside the error budget the kernels assume:

  * operands cut to TF32 by truncation or by round-to-nearest-even,
  * accumulation exact-then-rounded, or sequential with every add rounded toward zero (worst case),
  * the 3xTF32 refinement operands  A' = [xh|xh|xl], B' = [ch|cl|ch]  with tau' = (2^-13 + 3d 2^-25)(...),
  * native f16 operands (exact products) with tau16 = (2^-13 + d 2^-23)(...),

on clustered data, integer-valued (SIFT-like) data full of exact ties, rows placed on bisectors of two centroids,
duplicated centroids and a balance bias.  No GPU, no product code: numpy + the oracle only.

The norm floor.  Every error term above is relative to |x|^2 + max|c|^2, which holds while the operands, products and
partial sums are normal f32 numbers.  Below that range roundings are absolute: up to 2^-149 per rounded operation, a
product flushed to zero loses < 2^-126 (a flushed subnormal operand x_i loses < 2^-126 |c_i|: inside the relative
bound while |c| >= 2^-110, inside the floor below), and packing the column index into the low mantissa byte moves a
subnormal score by up to 255 * 2^-149 < 2^-141 -- while tau_scale (|x|^2 + max|c|^2) itself underflows to 0 (then
the filter certifies whichever column packs highest).  So the norm term gets a floor F = 2^-90: tau >= 2^-13 F =
2^-103 for the smallest tau_scale, which covers twice the worst absolute error of one compared score,
d 2^-126 + 2^-141 <= 2^-114 at d <= 4096, with or without flushing.  Rows whose norms sit below the floor simply
become undecided and take the exact path; for every other row tau is unchanged.  The comparison is `s < F ? F : s`,
so a NaN or Inf norm still makes tau NaN / Inf and the row undecided.  test_assignment_routes.py
checks the floor at magnitudes from 2^62 down to 2^-100."""
import numpy as np
import pytest

from oracle import binding as ob

TAU_TF32 = np.float32(3.0 * 2.0 ** -10)          # tc_assign.cu: TAU_TF32
NORM_FLOOR = np.float32(2.0 ** -90)              # tc_common.cuh: NORM_FLOOR (module docstring)


def tau_of(tau_scale, rn2, cmax2):
    """tau = tau_scale * max(|x|^2 + max|c|^2, NORM_FLOOR) in f32, NaN-preserving (tc_common.cuh: cert_tau)"""
    s = (np.asarray(rn2, np.float32) + np.float32(cmax2)).astype(np.float32)
    return (np.float32(tau_scale) * np.where(s < NORM_FLOOR, NORM_FLOOR, s)).astype(np.float32)


def tau3x_scale(d3):                              # tc_assign.cu: tau3x_scale(3d)
    return np.float32(2.0 ** -13 + d3 * 2.0 ** -25)


def tau16_scale(d):                               # tc_assign.cu: tau16_scale(d)
    return np.float32(2.0 ** -13 + d * 2.0 ** -23)


def tf32_trunc(a):
    b = np.ascontiguousarray(a, np.float32).view(np.uint32) & np.uint32(0xFFFFE000)
    return b.view(np.float32)


def tf32_rne(a):                                  # tc_assign.cu: rn_tf32
    b = np.ascontiguousarray(a, np.float32).view(np.uint32).astype(np.uint64)
    b = (b + 0xFFF + ((b >> 13) & 1)) & 0xFFFFE000
    return b.astype(np.uint32).view(np.float32)


def round_toward_zero_f32(v64):
    """f64 -> f32 rounded toward zero (the pessimistic model of the accumulator's adds)"""
    r = v64.astype(np.float32)
    over = np.abs(r.astype(np.float64)) > np.abs(v64)
    r[over] = np.nextafter(r[over], np.float32(0.0))
    return r


def mma_scores(a, b, accumulate):
    """a [n][d], b [K][d] (already in the operand format): the accumulator the epilogue reads, f32 [n][K]"""
    if accumulate == "exact":
        return (a.astype(np.float64) @ b.astype(np.float64).T).astype(np.float32)
    acc = np.zeros((a.shape[0], b.shape[0]), np.float32)
    for e in range(a.shape[1]):                   # sequential, every add rounded toward zero
        prod = a[:, e:e + 1].astype(np.float64) * b[None, :, e].astype(np.float64)   # exact: <= 22 significant bits
        acc = round_toward_zero_f32(acc.astype(np.float64) + prod)
    return acc


def top3_packed(scores):
    """the epilogue's view: low mantissa byte replaced by the column index, then top-3 of the packed values"""
    K = scores.shape[1]
    assert K <= 256
    bits = (np.ascontiguousarray(scores, np.float32).view(np.uint32) & np.uint32(0xFFFFFF00)) | np.arange(K, dtype=np.uint32)[None, :]
    packed = bits.view(np.float32)
    order = np.argsort(-packed, axis=1, kind="stable")[:, :3]
    vals = np.take_along_axis(packed, order, axis=1)
    return vals, order


def certificate(x_op, c_op, cnh, tau, accumulate):
    s = mma_scores(x_op, c_op, accumulate) + cnh[None, :]          # one f32 add per column (tour_chunk)
    vals, idx = top3_packed(s.astype(np.float32))
    flag = np.full(len(x_op), 2)
    flag[(vals[:, 0] - vals[:, 2]) > tau] = 1
    flag[(vals[:, 0] - vals[:, 1]) > tau] = 0
    return flag, idx


def check(flag, idx, ref, min_decided):
    uniq, two = flag == 0, flag == 1
    assert np.array_equal(idx[uniq, 0], ref[uniq]), "a row certified unique has another reference argmin"
    assert np.all((idx[two, 0] == ref[two]) | (idx[two, 1] == ref[two])), "two-candidate row: argmin is neither candidate"
    assert (uniq | two).mean() >= min_decided, f"the model decides only {(uniq | two).mean():.3f} of the rows"


def datasets(d, K, n, rng):
    cent = rng.standard_normal((K, d)).astype(np.float32) * 4
    yield "clustered", cent, cent[rng.integers(0, K, n)] + rng.standard_normal((n, d)).astype(np.float32), 0.5
    ci = np.rint(np.clip(cent * 10 + 60, 0, 255)).astype(np.float32)           # integer-valued: exact ties happen
    xi = np.rint(np.clip(ci[rng.integers(0, K, n)] + rng.integers(-6, 7, (n, d)), 0, 255)).astype(np.float32)
    yield "sift-like integers", ci, xi, 0.3
    a, b = rng.integers(0, K, n), rng.integers(0, K, n)                        # rows on / next to bisectors
    xb = ((cent[a] + cent[b]) * np.float32(0.5) + rng.standard_normal((n, d)).astype(np.float32) * np.float32(1e-3)).astype(np.float32)
    yield "bisectors", cent, xb, 0.0
    cd = cent.copy()
    cd[K // 2:] = cd[:K - K // 2]                                              # every centroid duplicated
    yield "duplicated centroids", cd, cd[rng.integers(0, K, n)] + rng.standard_normal((n, d)).astype(np.float32), 0.0


@pytest.mark.parametrize("cut", ["trunc", "rne"])
@pytest.mark.parametrize("accumulate", ["exact", "toward_zero"])
@pytest.mark.parametrize("d,K", [(64, 96), (8, 256)], ids=["ivf-64x96", "pq-subspace-8x256"])   # tc_filter / tc_pq
def test_tf32_first_pass_certificate(cut, accumulate, d, K):
    rng = np.random.default_rng(11)
    n = 700
    for name, cent, x, min_decided in datasets(d, K, n, rng):
        if d == 8:
            min_decided = 0.0   # 256 codewords in 8 dimensions: many near neighbours, the claim is what is checked
        ref, _, valid = ob.compute_membership(cent, x)
        assert valid.all()
        cutf = tf32_trunc if cut == "trunc" else tf32_rne
        n2 = (cent * cent).sum(1, dtype=np.float32)
        tau = tau_of(TAU_TF32, (x * x).sum(1, dtype=np.float32), n2.max())
        flag, idx = certificate(cutf(x), cutf(cent), np.float32(-0.5) * n2, tau, accumulate)
        check(flag, idx, ref, min_decided)


def test_tf32_first_pass_with_balance_bias():
    rng = np.random.default_rng(12)
    d, K, n = 32, 64, 600
    cent = rng.standard_normal((K, d)).astype(np.float32) * 3
    x = cent[rng.integers(0, K, n)] + rng.standard_normal((n, d)).astype(np.float32)
    sizes = rng.integers(0, 50, K).astype(np.uint64)
    bf = 0.05
    ref, _, _ = ob.compute_membership(cent, x, balance_factor=bf, cluster_sizes=sizes)
    bias = (np.float32(bf) * sizes.astype(np.float32)).astype(np.float32)      # kmeans.rs:234-237
    n2 = (cent * cent).sum(1, dtype=np.float32)
    tau = tau_of(TAU_TF32, (x * x).sum(1, dtype=np.float32), n2.max())
    for accumulate in ("exact", "toward_zero"):
        flag, idx = certificate(tf32_trunc(x), tf32_trunc(cent), np.float32(-0.5) * (n2 + bias), tau, accumulate)
        check(flag, idx, ref, 0.5)


@pytest.mark.parametrize("accumulate", ["exact", "toward_zero"])
def test_3xtf32_refinement_certificate(accumulate):
    rng = np.random.default_rng(13)
    d, K, n = 32, 80, 500
    for name, cent, x, _ in datasets(d, K, n, rng):
        ref, _, _ = ob.compute_membership(cent, x)
        xh, ch = tf32_rne(x), tf32_rne(cent)
        xl, cl = tf32_rne(x - xh), tf32_rne(cent - ch)
        a3 = np.concatenate([xh, xh, xl], 1)                                   # gather_split_kernel
        b3 = np.concatenate([ch, cl, ch], 1)                                   # split_centroids_kernel
        n2 = (cent * cent).sum(1, dtype=np.float32)
        tau = tau_of(tau3x_scale(3 * d), (x * x).sum(1, dtype=np.float32), n2.max())
        flag, idx = certificate(a3, b3, np.float32(-0.5) * n2, tau, accumulate)
        # the refinement is ~20x sharper than the first pass: it must decide nearly everything that has no true tie
        check(flag, idx, ref, 0.9 if name == "clustered" else 0.0)


@pytest.mark.parametrize("accumulate", ["exact", "toward_zero"])
def test_native_f16_operand_certificate(accumulate):
    rng = np.random.default_rng(14)
    d, K, n = 64, 96, 600
    for name, cent, x, _ in datasets(d, K, n, rng):
        c16, x16 = cent.astype(np.float16), x.astype(np.float16)               # f16 columns: T-valued models
        cf, xf = c16.astype(np.float32), x16.astype(np.float32)
        ref, _, _ = ob.compute_membership(cf, xf)                               # l2.rs:100-106: converted exactly, f32 sums
        n2 = (cf * cf).sum(1, dtype=np.float32)
        tau = tau_of(tau16_scale(d), (xf * xf).sum(1, dtype=np.float32), n2.max())
        flag, idx = certificate(xf, cf, np.float32(-0.5) * n2, tau, accumulate)
        check(flag, idx, ref, 0.9 if name == "clustered" else 0.0)


def test_model_would_catch_a_tau_that_is_too_small():
    """the checks above are not vacuous: with tau = 0 the same model certifies rows whose reference argmin differs"""
    rng = np.random.default_rng(15)
    d, K, n = 64, 96, 3000
    cent = rng.standard_normal((K, d)).astype(np.float32) * 4
    a, b = rng.integers(0, K, n), rng.integers(0, K, n)
    x = ((cent[a] + cent[b]) * np.float32(0.5) + rng.standard_normal((n, d)).astype(np.float32) * np.float32(1e-3)).astype(np.float32)
    ref, _, _ = ob.compute_membership(cent, x)
    n2 = (cent * cent).sum(1, dtype=np.float32)
    flag, idx = certificate(tf32_trunc(x), tf32_trunc(cent), np.float32(-0.5) * n2, np.zeros(n, np.float32), "toward_zero")
    assert (flag == 0).all() and (idx[:, 0] != ref).any()


# ---- the FMA pre-screen of pq_fallback_kernel (tc_pq.cu) -------------------------------------------------------
# Undecided (row, sub-space) pairs are finished by a scan of all 256 codewords that first computes
#   s'(c) = fma-chain(r . c) - |c|^2/2   (8 fused steps, cnh from an fma chain too)
# and gives the reference-order distance only to the codewords with s'(c) >= max s' - 2^-18 max(|r|^2 + max|c|^2, 2^-90)
# (the norm floor of the module docstring: below it the roundings of s' and of the reference are absolute).
# Claim: the reference's argmin (sequential 8-term f32 sum, l2.rs:69-79; strict `<`, lowest index) is among them.
def _fma(a, b, c):
    """fused multiply-add in f32: the product of two f32 is exact in f64; one rounding of the f64 sum to f32
    (double rounding could differ from a true fma in the last bit of rare cases -- far inside the budget tested)"""
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(np.float32)


def test_pq_fallback_prescreen_keeps_the_reference_argmin():
    rng = np.random.default_rng(21)
    ds, K = 8, 256
    for scale, near_ties in ((1.0, False), (300.0, False), (1.0, True), (40.0, True)):
        cb = (rng.standard_normal((K, ds)) * scale).astype(np.float32)
        n = 1500
        if near_ties:   # residuals on bisectors of two codewords, and exactly duplicated codewords
            a, b = rng.integers(0, K, n), rng.integers(0, K, n)
            r = ((cb[a] + cb[b]) * np.float32(0.5) + (rng.standard_normal((n, ds)) * scale * 1e-4).astype(np.float32)).astype(np.float32)
            cb[K - 8:] = cb[:8]
        else:
            r = (cb[rng.integers(0, K, n)] + rng.standard_normal((n, ds)).astype(np.float32) * np.float32(scale)).astype(np.float32)
        ref, _, valid = ob.compute_membership(cb, r)
        assert valid.all()
        n2 = np.zeros(K, np.float32)
        for t in range(ds):
            n2 = _fma(cb[:, t], cb[:, t], n2)
        cnh = (np.float32(-0.5) * n2).astype(np.float32)
        rn = np.zeros(n, np.float32)
        for t in range(ds):
            rn = _fma(r[:, t], r[:, t], rn)
        s = np.broadcast_to(cnh[None, :], (n, K)).astype(np.float32)
        for t in range(ds):
            s = _fma(np.broadcast_to(r[:, t:t + 1], (n, K)), np.broadcast_to(cb[None, :, t], (n, K)), s)
        thr = s.max(1) - tau_of(2.0 ** -18, rn, n2.max())
        kept = ~(s < thr[:, None])
        assert kept[np.arange(n), ref].all(), "the pre-screen dropped the reference's argmin"
        assert kept.sum(1).mean() < (64 if near_ties else 8)      # ... and it is selective (that is its point)
