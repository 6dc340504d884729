"""The PQ filter's tournament over COLUMN PAIRS (tc_common.cuh: top3_half<HALF, 2>; tc_pq.cu: decide).

tc_pq_kernel does not rank the 256 codewords of a sub-space one by one: a lane first takes the larger score of the two
neighbouring codewords (c, c ^ 1), packs the PAIR id (c >> 1) into its low mantissa byte, and the top-3 tournament runs
over the 128 pair maxima.  m1 >= m2 >= m3 being the three best, m1 - m2 > tau certifies that the reference's argmin is
one of the two codewords of pair 1, m1 - m3 > tau that it is one of the four of pairs 1 and 2; the kernel then gives
those 2 or 4 codewords the reference-order exact distance (strict `<`, lowest index).  tau, the scores and the size of
the packing error are those of the per-column certificate (tests/test_filter_certificate_model.py).  (Two best pairs
with the same score bits -- duplicated codewords -- are left to pq_fallback_kernel.)

CPU part: the numpy model of that claim on the 8 x 256 sub-space shape, under every rounding the hardware could apply.
GPU part: bit for bit against the oracle and the exact path on inputs made for the pairing: partners that are best and
second best, identical partners, near-ties across two pairs, a NaN / Inf partner."""
import re

import numpy as np
import pytest

import lance_b200 as lb
from oracle import binding as ob
from test_filter_certificate_model import TAU_TF32, datasets, mma_scores, tau_of, tf32_rne, tf32_trunc

NT = 16
DS, KC = 8, 256


# ---- CPU: the pair certificate ---------------------------------------------------------------------------------------
def pair_certificate(x_op, c_op, cnh, tau, accumulate):
    """flag (0 pair 1 certified, 1 pairs 1 and 2, 2 undecided) and the ids of the two best pairs, as the epilogue sees
    them: max of the two raw scores, low mantissa byte replaced by the pair id, top 3 of the packed values"""
    s = (mma_scores(x_op, c_op, accumulate) + cnh[None, :]).astype(np.float32)
    pm = np.maximum(s[:, 0::2], s[:, 1::2])
    bits = (np.ascontiguousarray(pm).view(np.uint32) & np.uint32(0xFFFFFF00)) | np.arange(KC // 2, dtype=np.uint32)[None, :]
    packed = bits.view(np.float32)
    order = np.argsort(-packed, axis=1, kind="stable")[:, :3]
    vals = np.take_along_axis(packed, order, axis=1)
    flag = np.full(len(x_op), 2)
    flag[(vals[:, 0] - vals[:, 2]) > tau] = 1
    flag[(vals[:, 0] - vals[:, 1]) > tau] = 0
    return flag, order


def check_pairs(flag, pairs, ref):
    rp = ref >> 1
    uniq, two = flag == 0, flag == 1
    assert np.array_equal(pairs[uniq, 0], rp[uniq]), "pair 1 certified, the reference's argmin is in another pair"
    assert np.all((pairs[two, 0] == rp[two]) | (pairs[two, 1] == rp[two])), "argmin outside the two certified pairs"
    return (uniq | two).mean()


def _pq_datasets(rng, n):
    yield from datasets(DS, KC, n, rng)
    # partners as near neighbours: every odd codeword a small step from its even partner
    cent = rng.standard_normal((KC, DS)).astype(np.float32) * 4
    cent[1::2] = cent[0::2] + (rng.standard_normal((KC // 2, DS)) * 1e-3).astype(np.float32)
    yield "close partners", cent, cent[rng.integers(0, KC, n)] + rng.standard_normal((n, DS)).astype(np.float32) * np.float32(0.5), 0.5
    cent = cent.copy()
    cent[1::2] = cent[0::2]                                                    # identical partners
    yield "identical partners", cent, cent[rng.integers(0, KC, n)] + rng.standard_normal((n, DS)).astype(np.float32) * np.float32(0.5), 0.5


@pytest.mark.parametrize("cut", ["trunc", "rne"])
@pytest.mark.parametrize("accumulate", ["exact", "toward_zero"])
def test_pair_certificate_keeps_the_reference_argmin(cut, accumulate):
    rng = np.random.default_rng(31)
    n = 700
    cutf = tf32_trunc if cut == "trunc" else tf32_rne
    for name, cent, x, min_decided in _pq_datasets(rng, n):
        ref, _, valid = ob.compute_membership(cent, x)
        assert valid.all()
        n2 = (cent * cent).sum(1, dtype=np.float32)
        tau = tau_of(TAU_TF32, (x * x).sum(1, dtype=np.float32), n2.max())
        flag, pairs = pair_certificate(cutf(x), cutf(cent), np.float32(-0.5) * n2, tau, accumulate)
        decided = check_pairs(flag, pairs, ref)
        if name in ("close partners", "identical partners"):
            # partners never compete inside the filter: such rows are decided although their two best columns tie
            assert decided >= min_decided, f"{name}: the model decides only {decided:.3f} of the rows"


def test_pair_model_would_catch_a_tau_that_is_too_small():
    """not vacuous: with tau = 0 the model certifies pairs that do not hold the reference's argmin"""
    rng = np.random.default_rng(32)
    n = 4000
    cent = rng.standard_normal((KC, DS)).astype(np.float32) * 4
    a, b = rng.integers(0, KC, n), rng.integers(0, KC, n)
    x = ((cent[a] + cent[b]) * np.float32(0.5) + rng.standard_normal((n, DS)).astype(np.float32) * np.float32(1e-4)).astype(np.float32)
    ref, _, _ = ob.compute_membership(cent, x)
    n2 = (cent * cent).sum(1, dtype=np.float32)
    flag, pairs = pair_certificate(tf32_trunc(x), tf32_trunc(cent), np.float32(-0.5) * n2, np.zeros(n, np.float32), "toward_zero")
    assert (flag == 0).all() and (pairs[:, 0] != (ref >> 1)).any()


# ---- GPU: inputs made for the pairing ----------------------------------------------------------------------------------
_PQ = re.compile(r"\[lb2 tc_pq\] n=(\d+) M=(\d+): exact-fallback pairs ([\d.]+)%")


def _nudge(v, steps):
    v = np.float32(v)
    for _ in range(abs(steps)):
        v = np.nextafter(v, np.float32(np.inf if steps > 0 else -np.inf))
    return v


def _paired_codebook(rng, M):
    """[M][256][8] ~ 2 N(0, 1) with, in every sub-space:
    pairs 0..15 (codewords 0..31): the odd partner a tiny step from the even one (best and second best are partners);
    pairs 16..23: identical partners (the lower index must win);
    codewords 67 (odd, pair 33) and 70 (even, pair 35), 73 and 76, 79 and 82: a few ulps apart in one coordinate"""
    cb = (rng.standard_normal((M, KC, DS)) * 2).astype(np.float32)
    cb[:, 1:32:2] = cb[:, 0:32:2] + (rng.standard_normal((M, 16, DS)) * 2e-4).astype(np.float32)
    cb[:, 33:48:2] = cb[:, 32:48:2]
    for m in range(M):
        for k, (a, b) in enumerate(((67, 70), (73, 76), (79, 82))):
            cb[m, b] = cb[m, a]
            cb[m, b, (m + k) % DS] = _nudge(cb[m, a, (m + k) % DS], (-1) ** m * (k + 1))
    return cb


def _paired_rows(rng, cb, n):
    """a row = per sub-space a codeword + noise; the first rows sit on / next to the special codewords"""
    M = cb.shape[0]
    pick = rng.integers(0, KC, (n, M))
    noise = (rng.standard_normal((n, M, DS)) * 0.3).astype(np.float32)
    special = np.concatenate([np.arange(48), [67, 70, 73, 76, 79, 82]])
    k = 0
    for rep, amp in enumerate((0.0, 1e-4, 1e-2, 0.2)):          # on the codeword, within TF32 resolution, nearby
        for c in special:
            pick[k] = c
            noise[k] = (rng.standard_normal((M, DS)) * amp).astype(np.float32)
            k += 1
    for c in range(0, 32, 2):                                    # the exact midpoint of two close partners, +- ulps
        pick[k] = c
        noise[k] = (cb[:, c + 1] - cb[:, c]) * np.float32(0.5)
        noise[k, :, 0] += np.float32(1e-7) * (c - 16)
        k += 1
    assert k < n
    vec = cb[np.arange(M)[None, :], pick] + noise
    return vec.reshape(n, M * DS).astype(np.float32)


def _traced(fn, capfd, monkeypatch):
    monkeypatch.delenv("LB2_DISABLE_TC", raising=False)
    monkeypatch.setenv("LB2_TC_STATS", "1")
    capfd.readouterr()
    lb.profile.enable(True)
    lb.profile.reset()
    try:
        out = fn()
    finally:
        lb.profile.enable(False)
    prof = lb.profile.dump()
    calls = [(int(m[1]), int(m[2]), float(m[3])) for m in _PQ.finditer(capfd.readouterr().err)]
    launches = sum(c for name, (c, _) in prof.items() if name.endswith("tc_pq_filter"))
    pairs = sum(n * M for n, M, _ in calls)
    share = sum(p * n * M / 100 for n, M, p in calls) / pairs if pairs else None
    return out, launches, share


def _exact_path(fn, monkeypatch):
    monkeypatch.setenv("LB2_DISABLE_TC", "1")
    try:
        return fn()
    finally:
        monkeypatch.delenv("LB2_DISABLE_TC", raising=False)


@pytest.mark.gpu
@pytest.mark.parametrize("M", [16, 48], ids=["resident-codebook", "streamed-codebook"])
@pytest.mark.parametrize("n", [4099, 448], ids=["rows-4099", "rows-448"])
def test_encode_partner_codewords(n, M, capfd, monkeypatch):
    rng = np.random.default_rng(9000 + M + n)
    cb = _paired_codebook(rng, M)
    vec = _paired_rows(rng, cb, n)
    pq = lb.ProductQuantizer(M, 8, M * DS, cb)
    got, launches, share = _traced(lambda: pq.quantize(vec), capfd, monkeypatch)
    want = ob.pq_encode(cb, vec, nthreads=NT)
    assert np.array_equal(got, want)
    assert np.array_equal(got, _exact_path(lambda: pq.quantize(vec), monkeypatch))
    assert launches == 1
    # the inputs do what they were made for: partners win and lose against each other, identical partners resolve to
    # the even one, and both codewords of an ulp-apart cross pair are chosen somewhere
    close = want[(want < 32)]
    assert (close % 2 == 0).any() and (close % 2 == 1).any()
    dup = want[(want >= 32) & (want < 48)]
    assert dup.size and (dup % 2 == 0).all()
    assert {67, 70} <= set(np.unique(want).tolist())
    # the filter, not pq_fallback_kernel, decided nearly all pairs (close and identical partners included)
    assert share is not None and share < 0.10, share


@pytest.mark.gpu
@pytest.mark.parametrize("M", [16, 48], ids=["resident-codebook", "streamed-codebook"])
@pytest.mark.parametrize("bad", ["nan", "inf"])
def test_encode_non_finite_partner(bad, M, capfd, monkeypatch):
    n = 3001
    rng = np.random.default_rng(9100 + M)
    cb = _paired_codebook(rng, M)
    vec = _paired_rows(rng, cb, n)                               # rows made before the codebook is damaged: they still
    if bad == "nan":                                             # sit next to the finite partner
        cb[:, 5, 3] = np.nan                                     # odd partner of a close pair, every sub-space
        cb[:, 40, 0] = np.nan                                    # even partner of an identical pair
    else:
        cb[0, 5, 3] = np.inf                                     # |c|^2 = inf: tau = inf, sub-space 0 is all fallback
        cb[0, 40, 0] = -np.inf
    pq = lb.ProductQuantizer(M, 8, M * DS, cb)
    got, launches, share = _traced(lambda: pq.quantize(vec), capfd, monkeypatch)
    assert np.array_equal(got, ob.pq_encode(cb, vec, nthreads=NT))
    assert np.array_equal(got, _exact_path(lambda: pq.quantize(vec), monkeypatch))
    assert launches == 1
    hit = got if bad == "nan" else got[:, :1]
    assert (hit == 4).any() and (hit == 41).any()                # the finite partner of a damaged pair is chosen
    assert share is not None and share < (0.10 if bad == "nan" else 1.0 / M + 0.10), share


@pytest.mark.gpu
@pytest.mark.parametrize("M", [16, 48], ids=["resident-codebook", "streamed-codebook"])
def test_training_from_a_paired_codebook(M, capfd, monkeypatch):
    """PQ training (ids and exact distances from the filter's epilogue) started from the paired codebook: the first
    iterations assign against close and identical partners, then the partners drift apart"""
    n, iters = 5003, 6
    rng = np.random.default_rng(9200 + M)
    init = _paired_codebook(rng, M)
    data = _paired_rows(rng, init, n)
    build = lambda: lb.PQBuildParams(M, 8, max_iters=iters, codebook=init).build(data)
    pq, launches, share = _traced(build, capfd, monkeypatch)
    cbo, iters_o = ob.pq_train(data, M, max_iters=iters, init_codebook=init, nthreads=NT)
    assert np.array_equal(pq.train_iters.astype(np.int32), iters_o)
    assert np.array_equal(pq.codebook.view(np.uint32), cbo.view(np.uint32))
    ex = _exact_path(build, monkeypatch)
    assert np.array_equal(pq.codebook.view(np.uint32), ex.codebook.view(np.uint32))
    assert launches >= 1
    assert share is not None and share < 0.10, share
