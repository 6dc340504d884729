"""Every route of centroid and PQ-code assignment against the oracle, down to subnormal magnitudes.

A partition id or a PQ code goes through one decision chain: a tensor-core filter (tc_filter_kernel,
tc_filter_general_kernel<OPK, MODE>, tc_pq_kernel) certifies a row as unique / two-candidate with a bound tau, and
the rest is settled by exact passes (rerank_kernel, the 3xTF32 pass, the candidate pass and cand_exact_kernel,
forward_overflow_kernel, the regimes of assign_rows_f32, pq_fallback_kernel).  Each GPU case below compares the
product with the oracle bit for bit (ids, distances, valid; PQ codes) and, where both exist, with LB2_DISABLE_TC=1,
and proves that the route it names carried rows: launch names from lb.profile, row counts from LB2_TC_STATS.

Undecided rows are built on purpose: a row placed exactly on a centroid that appears four times has top1 = top2 =
top3 up to the packed column index, so no tau certifies it.

The CPU test at the end extends the certificate model (test_filter_certificate_model.py) to the magnitudes of the
GPU cases, with an MMA model that flushes subnormal operands and products to zero, and shows that the norm floor of
tau is what keeps certified rows right below ~2^-60."""
import ctypes as C
import re

import numpy as np
import pytest

import lance_b200 as lb
from oracle import binding as ob
from test_filter_certificate_model import (NORM_FLOOR, TAU_TF32, _fma, mma_scores, tau3x_scale, tau_of, tf32_rne,
                                           tf32_trunc, top3_packed)

NT = 16
SCALES = (62, 60, 0, -60, -66, -70, -76, -80, -100)     # data and model scaled by 2^e (exact: powers of two)
ENV_KEYS = ("LB2_DISABLE_TC", "LB2_FORCE_REFINE", "LB2_NO_NATIVE16", "LB2_TC_STATS")

_FIRST = re.compile(r"\[lb2 (\S+)\] n=(\d+) K=(\d+) d=(\d+): unique ([\d.]+)%, two-candidate ([\d.]+)%, "
                    r"undecided ([\d.]+)%")
_REFINE = re.compile(r"\[lb2 (\S+)\] undecided after pass 1: (\d+), after the top-3 refinement: (\d+), "
                     r"full-K exact scan: (\d+)")
_PQ = re.compile(r"\[lb2 tc_pq\] n=(\d+) M=(\d+): exact-fallback pairs ([\d.]+)%")


class Trace:
    """What one call did: kernel families launched (lb.profile) and the LB2_TC_STATS counts it printed."""

    def __init__(self, prof, err):
        self.prof = prof
        self.first = [(m[1], int(m[2]), float(m[7])) for m in _FIRST.finditer(err)]
        self.refine = [tuple(int(v) for v in m.groups()[1:]) for m in _REFINE.finditer(err)]
        self.pq = [(int(m[1]), int(m[2]), float(m[3])) for m in _PQ.finditer(err)]

    def launched(self, name):
        return self.prof.get(name, (0, 0.0))[0]

    def filters(self):
        return {f for f, _, _ in self.first}

    def undecided(self):
        """rows the first pass left undecided (printed as a percentage with two decimals: +-0.005 % of n)"""
        return sum(round(p * n / 100) for _, n, p in self.first)

    def refined(self):
        """(undecided after pass 1, after the 3xTF32 top-3 pass, sent to the full-K exact scan), summed over calls"""
        return tuple(sum(r[i] for r in self.refine) for i in range(3)) if self.refine else None

    def pq_pairs(self):
        return sum(p * n * M / 100 for n, M, p in self.pq)


def _traced(fn, capfd, monkeypatch, **env):
    for k in ENV_KEYS:
        monkeypatch.delenv(k, raising=False)
    monkeypatch.setenv("LB2_TC_STATS", "1")
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    capfd.readouterr()
    lb.profile.enable(True)
    lb.profile.reset()
    try:
        out = fn()
    finally:
        lb.profile.enable(False)
    return out, Trace(lb.profile.dump(), capfd.readouterr().err)


def _same(a, b):
    """ids, distances (bit patterns) and valid flags are identical"""
    return (np.array_equal(a[0], b[0]) and np.array_equal(np.asarray(a[1], np.float32).view(np.uint32),
                                                         np.asarray(b[1], np.float32).view(np.uint32))
            and np.array_equal(a[2], b[2]))


def _oracle(cent32, data32, metric="l2"):
    return ob.compute_membership(cent32, data32, metric=metric, nthreads=NT)


def _exact_path(fn, monkeypatch):
    monkeypatch.setenv("LB2_DISABLE_TC", "1")
    try:
        return fn()
    finally:
        monkeypatch.delenv("LB2_DISABLE_TC")


def _refines(n, d, K, force):
    """tc_refine_and_fallback's choice (H100: the refinement's shared memory always fits)"""
    return bool(force) or n * K >= 1 << 26 or n * K * d >= 1 << 32


# ---- data ----------------------------------------------------------------------------------------------------------
def _to_bf16(a):
    return (np.ascontiguousarray(a, np.float32).view(np.uint32) >> 16).astype(np.uint16)


def _from_bf16(t):
    return (t.astype(np.uint32) << 16).view(np.float32)


def _clustered(rng, n, d, K, n_tied=64, dup=(10, 4), noise=0.3, n_nonfinite=2, scale=1.0):
    """K Gaussian centroids, rows = a centroid + noise.  Centroids dup[0] .. dup[0] + dup[1] - 1 are identical and
    the first n_tied rows lie exactly on them (undecided for every filter); the next n_nonfinite rows hold a NaN or an
    Inf.  Everything is scaled by the power of two `scale` at the end, which keeps every value exact."""
    cent = rng.standard_normal((K, d)).astype(np.float32)
    if K >= dup[0] + dup[1]:
        cent[dup[0]:dup[0] + dup[1]] = cent[dup[0]]
    data = (cent[rng.integers(0, K, n)] + (rng.standard_normal((n, d)) * noise).astype(np.float32)).astype(np.float32)
    if K >= dup[0] + dup[1]:
        data[:n_tied] = cent[dup[0]]
    s = np.float32(scale)
    cent, data = (cent * s).astype(np.float32), (data * s).astype(np.float32)
    for i in range(n_nonfinite):
        data[n_tied + i, i % d] = np.nan if i % 2 == 0 else np.inf
    return cent, data


# ---- 1. the first pass: every kernel and operand kind, refinement off and forced ------------------------------------
def _check_first_pass(cent, data, cent32, data32, capfd, monkeypatch, force, filt, bf16=False):
    n, d = data.shape
    K = cent.shape[0]
    run = lambda: lb.compute_partitions(cent, data, bf16=bf16)
    got, tr = _traced(run, capfd, monkeypatch, **({"LB2_FORCE_REFINE": "1"} if force else {}))
    ref = _oracle(cent32, data32)
    assert _same(got, ref) and _same(got, _exact_path(run, monkeypatch))
    assert tr.filters() == {filt} and tr.launched(filt) >= 1
    assert tr.undecided() >= 2                       # at least the non-finite rows
    if _refines(n, d, K, force):
        a, b, c = tr.refined()
        assert a >= 2 and c >= 2                     # NaN / Inf rows: no candidate -> full-K exact scan
        assert tr.launched("tc_candidates") >= 1 and tr.launched("tc_candidates_exact") >= 1
        if K >= 14:
            assert a >= 64 + 2                       # the rows on the 4-fold centroid ...
            if filt != "tc_filter_general16":
                assert b >= 64 + 2 and tr.launched("tc_refine_filter") == 1   # ... tie in the 3xTF32 pass too
    else:
        assert tr.refined() is None and tr.launched("tc_refine_filter") == 0
        assert tr.launched("assign_exact_fallback") >= 1
    return tr


@pytest.mark.gpu
@pytest.mark.parametrize("force", ["", "1"], ids=["auto", "forced-refine"])
@pytest.mark.parametrize("K", [2, 255, 256])
@pytest.mark.parametrize("d", [32, 64, 128])
def test_resident_tf32_first_pass(d, K, force, capfd, monkeypatch):
    rng = np.random.default_rng(1000 + d + K)
    cent, data = _clustered(rng, 3000, d, K)
    _check_first_pass(cent, data, cent, data, capfd, monkeypatch, force, "tc_filter")


@pytest.mark.gpu
@pytest.mark.parametrize("force", ["", "1"], ids=["auto", "forced-refine"])
@pytest.mark.parametrize("K", [257, 1000, 4096])
@pytest.mark.parametrize("d", [160, 768, 1536])
def test_general_tf32_first_pass(d, K, force, capfd, monkeypatch):
    rng = np.random.default_rng(2000 + d + K)
    cent, data = _clustered(rng, 2000, d, K)
    _check_first_pass(cent, data, cent, data, capfd, monkeypatch, force, "tc_filter_general")


def _native(rng, n, d, K, dtype, scale=1.0):
    """16-bit rows and a model of the same type (models trained on such columns are exactly representable)"""
    cent, data = _clustered(rng, n, d, K, scale=scale)
    if dtype == "f16":
        ct, xt = cent.astype(np.float16), data.astype(np.float16)
        return ct, xt, ct.astype(np.float32), xt.astype(np.float32)
    ct, xt = _to_bf16(cent), _to_bf16(data)
    return ct, xt, _from_bf16(ct), _from_bf16(xt)


@pytest.mark.gpu
@pytest.mark.parametrize("force", ["", "1"], ids=["auto", "forced-refine"])
@pytest.mark.parametrize("d,K", [(192, 300), (128, 1000), (1536, 257)])
@pytest.mark.parametrize("dtype", ["f16", "bf16"])
def test_native_16bit_first_pass(dtype, d, K, force, capfd, monkeypatch):
    # a resident shape (d <= 128, K <= 256) never reads native rows: general shapes only
    ct, xt, c32, x32 = _native(np.random.default_rng(3000 + d + K), 2000, d, K, dtype)
    _check_first_pass(ct, xt, c32, x32, capfd, monkeypatch, force, "tc_filter_general16", bf16=dtype == "bf16")


# ---- 2. fall-backs to other routes -----------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dtype", ["f16", "bf16"])
@pytest.mark.parametrize("case", ["d96", "no-native16"])
def test_native_rows_fall_back_to_tf32(dtype, case, capfd, monkeypatch):
    # d % 64 != 0, or LB2_NO_NATIVE16: the filter reads the f32 view of the 16-bit rows
    d, K = (96, 300) if case == "d96" else (192, 300)
    ct, xt, c32, x32 = _native(np.random.default_rng(3100 + d), 2000, d, K, dtype)
    run = lambda: lb.compute_partitions(ct, xt, bf16=dtype == "bf16")
    env = {"LB2_NO_NATIVE16": "1"} if case == "no-native16" else {}
    got, tr = _traced(run, capfd, monkeypatch, **env)
    assert _same(got, _oracle(c32, x32))
    assert tr.filters() == {"tc_filter_general"} and tr.launched("tc_filter_general16") == 0
    assert tr.undecided() >= 64 + 2 and tr.launched("assign_exact_fallback") >= 1


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 255])
@pytest.mark.parametrize("d,metric", [(8, "l2"), (20, "l2"), (40, "l2"), (128, "l2"), (40, "dot"), (288, "dot"),
                                      (128, "dot")])
def test_exact_only_shapes(d, metric, n, capfd, monkeypatch):
    # d % 32 != 0, d < 32, n < 256 and DOT never take a tensor-core filter
    rng = np.random.default_rng(4000 + d + n)
    K = 300
    cent, data = _clustered(rng, n, d, K, n_tied=min(n, 8), n_nonfinite=0)
    got, tr = _traced(lambda: lb.compute_partitions(cent, data, metric), capfd, monkeypatch)
    assert _same(got, _oracle(cent, data, metric))
    assert not any(k.startswith("tc_") for k in tr.prof) and not tr.first
    exact = "assign_exact" if d % 16 == 0 and d <= 256 else "assign_exact_generic"
    assert tr.launched(exact) == 1
    if n == 255 and metric == "dot":     # DOT also where the shape alone would allow the filter
        big = np.concatenate([data, data])
        got, tr = _traced(lambda: lb.compute_partitions(cent, big, metric), capfd, monkeypatch)
        assert _same(got, _oracle(cent, big, metric)) and not any(k.startswith("tc_") for k in tr.prof)


def _partitions_from_device(cent, raw, n, d, dt, offset_bytes):
    """lb2_compute_partitions straight on a device pointer `offset_bytes` past the start of a DeviceArray"""
    from lance_b200 import _lib
    buf = lb.DeviceArray.from_numpy(raw)
    part, dist, valid = np.empty(n, np.uint32), np.empty(n, np.float32), np.empty(n, np.uint8)
    cent = np.ascontiguousarray(cent)
    _lib.check(_lib.lib().lb2_compute_partitions(
        C.c_void_p(cent.ctypes.data), C.c_uint32(cent.shape[0]), C.c_uint32(d), C.c_int(dt), C.c_int(_lib.L2),
        C.c_void_p(buf.ptr + offset_bytes), C.c_uint64(n), C.c_void_p(part.ctypes.data), C.c_void_p(dist.ctypes.data),
        C.c_void_p(valid.ctypes.data)))
    buf.free()
    return part, dist, valid.astype(bool)


@pytest.mark.gpu
def test_unaligned_f32_rows_take_the_exact_kernel(capfd, monkeypatch):
    # a row base that is not 16-byte aligned: no TMA, no float4 loads -- the scalar-load generic kernel
    from lance_b200 import _lib
    rng = np.random.default_rng(4100)
    n, d, K = 3000, 128, 256
    cent, data = _clustered(rng, n, d, K)
    raw = np.concatenate([np.zeros(1, np.float32), data.ravel()])
    got, tr = _traced(lambda: _partitions_from_device(cent, raw, n, d, _lib.F32, 4), capfd, monkeypatch)
    assert _same(got, _oracle(cent, data))
    assert not any(k.startswith("tc_") for k in tr.prof) and tr.launched("assign_exact_generic") == 1
    aligned, tr = _traced(lambda: _partitions_from_device(cent, raw[1:].copy(), n, d, _lib.F32, 0), capfd, monkeypatch)
    assert _same(aligned, got) and tr.launched("tc_filter") == 1


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", ["f16", "bf16"])
def test_unaligned_16bit_rows_take_the_tf32_filter(dtype, capfd, monkeypatch):
    # native rows 4 bytes off a 16-byte boundary: the filter reads the (aligned) f32 copy instead
    from lance_b200 import _lib
    n, d, K = 2000, 192, 300
    ct, xt, c32, x32 = _native(np.random.default_rng(4200), n, d, K, dtype)
    raw = np.concatenate([np.zeros(2, np.uint16), xt.view(np.uint16).ravel()])
    dt = _lib.F16 if dtype == "f16" else _lib.BF16
    got, tr = _traced(lambda: _partitions_from_device(ct.view(np.uint16), raw, n, d, dt, 4), capfd, monkeypatch)
    assert _same(got, _oracle(c32, x32))
    assert tr.filters() == {"tc_filter_general"} and tr.undecided() >= 64 + 2
    aligned, tr = _traced(lambda: _partitions_from_device(ct.view(np.uint16), raw[2:].copy(), n, d, dt, 0), capfd,
                          monkeypatch)
    assert _same(aligned, got) and tr.filters() == {"tc_filter_general16"}


# ---- 3. the regimes of assign_rows_f32 (refinement off) ---------------------------------------------------------------
def _num_sms():
    import torch  # device properties only
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.gpu
@pytest.mark.parametrize("n_tied", [1000, 5000, 36000], ids=["split-merge", "16-row", "64-row"])
def test_exact_fallback_tile_regimes(n_tied, capfd, monkeypatch):
    # d <= 256, d % 16 == 0: lists < 2048 rows are split over the 64-centroid chunks and merged; longer ones take
    # 16-row tiles; lists of at least 64 * 2 * SMs rows 64-row tiles (only launched for K > 256)
    n, d, K = 40000, 128, 300
    assert not _refines(n, d, K, "")
    cent, data = _clustered(np.random.default_rng(5000 + n_tied), n, d, K, n_tied=n_tied)
    run = lambda: lb.compute_partitions(cent, data)
    got, tr = _traced(run, capfd, monkeypatch)
    assert _same(got, _oracle(cent, data)) and _same(got, _exact_path(run, monkeypatch))
    u, split = tr.undecided(), 64 * 2 * _num_sms()
    assert tr.filters() == {"tc_filter_general"} and tr.launched("assign_exact_fallback") == 4
    lo, hi = {1000: (n_tied, 2048), 5000: (2048, split), 36000: (split, n + 1)}[n_tied]
    assert lo <= u < hi, (u, lo, hi)


@pytest.mark.gpu
@pytest.mark.parametrize("n,K,n_tied", [(20000, 300, 1000), (10000, 1024, 1000), (20000, 300, 6000)],
                         ids=["split-2", "split-8", "unsplit"])
def test_exact_fallback_generic_regimes(n, K, n_tied, capfd, monkeypatch):
    # d > 256: the generic kernel; lists < 4096 rows against K >= 256 are split over min(64, K / 128) centroid ranges
    d = 288
    assert not _refines(n, d, K, "")
    cent, data = _clustered(np.random.default_rng(5100 + n + K + n_tied), n, d, K, n_tied=n_tied)
    run = lambda: lb.compute_partitions(cent, data)
    got, tr = _traced(run, capfd, monkeypatch)
    assert _same(got, _oracle(cent, data)) and _same(got, _exact_path(run, monkeypatch))
    u = tr.undecided()
    assert tr.filters() == {"tc_filter_general"} and tr.launched("assign_exact_fallback") == 3
    assert (n_tied <= u < 4096) if n_tied < 4096 else (u >= 4096), u


# ---- 4. more undecided rows than the refinement's gather capacity -----------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("dtype,d,K", [("f32", 128, 256), ("f32", 128, 512), ("f16", 128, 512), ("bf16", 128, 512)])
def test_refinement_capacity_overflow(dtype, d, K, capfd, monkeypatch):
    # cap = min(n, max(4096, n / 8)) = 5000 gathered rows; the rest is forwarded to the full-K exact scan (f32:
    # rerank_kernel's list mode; 16-bit: forward_overflow_kernel).  5000 rows on a 4-fold centroid (4 candidates) and
    # 4000 on a 20-fold one (more candidates than slots: the full-K scan in any case).
    n, cap = 40000, 5000
    rng = np.random.default_rng(6000 + K + len(dtype))
    cent = rng.standard_normal((K, d)).astype(np.float32)
    cent[10:14] = cent[10]
    cent[100:120] = cent[100]
    data = (cent[rng.integers(0, K, n)] + (rng.standard_normal((n, d)) * 0.3).astype(np.float32)).astype(np.float32)
    data[:5000] = cent[10]
    data[5000:9000] = cent[100]
    data[9000, 3] = np.nan
    if dtype == "f32":
        ct, xt, c32, x32 = cent, data, cent, data
    elif dtype == "f16":
        ct, xt = cent.astype(np.float16), data.astype(np.float16)
        c32, x32 = ct.astype(np.float32), xt.astype(np.float32)
    else:
        ct, xt = _to_bf16(cent), _to_bf16(data)
        c32, x32 = _from_bf16(ct), _from_bf16(xt)
    run = lambda: lb.compute_partitions(ct, xt, bf16=dtype == "bf16")
    got, tr = _traced(run, capfd, monkeypatch, LB2_FORCE_REFINE="1")
    assert _same(got, _oracle(c32, x32))
    if dtype == "f32":
        assert _same(got, _exact_path(run, monkeypatch))
    a, b, c = tr.refined()
    assert a >= 9001 and c >= max(a - cap, 4001), (a, b, c)   # the overflow, the 20-fold rows and the NaN row
    assert tr.filters() == {"tc_filter" if K <= 256 else "tc_filter_general16" if dtype != "f32" else "tc_filter_general"}
    assert tr.launched("assign_exact_fallback") >= 1 and tr.launched("tc_candidates_exact") >= 1


# ---- 5. magnitude edges -----------------------------------------------------------------------------------------------
_ROUTES = {  # name: (d, K, LB2_FORCE_REFINE, filter)
    "resident": (128, 256, "", "tc_filter"),
    "resident-refine": (128, 256, "1", "tc_filter"),
    "general": (160, 300, "", "tc_filter_general"),
    "general-refine": (160, 300, "1", "tc_filter_general"),
}


@pytest.mark.gpu
@pytest.mark.parametrize("route", list(_ROUTES))
@pytest.mark.parametrize("e", SCALES)
def test_f32_routes_at_every_magnitude(e, route, capfd, monkeypatch):
    # rows a centroid + 0.3x noise at scale 2^e.  Below ~2^-60 |x|^2 and the distances leave the normal range (the
    # reference's distances to nearby centroids underflow to 0 from ~2^-76 on: its first minimum wins); at 2^62
    # |x|^2 overflows while the distance to the row's own centroid stays finite.
    d, K, force, filt = _ROUTES[route]
    cent, data = _clustered(np.random.default_rng(7000 + d), 2000, d, K, scale=2.0 ** e)
    _check_first_pass(cent, data, cent, data, capfd, monkeypatch, force, filt)


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["tiny-rows", "tiny-centroids"])
@pytest.mark.parametrize("e", [-66, -76, -100])
@pytest.mark.parametrize("route", ["resident", "general-refine"])
def test_f32_tiny_rows_against_unit_centroids_and_reverse(route, e, which, capfd, monkeypatch):
    d, K, force, filt = _ROUTES[route]
    rng = np.random.default_rng(7100 + d - e)
    cent = rng.standard_normal((K, d)).astype(np.float32)
    small = (rng.standard_normal((2000, d)) * np.float32(2.0 ** e)).astype(np.float32)
    if which == "tiny-rows":
        data = small
        data[:64] = np.float32(0.0)                  # exactly at the origin
    else:
        data, cent = (cent[rng.integers(0, K, 2000)] * np.float32(2.0 ** e)).astype(np.float32), small[:K].copy()
        cent[10:14] = cent[10]
        data[:64] = cent[10]
    data[100, 0] = np.nan
    data[101, 1] = np.inf
    run = lambda: lb.compute_partitions(cent, data)
    got, tr = _traced(run, capfd, monkeypatch, **({"LB2_FORCE_REFINE": "1"} if force else {}))
    assert _same(got, _oracle(cent, data)) and _same(got, _exact_path(run, monkeypatch))
    assert tr.filters() == {filt} and tr.undecided() >= 2


@pytest.mark.gpu
@pytest.mark.parametrize("force", ["", "1"], ids=["auto", "forced-refine"])
@pytest.mark.parametrize("e", SCALES)
def test_bf16_native_rows_at_every_magnitude(e, force, capfd, monkeypatch):
    ct, xt, c32, x32 = _native(np.random.default_rng(7200), 2000, 192, 300, "bf16", scale=2.0 ** e)
    _check_first_pass(ct, xt, c32, x32, capfd, monkeypatch, force, "tc_filter_general16", bf16=True)


@pytest.mark.gpu
@pytest.mark.parametrize("force", ["", "1"], ids=["auto", "forced-refine"])
@pytest.mark.parametrize("e", [-14, -18, -20, -22])
def test_f16_native_rows_in_the_subnormal_range(e, force, capfd, monkeypatch):
    # f16 subnormals start below 2^-14; at 2^-22 most elements keep 1..3 significant bits
    ct, xt, c32, x32 = _native(np.random.default_rng(7300), 2000, 192, 300, "f16", scale=2.0 ** e)
    assert (np.abs(xt[np.isfinite(xt)]) < np.float16(2.0 ** -14)).mean() > 0.5
    _check_first_pass(ct, xt, c32, x32, capfd, monkeypatch, force, "tc_filter_general16")


def _pq_data(rng, n, M, scale):
    """codebook [M][256][8] ~ N(0, 1), rows = a codeword per sub-space + 0.3x noise; codewords 100..103 identical in
    every sub-space and rows 0..63 exactly on them (undecided pairs for pq_fallback_kernel); scaled by `scale`"""
    cb = rng.standard_normal((M, 256, 8)).astype(np.float32)
    cb[:, 101:104] = cb[:, 100:101]
    pick = rng.integers(0, 256, (n, M))
    vec = (cb[np.arange(M)[None, :], pick] + (rng.standard_normal((n, M, 8)) * 0.3).astype(np.float32)).astype(np.float32)
    vec[:64] = cb[None, :, 100]
    vec = vec.reshape(n, M * 8)
    s = np.float32(scale)
    cb, vec = (cb * s).astype(np.float32), (vec * s).astype(np.float32)
    vec[64, 5] = np.nan
    return cb, vec


@pytest.mark.gpu
@pytest.mark.parametrize("M", [16, 48], ids=["resident-codebook", "streamed-codebook"])
@pytest.mark.parametrize("e", SCALES)
def test_pq_encode_at_every_magnitude(e, M, capfd, monkeypatch):
    n = 2000
    cb, vec = _pq_data(np.random.default_rng(8000 + M), n, M, 2.0 ** e)
    pq = lb.ProductQuantizer(M, 8, M * 8, cb)
    got, tr = _traced(lambda: pq.quantize(vec), capfd, monkeypatch)
    assert np.array_equal(got, ob.pq_encode(cb, vec, nthreads=NT))
    assert np.array_equal(got, _exact_path(lambda: pq.quantize(vec), monkeypatch))
    assert tr.launched("tc_pq_filter") == 1 and tr.launched("tc_pq_fallback") == 1
    # the rows on the 4-fold codeword went to pq_fallback_kernel (the count is printed to 0.005 % of n * M)
    assert tr.pq_pairs() >= 64 * M - 5e-5 * n * M


@pytest.mark.gpu
@pytest.mark.parametrize("e", [60, 0, -66, -76, -100])
def test_ivfpq_transform_at_every_magnitude(e, capfd, monkeypatch):
    # partition, residual and PQ code in one call: the residuals of tiny rows are tiny too
    n, d, K, M = 2000, 128, 64, 16
    rng = np.random.default_rng(8100)
    cb, vec = _pq_data(rng, n, M, 2.0 ** e)
    cent = (vec[rng.choice(np.arange(100, n), K, replace=False)] * np.float32(0.5)).astype(np.float32)
    run = lambda: lb.ivfpq_transform(cent, cb, vec)
    (part, codes, valid), tr = _traced(run, capfd, monkeypatch)
    ex = _exact_path(run, monkeypatch)
    assert np.array_equal(part, ex[0]) and np.array_equal(codes, ex[1]) and np.array_equal(valid, ex[2])
    po, _, vo = _oracle(cent, vec)
    assert np.array_equal(valid, vo) and np.array_equal(part[vo], po[vo])
    res = ob.compute_residual(cent, vec[vo], po[vo], nthreads=NT)
    assert np.array_equal(codes[vo], ob.pq_encode(cb, res, nthreads=NT))
    assert tr.filters() == {"tc_filter"} and tr.launched("tc_pq_filter") == 1


# ---- CPU: the certificate model at the magnitudes above -------------------------------------------------------------
def _flush(a):
    a = np.array(a, np.float32, copy=True)
    a[np.abs(a) < np.float32(2.0 ** -126)] = 0
    return a


def mma_scores_ftz(a, b, accumulate):
    """mma_scores with every subnormal operand, product and (sequential model) partial sum flushed to zero"""
    a, b = _flush(a).astype(np.float64), _flush(b).astype(np.float64)
    acc64 = np.zeros((a.shape[0], b.shape[0]))
    acc = np.zeros((a.shape[0], b.shape[0]), np.float32)
    for e in range(a.shape[1]):
        p = a[:, e:e + 1] * b[None, :, e]                                     # exact in f64
        p[np.abs(p) < 2.0 ** -126] = 0
        if accumulate == "exact":
            acc64 += p
        else:                                                                 # rounded toward zero, then flushed
            v = acc.astype(np.float64) + p
            r = v.astype(np.float32)
            over = np.abs(r.astype(np.float64)) > np.abs(v)
            r[over] = np.nextafter(r[over], np.float32(0.0))
            acc = _flush(r)
    return _flush(acc64.astype(np.float32)) if accumulate == "exact" else acc


def _model_rows(e, d, K, n, seed):
    """the data of the GPU magnitude cases: K Gaussian centroids and rows = a centroid + 0.3x noise, scaled by 2^e"""
    rng = np.random.default_rng(seed)
    s = np.float32(2.0 ** e)
    cent = rng.standard_normal((K, d)).astype(np.float32)
    x = (cent[rng.integers(0, K, n)] + (rng.standard_normal((n, d)) * 0.3).astype(np.float32)).astype(np.float32)
    return (cent * s).astype(np.float32), (x * s).astype(np.float32)


def _certified_wrong(x_op, c_op, cent, x, ref, scale, accumulate, ftz, floor):
    """rows certified unique whose reference argmin differs, and two-candidate rows whose argmin is neither"""
    with np.errstate(over="ignore", invalid="ignore"):
        s = (mma_scores_ftz if ftz else mma_scores)(x_op, c_op, accumulate)
        n2 = (cent * cent).sum(1, dtype=np.float32)
        s = (s + np.float32(-0.5) * n2[None, :]).astype(np.float32)
        vals, idx = top3_packed(s)
        rn = (x * x).sum(1, dtype=np.float32)
        tau = tau_of(scale, rn, n2.max()) if floor else (scale * (rn + n2.max())).astype(np.float32)
        uniq = (vals[:, 0] - vals[:, 1]) > tau
        two = ~uniq & ((vals[:, 0] - vals[:, 2]) > tau)
    return int((uniq & (idx[:, 0] != ref)).sum() + (two & (idx[:, 0] != ref) & (idx[:, 1] != ref)).sum())


@pytest.mark.parametrize("e", SCALES)
@pytest.mark.parametrize("d,K", [(128, 256), (8, 256)], ids=["ivf-128x256", "pq-subspace-8x256"])
def test_certificate_with_norm_floor_holds_at_every_magnitude(d, K, e):
    cent, x = _model_rows(e, d, K, 600, 31 + d)
    ref, _, _ = ob.compute_membership(cent, x, nthreads=NT)
    for accumulate in ("exact", "toward_zero"):
        for ftz in (False, True):
            assert _certified_wrong(tf32_trunc(x), tf32_trunc(cent), cent, x, ref, TAU_TF32, accumulate, ftz,
                                    True) == 0, (accumulate, ftz)
    # the 3xTF32 refinement operands (gather_split_kernel / split_centroids_kernel) under their own tau
    xh, ch = tf32_rne(x), tf32_rne(cent)
    a3 = np.concatenate([xh, xh, tf32_rne(x - xh)], 1)
    b3 = np.concatenate([ch, tf32_rne(cent - ch), ch], 1)
    for ftz in (False, True):
        assert _certified_wrong(a3, b3, cent, x, ref, tau3x_scale(3 * d), "toward_zero", ftz, True) == 0, ftz


def test_certificate_without_norm_floor_is_wrong_at_tiny_magnitudes():
    """the check above is not vacuous: with tau = s (|x|^2 + max|c|^2) alone, tau underflows to 0 and the model
    certifies the centroid with the largest -|c|^2/2 (or the largest packed column of an all-zero row) at 2^-76, where
    the reference's distances to nearby centroids underflow to 0 and its first minimum wins; if the MMA flushed
    subnormals, rows would already be certified wrong at 2^-66"""
    cent, x = _model_rows(-76, 128, 256, 600, 31 + 128)
    ref, _, _ = ob.compute_membership(cent, x, nthreads=NT)
    assert _certified_wrong(tf32_trunc(x), tf32_trunc(cent), cent, x, ref, TAU_TF32, "exact", False, False) > 300
    cent, x = _model_rows(-66, 128, 256, 600, 31 + 128)
    ref, _, _ = ob.compute_membership(cent, x, nthreads=NT)
    assert _certified_wrong(tf32_trunc(x), tf32_trunc(cent), cent, x, ref, TAU_TF32, "exact", False, False) == 0
    assert _certified_wrong(tf32_trunc(x), tf32_trunc(cent), cent, x, ref, TAU_TF32, "exact", True, False) > 300


def _prescreen_drops_argmin(cb, r, floor):
    """pq_fallback_kernel's FMA pre-screen (see test_filter_certificate_model.py): does it drop the reference argmin?"""
    ref, _, _ = ob.compute_membership(cb, r)
    n, K, ds = len(r), len(cb), cb.shape[1]
    n2 = np.zeros(K, np.float32)
    for t in range(ds):
        n2 = _fma(cb[:, t], cb[:, t], n2)
    rn = np.zeros(n, np.float32)
    for t in range(ds):
        rn = _fma(r[:, t], r[:, t], rn)
    s = np.broadcast_to((np.float32(-0.5) * n2)[None, :], (n, K)).astype(np.float32)
    for t in range(ds):
        s = _fma(np.broadcast_to(r[:, t:t + 1], (n, K)), np.broadcast_to(cb[None, :, t], (n, K)), s)
    with np.errstate(over="ignore", invalid="ignore"):
        t = (rn + n2.max()).astype(np.float32)
        if floor:
            t = np.where(t < NORM_FLOOR, NORM_FLOOR, t).astype(np.float32)
        thr = s.max(1) - np.float32(2.0 ** -18) * t
    return int((s[np.arange(n), ref] < thr).sum())


def test_pq_prescreen_with_norm_floor_keeps_the_argmin_at_tiny_magnitudes():
    rng = np.random.default_rng(41)
    dropped = {}
    for e in (0, -60, -66, -70, -72, -76, -80, -100):
        cb = (rng.standard_normal((256, 8)) * np.float32(2.0 ** e)).astype(np.float32)
        r = (cb[rng.integers(0, 256, 1500)] + (rng.standard_normal((1500, 8)) * 0.3).astype(np.float32)
             * np.float32(2.0 ** e)).astype(np.float32)
        assert _prescreen_drops_argmin(cb, r, True) == 0, e
        dropped[e] = _prescreen_drops_argmin(cb, r, False)
    assert dropped[0] == 0 and max(dropped.values()) > 0, dropped     # without the floor some scale loses rows
