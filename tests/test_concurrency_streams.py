"""The threading contract of include/lance_b200.h: every symbol is re-entrant, each calling thread owns a stream,
lb2_set_stream orders a thread's later calls on a stream the caller owns and lb2_index_search_async only enqueues.

The ground truth of every check is the same call made serially on the calling thread's own stream, compared bit for
bit (ids, distance bits, counts, nprobes_out, exported arrays); the serial calls themselves are anchored to the
restatements (the oracle's IVF_FLAT search, tests/sq_reference.py, tests/rq_reference.py, tests/hnsw_reference.py).

  1. many host threads search shared indexes of every kind through every entry point at once;
  2. builds, hierarchical k-means trainings and the index-producing calls (optimize, split, join, export_storage)
     run while other threads search;
  3. under lb2_set_stream every kernel and copy of a call runs behind the caller's earlier work: the call's inputs are
     written on the caller's stream behind a long sleep, so a launch on any other stream would read a sentinel;
  4. lb2_index_search_async returns before the sleep queued ahead of it on the caller's stream has finished.

No mutating call (set_partition_index, close) runs on an index while another thread uses it."""
import threading

import numpy as np
import pytest

import lance_b200 as lb
from lance_b200._lib import DeviceArray, PinnedArray
from oracle import binding as ob

import hnsw_reference as hr
from rq_reference import ivfrq_search
from sq_reference import ivfsq_search

pytestmark = pytest.mark.gpu

THREADS, ROUNDS = 6, 2
N, D, K, NQ = 24000, 32, 6, 16
SLEEP = 200_000_000           # GPU cycles (~100 ms): far longer than the host takes to enqueue one call
SPARSE_BASE, SPARSE_STRIDE = (1 << 40) + 12345, 7
U64MAX = np.uint64(0xFFFFFFFFFFFFFFFF)

# (name, kind, metric): every index kind, a cosine and two dot indexes; the IVF_PQ index assigns through a centroid
# graph and two indexes carry sparse 64-bit row ids (their refine calls take the rows they name: refine_taken)
SPECS = [("pq8", "pq8", "l2"), ("pq4", "pq4", "cosine"), ("flat", "flat", "l2"), ("flat_f16", "flat_f16", "l2"),
         ("flat_bf16", "flat_bf16", "dot"), ("sq", "sq", "dot"), ("rq", "rq", "l2"), ("hnsw_sq", "hnsw_sq", "l2"),
         ("hnsw_pq", "hnsw_pq", "l2"), ("hnsw_flat", "hnsw_flat", "l2")]
SPARSE = {"sq", "hnsw_flat"}


def _bf16(x):
    return np.ascontiguousarray((np.ascontiguousarray(x, np.float32).view(np.uint32) >> 16).astype(np.uint16))


def _native(kind, x):
    """x in the element type of the kind's column (bf16: uint16 bit patterns)"""
    if kind == "flat_f16":
        return np.ascontiguousarray(x, np.float16)
    if kind == "flat_bf16":
        return _bf16(x)
    return np.ascontiguousarray(x, np.float32)


def _data(n, d, seed):
    """clustered rows, one cluster holding half of them: its partition passes the 4096-row scan chunk"""
    rng = np.random.default_rng(seed)
    w = np.array([0.5, 0.2, 0.1, 0.1, 0.05, 0.05])
    centres = rng.standard_normal((len(w), d)).astype(np.float32) * 6
    x = centres[rng.choice(len(w), n, p=w)] + rng.standard_normal((n, d)).astype(np.float32)
    return np.ascontiguousarray(x, np.float32)


def _build(kind, col, metric, row_ids):
    hp = lb.HnswBuildParams(max_level=4, m=8, ef_construction=40)
    bf16 = kind == "flat_bf16"
    if kind in ("pq8", "pq4", "hnsw_pq"):
        p = lb.IvfBuildParams(num_partitions=K, num_sub_vectors=8, num_bits=4 if kind == "pq4" else 8, max_iters=4,
                              pq_max_iters=4, seed=1)
        if kind == "hnsw_pq":
            return lb.IvfHnswPqIndex.build(col, metric, p, hp, row_ids=row_ids)
        return lb.IvfPqIndex.build(col, metric, p, row_ids=row_ids)
    cls = {"flat": lb.IvfFlatIndex, "flat_f16": lb.IvfFlatIndex, "flat_bf16": lb.IvfFlatIndex, "sq": lb.IvfSqIndex,
           "rq": lb.IvfRqIndex, "hnsw_sq": lb.IvfHnswSqIndex, "hnsw_flat": lb.IvfHnswFlatIndex}[kind]
    kw = dict(hnsw_params=hp) if kind.startswith("hnsw") else {}
    if bf16:
        kw["bf16"] = True
    return cls.build(col, metric, num_partitions=K, max_iters=4, seed=1, row_ids=row_ids, **kw)


def _bitmap(n, rows):
    bm = np.zeros((n + 63) // 64, np.uint64)
    rows = np.asarray(rows, np.int64)
    np.bitwise_or.at(bm, rows >> 6, np.left_shift(np.uint64(1), (rows & 63).astype(np.uint64)))
    return bm


class Entry(dict):
    __getattr__ = dict.__getitem__


@pytest.fixture(scope="module")
def indexes():
    """one small index of every kind, each with an empty partition and one past 4096 rows, and each call's inputs"""
    lb.set_device(0)
    out = {}
    for si, (name, kind, metric) in enumerate(SPECS):
        rng = np.random.default_rng(7000 + si)
        x = _data(N, D, seed=100 + si)
        col = _native(kind, x)
        sparse = name in SPARSE
        rid = (SPARSE_BASE + SPARSE_STRIDE * np.arange(N, dtype=np.uint64)).astype(np.uint64) if sparse else None
        built = _build(kind, col, metric, rid)
        e0 = built.export()
        sizes = np.diff(e0["part_offsets"].astype(np.int64))
        small = int(np.argmin(sizes))
        gone = e0["row_ids"][e0["part_offsets"][small]:e0["part_offsets"][small + 1]]
        ix = built.optimize(remove_row_ids=gone)                       # the smallest partition, emptied
        built.close()
        if name == "pq8":
            ix.set_partition_index("hnsw", seed=3)                      # before any thread uses the index
        e = ix.export()
        sizes = np.diff(e["part_offsets"].astype(np.int64))
        assert sizes.min() == 0 and sizes.max() > 4096, (name, sizes)
        kept = np.setdiff1d(np.arange(N), (gone - SPARSE_BASE) // SPARSE_STRIDE if sparse else gone)
        q = _native(kind, x[rng.choice(kept, NQ, replace=False)] + rng.standard_normal((NQ, D)).astype(np.float32))
        n_store = int(e["row_ids"].size)
        bm = ix.row_mask(rng.choice(e["row_ids"], n_store // 2, replace=False), None)
        sel = ix.row_mask(rng.choice(e["row_ids"], 40, replace=False), None)   # selective: the late search runs
        _, pd = ix.search(q, k=50, nprobes=K)
        finite = pd[np.isfinite(pd)]
        lo, hi = float(np.quantile(finite, 0.05)), float(np.quantile(finite, 0.7))
        ucount = 700                                                    # unindexed rows (ids past the column)
        ux = _native(kind, _data(ucount, D, seed=900 + si))
        uid = np.arange(N, N + ucount, dtype=np.uint64)
        hnsw = kind.startswith("hnsw")
        ks = rng.integers(1, 31, NQ)
        rf = np.where(rng.random(NQ) < 0.5, rng.integers(1, 5, NQ), 0)
        ef = np.where(rng.random(NQ) < 0.5, ks * np.maximum(rf, 1) + rng.integers(0, 30, NQ), 0) if hnsw else None
        out[name] = Entry(
            name=name, kind=kind, metric=metric, ix=ix, x=x, col=col, q=q, sparse=sparse, rid=rid, hnsw=hnsw,
            bf16=kind == "flat_bf16", export=e, bm=bm, sel=sel, lo=lo, hi=hi, qdev=DeviceArray.from_numpy(q),
            coldev=DeviceArray.from_numpy(col), ux=ux, uid=uid, ubm=_bitmap(ucount, rng.choice(ucount, 300, False)),
            fbm=_bitmap(N, rng.choice(N, N // 3, replace=False)), ks=ks, rf=rf, ef=ef,
            nps=np.where(rng.random(NQ) < 0.3, 0, rng.integers(1, K + 3, NQ)), fof=rng.integers(-1, 2, NQ),
            qlo=np.where(rng.random(NQ) < 0.2, lo, np.nan).astype(np.float32),
            qhi=np.where(rng.random(NQ) < 0.2, hi, np.nan).astype(np.float32),
            cent=np.ascontiguousarray(e["centroids"], np.float32),
            pi=lb.PartitionIndex.build(e["centroids"], "l2", mode="hnsw", seed=5))
    yield out
    for e in out.values():
        e.pi.close()
        e.ix.close()


def _taken_rows(e, ids):
    """the column's rows of the row ids `ids`"""
    ids = np.asarray(ids, np.uint64)
    rows = (ids - np.uint64(SPARSE_BASE)) // np.uint64(SPARSE_STRIDE) if e.sparse else ids
    return e.col[rows.astype(np.int64)]


def _calls(e, q=None):
    """{call name: () -> tuple of arrays}: every entry point over index e (queries q, default e.q)"""
    ix = e.ix
    q = e.q if q is None else q
    dt = {"bf16": True} if e.bf16 else {}
    refine = {} if e.sparse else dict(refine_factor=2, vectors=e.col)
    c = {
        "search": lambda: ix.search(q, k=10, nprobes=3),
        "search_ex": lambda: ix.search_ex(q, k=10, nprobes=4, allow_bitmap=e.bm, lower_bound=e.lo,
                                          upper_bound=e.hi, **refine),
        "search_probed": lambda: ix.search_probed(q, k=10, minimum_nprobes=1, maximum_nprobes=K, late_width=4,
                                                  allow_bitmap=e.sel),
        "search_batch": lambda: ix.search_batch(q, k=e.ks, nprobes=e.nps, refine_factor=0 if e.sparse else e.rf,
                                                vectors=None if e.sparse else e.col, filters=[e.bm, e.sel],
                                                filter_of=e.fof, lower_bound=e.qlo, upper_bound=e.qhi, ef=e.ef,
                                                late_width=3),
        "candidates_refine_taken": lambda: _candidates_refine(e, q),
        "flat_search": lambda: lb.flat_search(e.col, q, 10, e.metric, allow_bitmap=e.fbm, **dt),
        "flat_search_batch": lambda: lb.flat_search_batch(e.col, q, e.ks, e.metric, filters=[e.fbm, None],
                                                          filter_of=e.fof, lower_bound=e.qlo, **dt),
        "compute_partitions_f16": lambda: lb.compute_partitions(e.cent.astype(np.float16),
                                                                e.x[:3000].astype(np.float16)),
        "partition_index_assign": lambda: e.pi.assign(e.x[:3000]),
        "transform": lambda: tuple(v for v in ix.transform(e.col[:3000]).values() if v is not None),
    }
    if not e.sparse:
        c["search_ex_device_refine"] = lambda: ix.search_ex(e.qdev, k=7, nprobes=K, refine_factor=3,
                                                            vectors=e.coldev)
        c["search_combined_batch"] = lambda: ix.search_combined_batch(
            q, e.ks, e.col, e.ux, e.uid, nprobes=3, refine_factor=e.rf, filters=[e.bm], filter_of=np.minimum(e.fof, 0),
            unindexed_filters=[e.ubm], ef=e.ef)
    if e.hnsw:
        c["search_hnsw_ef"] = lambda: ix.search(q, k=10, nprobes=3, ef=40)
    return c


def _candidates_refine(e, q):
    ids, dists, counts, probes, uniq, pos = e.ix.search_candidates(q, e.ks, nprobes=3, refine_factor=4,
                                                                    filters=[e.bm], filter_of=np.minimum(e.fof, 0),
                                                                    distinct=True)
    got = e.ix.refine_taken(q, (ids, dists, counts), _taken_rows(e, uniq), pos, e.ks, refine_factor=4)
    return (ids, dists, counts, probes, uniq, pos) + tuple(got)


def _arrays(r):
    if isinstance(r, dict):
        return tuple(np.asarray(v) for v in r.values() if v is not None and not np.isscalar(v))
    if isinstance(r, (tuple, list)):
        return tuple(a for x in r for a in _arrays(x))
    if isinstance(r, DeviceArray):
        return (r.numpy(),)
    return () if r is None else (np.asarray(r),)


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view({2: np.uint16, 4: np.uint32, 8: np.uint64}[a.itemsize]) if a.dtype.kind == "f" else a


def _same(got, want, what):
    got, want = _arrays(got), _arrays(want)
    assert len(got) == len(want), what
    for i, (g, w) in enumerate(zip(got, want)):
        assert g.shape == w.shape and np.array_equal(_bits(g), _bits(w)), (what, i)


def _timed(fn):
    """(fn's arrays, kernel launches of this thread during the call)"""
    l0 = lb.launch_count()
    r = _arrays(fn())
    return r, lb.launch_count() - l0


def _run_threads(workers):
    """run every worker on its own thread, join them all; the exceptions they raised"""
    errs, lock = [], threading.Lock()

    def wrap(f):
        def run():
            try:
                f()
            except BaseException as ex:  # noqa: BLE001 - reported by the caller
                with lock:
                    errs.append(ex)
        return run
    th = [threading.Thread(target=wrap(f)) for f in workers]
    for t in th:
        t.start()
    for t in th:
        t.join()
    return errs


def _search_worker(pairs, calls, base, seed, rounds, failures):
    """a worker that runs (index, call) pairs in its own shuffled order and checks each against its baseline"""
    def work():
        rng = np.random.default_rng(seed)
        for _ in range(rounds):
            for i in rng.permutation(len(pairs)):
                key = pairs[i]
                got, launches = _timed(calls[key])
                want, want_launches = base[key]
                try:
                    _same(got, want, key)
                    assert launches == want_launches, (key, launches, want_launches)
                except AssertionError as ex:
                    failures.append(ex)
    return work


# ---- the serial baseline against the restatements ------------------------------------------------------------------
def _same_as_restatement(got, want):
    (gi, gd), (wi, wd, wc) = got, want
    for i in range(wi.shape[0]):
        c = int(wc[i])
        assert np.array_equal(gi[i, :c], wi[i, :c]), i
        assert np.array_equal(gd[i, :c].view(np.uint32), wd[i, :c].view(np.uint32)), i
        assert (gi[i, c:] == U64MAX).all() and np.isinf(gd[i, c:]).all(), i


def test_serial_baseline_equals_the_restatements(indexes):
    """the calls the threads are checked against compute what the reference computes"""
    e = indexes["flat"]
    p = e.export
    _same_as_restatement(_calls(e)["search"](),
                         ob.ivfflat_search(p["centroids"], p["part_offsets"], p["vectors"], p["row_ids"], e.q, 10, 3))
    e = indexes["sq"]
    p = e.export
    _same_as_restatement(_calls(e)["search"](), ivfsq_search(p["centroids"], p["bounds"], p["part_offsets"], p["codes"],
                                                             p["row_ids"], e.q, 10, 3, metric="dot"))
    e = indexes["rq"]
    p = e.export
    _same_as_restatement(_calls(e)["search"](), ivfrq_search(p["centroids"], p["rotation"], p["part_offsets"],
                                                             p["codes"], p["add_factors"], p["scale_factors"],
                                                             p["row_ids"], e.q, 10, 3))
    e = indexes["hnsw_sq"]
    p = e.export
    q = e.q[:6]
    _same_as_restatement(_calls(e, q)["search_hnsw_ef"](),
                         hr.search(p["centroids"], p["bounds"], p["part_offsets"], p["codes"], p["row_ids"],
                                   p["graph"], q, 10, 3, ef=40))


# ---- 1. concurrent searches of shared indexes ----------------------------------------------------------------------
def test_concurrent_searches_of_every_kind_and_entry_point(indexes, monkeypatch):
    """THREADS threads, each through its own shuffled list of every (index, call) pair, ROUNDS times: every result and
    every call's launch count equal the serial call's"""
    monkeypatch.setenv("LB2_CHUNK_ROWS", "3000")      # the flat searches stage the host column through both slots
    calls = {(name, c): f for name, e in indexes.items() for c, f in _calls(e).items()}
    pairs = sorted(calls)
    base = {key: _timed(calls[key]) for key in pairs}
    failures = []
    errs = _run_threads([_search_worker(pairs, calls, base, 11 + t, ROUNDS, failures) for t in range(THREADS)])
    assert not errs, errs
    assert not failures, failures[:5]


# ---- 2. builds and index-producing calls alongside other work ------------------------------------------------------
def _export(ix):
    try:
        e = ix.export()
        g = e.pop("graph", None)
        return (tuple(np.asarray(v) for v in e.values() if not isinstance(v, tuple)) + tuple(e.get("bounds", ()))
                + (() if g is None else tuple(np.asarray(v) for v in g.values())))
    finally:
        ix.close()


def _build_jobs(seed):
    rng = np.random.default_rng(seed)
    x = _data(30000, 64, seed)
    pinned = PinnedArray(x.shape, np.float32)
    pinned.array[...] = x
    xb = _bf16(_data(4000, 1536, seed + 1))
    bdev = DeviceArray.from_numpy(xb)
    xs = _data(20000, 32, seed + 2)
    ka, kb = _data(20000, 16, seed + 3), _data(24000, 16, seed + 4) + rng.standard_normal(16).astype(np.float32)
    pq = lb.IvfBuildParams(num_partitions=24, num_sub_vectors=16, max_iters=4, pq_max_iters=4, seed=2)
    hp = lb.HnswBuildParams(max_level=4, m=8, ef_construction=40)
    jobs = {
        "ivf_pq_host": lambda: _export(lb.IvfPqIndex.build(x, "l2", pq)),
        "ivf_pq_pinned": lambda: _export(lb.IvfPqIndex.build(pinned, "l2", pq)),
        "ivf_flat_bf16_device": lambda: _export(lb.IvfFlatIndex.build(bdev, "dot", num_partitions=12, max_iters=4,
                                                                     bf16=True)),
        "ivf_sq": lambda: _export(lb.IvfSqIndex.build(xs, "l2", num_partitions=16, max_iters=4)),
        "ivf_rq": lambda: _export(lb.IvfRqIndex.build(xs, "cosine", num_partitions=16, max_iters=4)),
        "ivf_hnsw_pq": lambda: _export(lb.IvfHnswPqIndex.build(
            xs, "l2", lb.IvfBuildParams(num_partitions=8, num_sub_vectors=8, max_iters=4, pq_max_iters=4), hp)),
        "kmeans_300": lambda: lb.train_kmeans(ka, 16, 300, max_iters=4, seed=3).centroids,
        "kmeans_520": lambda: lb.train_kmeans(kb, 16, 520, max_iters=4, seed=4).centroids,
    }
    return jobs, (pinned, bdev)


@pytest.mark.parametrize("resident", [None, "0"], ids=["resident", "streamed"])
def test_builds_and_trainings_alongside_searches(indexes, monkeypatch, resident):
    """every build and two hierarchical trainings (sharing the split-worker pool) at once, each on its own thread,
    while two threads search: exports, centroids and the trainings' launch counts equal the serial runs'"""
    if resident is None:
        monkeypatch.delenv("LB2_MAX_RESIDENT_MB", raising=False)
    else:
        monkeypatch.setenv("LB2_MAX_RESIDENT_MB", resident)
    jobs, keep = _build_jobs(41)
    try:
        base = {name: _timed(f) for name, f in jobs.items()}
        for name in ("kmeans_300", "kmeans_520"):    # a hierarchical training launches the same kernels every run
            assert _timed(jobs[name])[1] == base[name][1], name
        calls = {(name, c): f for name in ("pq8", "flat_bf16", "hnsw_sq", "rq")
                 for c, f in _calls(indexes[name]).items()}
        pairs = sorted(calls)
        sbase = {key: _timed(calls[key]) for key in pairs}
        got, failures = {}, []

        def job(name):
            def run():
                got[name] = _timed(jobs[name])
            return run
        errs = _run_threads([job(name) for name in jobs] +
                            [_search_worker(pairs, calls, sbase, 60 + t, 1, failures) for t in range(2)])
        assert not errs, errs
        assert not failures, failures[:5]
        for name, (want, launches) in base.items():
            _same(got[name][0], want, name)
            if name.startswith("kmeans"):
                assert got[name][1] == launches, (name, got[name][1], launches)
    finally:
        keep[0].free()                               # pinned memory is not freed with its Python object


def _derived(e):
    """optimize (append + remove), split, join and export_storage of index e -> {name: arrays}"""
    ix, p = e.ix, e.export
    offs = p["part_offsets"].astype(np.int64)
    sizes = np.diff(offs)

    def rows_of(part):
        ids = np.sort(p["row_ids"][offs[part]:offs[part + 1]])
        return e.col[ids.astype(np.int64)], ids
    add = _native(e.kind, _data(500, D, seed=77))
    out = {}
    o = ix.optimize(add_vectors=add, add_row_ids=np.arange(N, N + 500, dtype=np.uint64),
                    remove_row_ids=p["row_ids"][::9])
    out["optimize"] = _export(o)
    big = int(np.argmax(sizes))
    v, r = rows_of(big)
    cands = ix.reassign_candidates(big)
    cv, cr, cp = zip(*[rows_of(int(c)) + (np.full(int(sizes[c]), c, np.uint32),) for c in cands])
    s, info = ix.split(big, v, r, np.concatenate(cv), np.concatenate(cr), np.concatenate(cp), seed=5)
    out["split"] = _export(s) + (info["new_centroids"], info["dest"])
    small = int(np.argmin(np.where(sizes > 0, sizes, np.iinfo(np.int64).max)))
    v, r = rows_of(small)
    j, dest = ix.join(small, v, r, seed=6)
    out["join"] = _export(j) + (dest,)
    out["export_storage"] = _arrays(ix.export_storage())
    return out


def test_index_producing_calls_while_the_source_is_searched(indexes):
    """optimize, split, join and export_storage of an index that two other threads search: the derived indexes equal
    the serial ones, and the source's exports and search results are unchanged"""
    e = indexes["flat"]
    want = _derived(e)
    before = _export_keep(e.ix)
    calls = {("flat", c): f for c, f in _calls(e).items()}
    pairs = sorted(calls)
    sbase = {key: _timed(calls[key]) for key in pairs}
    got, failures = {}, []

    def derive():
        got.update(_derived(e))
    errs = _run_threads([derive] + [_search_worker(pairs, calls, sbase, 80 + t, 2, failures) for t in range(2)])
    assert not errs, errs
    assert not failures, failures[:5]
    for name, w in want.items():
        _same(got[name], w, name)
    _same(_export_keep(e.ix), before, "source export")
    for key in pairs:
        _same(_timed(calls[key])[0], sbase[key][0], key)


def _export_keep(ix):
    return _arrays(ix.export())


# ---- 3. caller streams: lb2_set_stream orders the library behind the caller's work ---------------------------------
def _torch():
    import torch  # CUDA streams, events and the sleep kernel only
    return torch


class TorchArray(DeviceArray):
    """a DeviceArray view of a torch tensor's memory (torch owns and frees it)"""

    def __init__(self, t, dtype):
        self.t, self.shape, self.dtype = t, tuple(t.shape), np.dtype(dtype)
        self.nbytes = t.numel() * t.element_size()
        self.ptr = t.data_ptr()

    def free(self):
        self.ptr = None


def _device_tensor(torch, a):
    """a contiguous device tensor of the bits of a (uint16 = bf16 bit patterns)"""
    a = np.ascontiguousarray(a)
    if a.dtype == np.uint16:
        return torch.from_numpy(a.view(np.int16)).cuda().view(torch.bfloat16)
    return torch.from_numpy(a).cuda()


# Every input but the one written behind the sleep is device memory, allocated before the sleep is queued: a
# pageable host input would be uploaded on the caller's stream, and the driver may hold the host there until the
# sleep has ended, after which a launch on the wrong stream would find the real values.  The only host inputs left
# are the per-query parameter tables of the batch calls (a few hundred bytes).
STREAM_CASES = ["search_pq8", "search_pq4", "search_ex", "search_ex_device_refine", "search_probed", "search_batch",
                "search_candidates", "refine_taken", "search_hnsw_ef", "search_combined_batch", "flat_search",
                "flat_search_batch", "transform", "compute_partitions_f16", "partition_index_assign"]


@pytest.fixture(scope="module")
def device_inputs(indexes):
    """the auxiliary inputs of every index as device arrays: bitmaps, the unindexed rows and their filter"""
    out = {}
    for name, e in indexes.items():
        out[name] = Entry({k: DeviceArray.from_numpy(e[k]) for k in ("bm", "sel", "fbm", "ux", "uid", "ubm")})
    return out


def _stream_case(name, ix, dev):
    """(index entry, the input written behind the sleep, fn(input buffer) -> result); all eight kinds over the cases"""
    if name in ("search_pq8", "search_pq4"):
        e = ix[name[7:]]
        return e, e.q, lambda b: e.ix.search(b, k=10, nprobes=3)
    if name == "search_ex":
        e, d = ix["flat_f16"], dev["flat_f16"]
        return e, e.q, lambda b: e.ix.search_ex(b, k=10, nprobes=4, allow_bitmap=d.bm, lower_bound=e.lo,
                                                upper_bound=e.hi, refine_factor=2, vectors=e.coldev)
    if name == "search_ex_device_refine":
        e = ix["flat"]
        return e, e.q, lambda b: e.ix.search_ex(b, k=7, nprobes=K, refine_factor=3, vectors=e.coldev)
    if name == "search_probed":
        e, d = ix["sq"], dev["sq"]
        return e, e.q, lambda b: e.ix.search_probed(b, k=10, minimum_nprobes=1, maximum_nprobes=K, late_width=4,
                                                    allow_bitmap=d.sel)
    if name == "search_batch":
        e, d = ix["hnsw_sq"], dev["hnsw_sq"]
        return e, e.q, lambda b: e.ix.search_batch(b, k=e.ks, nprobes=e.nps, refine_factor=e.rf, vectors=e.coldev,
                                                   filters=[d.bm, d.sel], filter_of=e.fof, lower_bound=e.qlo,
                                                   upper_bound=e.qhi, ef=e.ef, late_width=3)
    if name == "search_candidates":
        e, d = ix["hnsw_flat"], dev["hnsw_flat"]
        return e, e.q, lambda b: e.ix.search_candidates(b, e.ks, nprobes=3, refine_factor=4, filters=[d.bm],
                                                        filter_of=np.minimum(e.fof, 0), distinct=True)
    if name == "refine_taken":
        # the candidates of the real queries, then only refine_taken's queries written behind the sleep
        e, d = ix["hnsw_flat"], dev["hnsw_flat"]
        ids, dists, counts, _, uniq, pos = e.ix.search_candidates(e.q, e.ks, nprobes=3, refine_factor=4,
                                                                  filters=[e.bm], filter_of=np.minimum(e.fof, 0),
                                                                  distinct=True)
        cand = tuple(DeviceArray.from_numpy(a) for a in (ids, dists, counts))
        taken, posd = DeviceArray.from_numpy(_taken_rows(e, uniq)), DeviceArray.from_numpy(pos)
        return e, e.q, lambda b: e.ix.refine_taken(b, cand, taken, posd, e.ks, refine_factor=4)
    if name == "search_hnsw_ef":
        e = ix["hnsw_pq"]
        return e, e.q, lambda b: e.ix.search(b, k=10, nprobes=3, ef=40)
    if name == "search_combined_batch":
        e, d = ix["flat"], dev["flat"]
        return e, e.q, lambda b: e.ix.search_combined_batch(
            b, e.ks, e.coldev, d.ux, d.uid, nprobes=3, refine_factor=e.rf, filters=[d.bm],
            filter_of=np.minimum(e.fof, 0), unindexed_filters=[d.ubm])
    if name == "flat_search":
        e, d = ix["flat_bf16"], dev["flat_bf16"]
        return e, e.q, lambda b: lb.flat_search(e.coldev, b, 10, e.metric, allow_bitmap=d.fbm, bf16=True)
    if name == "flat_search_batch":
        e, d = ix["flat_bf16"], dev["flat_bf16"]
        return e, e.q, lambda b: lb.flat_search_batch(e.coldev, b, e.ks, e.metric, filters=[d.fbm, None],
                                                      filter_of=e.fof, lower_bound=e.qlo, bf16=True)
    e = ix["rq"]
    rows = np.ascontiguousarray(e.x[:3000], np.float32)
    if name == "transform":
        return e, rows, lambda b: _arrays(e.ix.transform(b))
    if name == "compute_partitions_f16":
        cent = e.cent.astype(np.float16)
        return e, rows.astype(np.float16), lambda b: lb.compute_partitions(cent, b)
    assert name == "partition_index_assign", name
    return e, rows, lambda b: e.pi.assign(b)


def _behind_sleep(torch, stream, buf, real):
    """on `stream`: the sentinel into buf, a long sleep, then the real values"""
    with torch.cuda.stream(stream):
        buf.fill_(float("nan") if buf.dtype.is_floating_point else 0)
        torch.cuda._sleep(SLEEP)
        buf.copy_(real)


@pytest.mark.parametrize("case", STREAM_CASES)
def test_set_stream_orders_the_call_behind_the_callers_work(indexes, device_inputs, case):
    """the call's input written on the caller's stream behind a sleep: the call under lb2_set_stream equals the
    serial call; a kernel or copy of the call on any other stream would read the sentinel"""
    torch = _torch()
    e, a, fn = _stream_case(case, indexes, device_inputs)
    real = _device_tensor(torch, a)                  # everything allocated first, kept until the end
    buf = torch.empty_like(real)
    torch.cuda.synchronize()
    want = _arrays(fn(TorchArray(real, a.dtype)))
    s = torch.cuda.Stream()
    _behind_sleep(torch, s, buf, real)
    lb.set_stream(s.cuda_stream)
    try:
        got = _arrays(fn(TorchArray(buf, a.dtype)))
    finally:
        lb.set_stream(None)
    s.synchronize()
    _same(got, want, case)


def test_after_set_stream_none_a_call_does_not_wait_for_the_callers_stream(indexes):
    torch = _torch()
    e = indexes["pq8"]
    qd = DeviceArray.from_numpy(e.q)
    want = _arrays(e.ix.search(qd, k=10, nprobes=3))
    s = torch.cuda.Stream()
    lb.set_stream(s.cuda_stream)
    lb.set_stream(None)
    slept = torch.cuda.Event()
    with torch.cuda.stream(s):
        torch.cuda._sleep(2 * SLEEP)
        slept.record(s)
    got = _arrays(e.ix.search(qd, k=10, nprobes=3))
    assert not slept.query(), "a call after set_stream(None) waited for the caller's stream"
    s.synchronize()
    _same(got, want, "search")


def test_set_stream_orders_a_build_from_device_rows_behind_the_callers_work():
    torch = _torch()
    x = _bf16(_data(20000, 64, seed=55))
    real = _device_tensor(torch, x)
    buf = torch.empty_like(real)
    torch.cuda.synchronize()

    def build(b):
        return _export(lb.IvfFlatIndex.build(TorchArray(b, np.uint16), "l2", num_partitions=12, max_iters=4,
                                             bf16=True))
    want = build(real)
    s = torch.cuda.Stream()
    _behind_sleep(torch, s, buf, real)
    lb.set_stream(s.cuda_stream)
    try:
        got = build(buf)
    finally:
        lb.set_stream(None)
    s.synchronize()
    _same(got, want, "build")


# ---- 4. lb2_index_search_async for every index kind ---------------------------------------------------------------
def test_search_async_only_enqueues_for_every_kind(indexes):
    """search_async on two caller streams, device and pinned outputs, a bitmap and a range, a done_event on the last
    call: each call returns while the sleep queued ahead of it still runs, and the results equal search_ex"""
    torch = _torch()
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    done = torch.cuda.Event()
    done.record()                                      # torch creates the cudaEvent_t lazily
    names = [name for name, _, _ in SPECS]
    want, args = {}, {}
    for i, name in enumerate(names):                   # everything allocated first, kept until the end
        e = indexes[name]
        q = DeviceArray.from_numpy(e.q) if i % 2 == 0 else PinnedArray(e.q.shape, e.q.dtype)
        if isinstance(q, PinnedArray):
            q.array[...] = e.q
        mk = DeviceArray if i % 3 else PinnedArray
        out = (mk((NQ, 10), np.uint64), mk((NQ, 10), np.float32))
        warm = (DeviceArray((NQ, 10), np.uint64), DeviceArray((NQ, 10), np.float32))
        args[name] = (q, out, DeviceArray.from_numpy(e.bm), warm)
        want[name] = e.ix.search_ex(e.q, k=10, nprobes=3, allow_bitmap=e.bm, lower_bound=e.lo, upper_bound=e.hi)
    try:
        def kw(name):
            return dict(k=10, nprobes=3, allow_bitmap=args[name][2], lower_bound=indexes[name].lo,
                        upper_bound=indexes[name].hi)
        for i, name in enumerate(names):               # one warm-up call per kind
            indexes[name].ix.search_async(args[name][0], args[name][3], cuda_stream=streams[i % 2].cuda_stream,
                                          **kw(name))
        torch.cuda.synchronize()
        slept = [torch.cuda.Event() for _ in names]
        for i, name in enumerate(names):
            s = streams[i % 2]
            with torch.cuda.stream(s):
                torch.cuda._sleep(SLEEP)
                slept[i].record(s)
            indexes[name].ix.search_async(args[name][0], args[name][1], cuda_stream=s.cuda_stream,
                                          done_event=done.cuda_event if i == len(names) - 1 else None, **kw(name))
            assert not slept[i].query() and not s.query(), f"{name}: search_async waited for the stream"
        done.synchronize()
        for s in streams:
            s.synchronize()
        for name in names:
            out = args[name][1]
            got = tuple(o.numpy() if isinstance(o, DeviceArray) else o.array.copy() for o in out)
            _same(got, want[name], name)
            _same(tuple(o.numpy() for o in args[name][3]), want[name], name + " (warm-up)")
    finally:
        torch.cuda.synchronize()
        for q, out, _, _ in args.values():           # pinned memory is not freed with its Python object
            for a in (q,) + out:
                if isinstance(a, PinnedArray):
                    a.free()
