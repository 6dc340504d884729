"""lb2_index_split / lb2_index_join and the choice helpers on the device, for every index kind, against
tests/split_join_reference.py (decisions from the oracle's per-type distances), the oracle's k-means and a numpy
restatement of the merge (tests/test_index_optimize.py)."""
import numpy as np
import pytest

import lance_b200 as lb
import rq_reference as rq
import split_join_reference as sj
import sq_reference as sqr
import test_index_optimize as tio
from oracle import binding as ob

pytestmark = pytest.mark.gpu
NT = 8
STAYS = sj.STAYS


def _bf16_bits(x):
    """f32 -> bfloat16 bit patterns, round to nearest even"""
    b = np.ascontiguousarray(x, np.float32).view(np.uint32).astype(np.uint64)
    return ((b + 0x7FFF + ((b >> 16) & 1)) >> 16).astype(np.uint16)


def _bf16_f32(bits):
    return (np.asarray(bits, np.uint32) << 16).view(np.float32)


def _as_f32(x, dt):
    return _bf16_f32(x) if dt == "bf16" else np.asarray(x, np.float32)


def _round(x, dt):
    """f32 values rounded to the model type"""
    if dt == "f16":
        return np.asarray(x, np.float32).astype(np.float16).astype(np.float32)
    if dt == "bf16":
        return _bf16_f32(_bf16_bits(x))
    return np.asarray(x, np.float32)


def _dist(metric, dt):
    """the oracle's lb2_distance_batch rule for one (from, to) pair (dot_distance = 1 - dot, dot.rs:68-70); cosine is
    the reference's own formula, which the device matches within its rounding (tests/test_linalg_primitives.py), so
    its decisions agree off exact ties"""
    if metric == "cosine":
        return lambda a, b: ob.cosine(_as_f32(a, dt), _as_f32(b, dt))
    if dt == "f16":
        f = ob.l2_f16 if metric == "l2" else ob.dot_f16
        g = lambda a, b: f(np.asarray(a, np.float16), np.asarray(b, np.float16))  # noqa: E731
    elif dt == "bf16":
        f = ob.l2_bf16 if metric == "l2" else ob.dot_bf16
        g = lambda a, b: f(*(x if np.asarray(x).dtype == np.uint16 else _bf16_bits(x) for x in (a, b)))  # noqa: E731
    else:
        g = ob.l2 if metric == "l2" else ob.dot
    if metric == "dot":
        return lambda a, b: float(np.float32(1.0) - np.float32(g(a, b)))
    return g


def _build(kind, x, metric, dt, K, seed=5, nbits=8):
    rid = np.arange(len(x), dtype=np.uint64)
    if dt == "f32" and nbits == 8:
        return tio._build(kind, x, metric, K=K, seed=seed, row_ids=rid)
    data = _raw(x, dt)
    bf = dt == "bf16"
    if kind == "pq":
        prm = lb.IvfBuildParams(num_partitions=K, num_sub_vectors=4, num_bits=nbits, max_iters=8, pq_max_iters=4,
                                seed=seed)
        return lb.IvfPqIndex.build(data, metric, prm, row_ids=rid, bf16=bf)
    assert kind == "flat"
    return lb.IvfFlatIndex.build(data, metric, num_partitions=K, max_iters=8, seed=seed, row_ids=rid, bf16=bf)


def _raw(x, dt):
    """the column as the index reads it"""
    return x if dt == "f32" else (x.astype(np.float16) if dt == "f16" else _bf16_bits(x))


def _split_inputs(ix, e, col, part):
    """the raw rows the host fetches: the partition's (ascending ids), then its candidates' grouped in order"""
    offs = e["part_offsets"].astype(np.int64)
    rid = e["row_ids"]

    def rows_of(p):
        ids = np.sort(rid[offs[p]:offs[p + 1]])
        return col[ids.astype(np.int64)], ids
    cands = ix.reassign_candidates(part)
    v, r = rows_of(part)
    cv, cr, cp = [], [], []
    for q in cands:
        a, b = rows_of(int(q))
        cv.append(a), cr.append(b), cp.append(np.full(len(b), q, np.uint32))
    return cands, v, r, np.concatenate(cv), np.concatenate(cr), np.concatenate(cp)


def _new_centroids(v, metric, dt, seed):
    """c1, c2: the oracle's k-means (k = 2) on the first 512 raw rows, normalised under cosine"""
    x = _as_f32(v[:512], dt)
    if metric == "cosine":
        x = _round(ob.normalize_rows(x, nthreads=NT), dt)
    c, _, _ = ob.kmeans_train(x, 2, max_iters=50, metric="dot" if metric == "dot" else "l2", seed=seed, nthreads=NT)
    return _round(c, dt)


def _moved_payload(kind, e, newc, rows, dest, metric, dt):
    """what the kind stores for the moved rows under the new centroids, from the oracle and the numpy restatements"""
    base = kind.replace("hnsw_", "")
    x = _as_f32(rows, dt)
    if base == "rq":  # codes and factors from the nearest new centroid (ivf.rs:301-304)
        _, codes, add, scale, valid = rq.rq_transform(newc, e["rotation"], x, metric)
        assert valid.all()
        return dict(payload=codes, add=add, scale=scale)
    if metric == "cosine":
        x = ob.normalize_rows(x, nthreads=NT)
    if base == "pq":  # residuals to the decided partition's new centroid (dot: none), PQ codes trained with L2
        nb = 4 if e["codebook"].shape[1] == 16 else 8
        r = x if metric == "dot" else ob.compute_residual(newc, x, dest, nthreads=NT)
        return dict(payload=ob.pq_encode(e["codebook"], r, nbits=nb, metric="l2", nthreads=NT))
    if base == "sq":
        return dict(payload=sqr.sq_encode(x, *e["bounds"]))
    return dict(payload=_raw(x, dt))                           # FLAT: the (normalised) row in the stored type


def _restated_split(kind, old, e, col, part, newc, cands, v, r, cv, cr, cp, dest, metric, dt):
    moved = dest != STAYS
    raw_ids = np.concatenate([r, cr])
    raw_rows = np.concatenate([v, cv])
    # add-op order: split rows, then the candidates' in candidate order -- the merge groups stably by partition
    order = np.flatnonzero(moved)
    add = dict(row_ids=raw_ids[order], **_moved_payload(kind, e, newc, raw_rows[order], dest[order], metric, dt))
    K = len(e["part_offsets"]) - 1
    pm = np.arange(K, dtype=np.uint32)
    pm[part] = tio.DROP
    return tio.merge(e["part_offsets"], tio._rows(kind, e), pm,
                     np.sort(cr[dest[len(r):] != STAYS]), dest[order], add, K + 1)


CASES = ([(k, m, "f32", 8) for k in tio.KINDS for m in ("l2", "cosine", "dot")]
         + [("pq", "dot", "f16", 8), ("pq", "dot", "bf16", 8), ("pq", "l2", "f16", 8), ("pq", "l2", "f32", 4),
            ("flat", "dot", "f16", 8), ("flat", "dot", "bf16", 8), ("flat", "l2", "bf16", 8)])


@pytest.mark.parametrize("kind,metric,dt,nbits", CASES)
def test_split_decisions_and_index_equal_restatement(kind, metric, dt, nbits):
    n, d, K, seed = 2400, 16, 9, 31
    x = tio._data(n, d, seed=11, k=K)
    col = _raw(x, dt)
    ix = _build(kind, x, metric, dt, K, nbits=nbits)
    e = ix.export()
    sizes = np.diff(e["part_offsets"]).astype(np.int64)
    part = int(np.argmax(sizes))
    cands, v, r, cv, cr, cp = _split_inputs(ix, e, col, part)
    dist = _dist(metric, dt)
    cent = e["centroids"] if dt == "f32" else _round(e["centroids"], dt)
    centc = cent if dt != "bf16" else _bf16_bits(cent)
    want_cands = sj.select_reassign_candidates([dist(centc[part], c) for c in centc], part)
    assert cands.tolist() == want_cands
    out, got = ix.split(part, v, r, cv, cr, cp, seed=seed)
    c12 = _new_centroids(v, metric, dt, seed)
    newc = np.asarray(got["new_centroids"], np.float32) if dt != "bf16" else _bf16_f32(got["new_centroids"])
    assert np.array_equal(newc[part].view(np.uint32), c12[0].view(np.uint32))
    assert np.array_equal(newc[K].view(np.uint32), c12[1].view(np.uint32))
    cc = (lambda a: _bf16_bits(a)) if dt == "bf16" else (lambda a: a)
    _, want_dest = sj.split_decisions(dist, centc, part, cc(c12[0]), cc(c12[1]), list(v), list(cv), cp)
    assert np.array_equal(got["dest"], want_dest)
    assert (got["dest"][:len(r)] != STAYS).all()
    offs, rows, src = _restated_split(kind, ix, e, col, part, newc, cands, v, r, cv, cr, cp, got["dest"], metric, dt)
    tio._check_merge(kind, ix, out, e, offs, rows, src, metric, seed)
    if dt == "f32":  # the new index searches as one loaded from its export
        ex = out.export()
        if nbits == 8:
            ld = tio._from_parts(kind, ex, metric)
        else:
            sizes = np.diff(ex["part_offsets"]).astype(np.int64)
            ld = lb.IvfPqIndex.from_parts(ex["centroids"], ex["codebook"], np.repeat(np.arange(K + 1, dtype=np.uint32), sizes),
                                          ex["codes"], ex["row_ids"], metric, num_bits=nbits)
        tio._same_search(out, ld, tio._data(8, d, seed=3, k=K))


def test_split_with_append_and_removals_and_100_partitions():
    """K = 100 (candidates cut at 64), an add list (its rows of `part` dropped, its moved rows removed) and removals"""
    n, d, K, seed = 20000, 8, 100, 4
    x = tio._data(n, d, seed=2, k=40)
    ix = lb.IvfFlatIndex.build(x, "l2", num_partitions=K, max_iters=6, seed=1, row_ids=np.arange(n, dtype=np.uint64))
    e = ix.export()
    part = int(np.argmax(np.diff(e["part_offsets"]).astype(np.int64)))
    xa = tio._data(600, d, seed=8, k=40)
    ida = np.arange(n, n + 600, dtype=np.uint64)
    t = ix.transform(xa)
    assert t["valid"].all()
    col = np.concatenate([x, xa])
    # the host's raw rows include the added rows of each partition
    offs = e["part_offsets"].astype(np.int64)
    cands = ix.reassign_candidates(part)
    assert len(cands) == 64

    def rows_of(p):
        ids = np.sort(np.concatenate([e["row_ids"][offs[p]:offs[p + 1]], ida[t["part_ids"] == p]]))
        return col[ids.astype(np.int64)], ids
    v, r = rows_of(part)
    parts = [rows_of(int(q)) for q in cands]
    cv = np.concatenate([a for a, _ in parts])
    cr = np.concatenate([b for _, b in parts])
    cp = np.concatenate([np.full(len(b), q, np.uint32) for (_, b), q in zip(parts, cands)])
    other = next(q for q in range(K) if q != part and q not in cands and offs[q + 1] - offs[q] >= 3)
    removed = np.sort(e["row_ids"][offs[other]:offs[other] + 3])      # rows of a partition the split does not touch
    assert removed.size == 3
    out, got = ix.split(part, v, r, cv, cr, cp, add_part_ids=t["part_ids"], add_payload=t["payload"], add_row_ids=ida,
                        remove_row_ids=removed, seed=seed)
    c12 = _new_centroids(v, "l2", "f32", seed)
    _, want = sj.split_decisions(ob.l2, e["centroids"], part, c12[0], c12[1], list(v), list(cv), cp)
    assert np.array_equal(got["dest"], want)
    dest = got["dest"]
    moved = dest != STAYS
    raw_ids = np.concatenate([r, cr])
    moved_cand = np.sort(cr[dest[len(r):] != STAYS])
    keep_add = (t["part_ids"] != part) & ~np.isin(ida, moved_cand)
    order = np.flatnonzero(moved)
    add = dict(row_ids=np.concatenate([ida[keep_add], raw_ids[order]]),
               payload=np.concatenate([t["payload"][keep_add], np.concatenate([v, cv])[order]]))
    pm = np.arange(K, dtype=np.uint32)
    pm[part] = tio.DROP
    o2, rows, src = tio.merge(e["part_offsets"], tio._rows("flat", e), pm, np.union1d(removed, moved_cand),
                              np.concatenate([t["part_ids"][keep_add], dest[order]]), add, K + 1)
    tio._check_merge("flat", ix, out, e, o2, rows, src, "l2", seed)
    assert sorted(out.export()["row_ids"].tolist()) == sorted(set(range(n + 600)) - set(removed.tolist()))


def test_constructed_ties_on_candidate_rows_and_join():
    """exact ties: d1 == d2 goes to c1, d0 == min(d1, d2) stays; equal candidate distances of a joined row take the
    first candidate"""
    p = np.array([1, 1, 0, 0], np.float32)
    split_rows = np.repeat(p[None], 40, 0)
    # k = 2 on identical rows: the empty cluster is split off the other, c1 / c2 = p -+ 2^-10 in two coordinates
    c12, _, _ = ob.kmeans_train(split_rows, 2, max_iters=50, seed=1, nthreads=NT)
    cent = np.stack([p, np.array([10, 10, 0, 0], np.float32), c12[0]])   # partition 2's centroid is exactly c1
    c1_tie = np.array([4, 4, 0, 0], np.float32)        # of partition 1: d1 == d2 (mirror images), d0 larger: to c1
    stay_tie = np.array([0, 2, 0, 0], np.float32)      # of partition 2: d0 == d1 < d2: stays
    vec = np.concatenate([split_rows, stay_tie[None], c1_tie[None]])
    parts = np.array([0] * 40 + [2, 1], np.uint32)
    ids = np.arange(len(vec), dtype=np.uint64)
    ix = lb.IvfFlatIndex.from_parts(cent, parts, vec, ids, "l2")
    assert ix.reassign_candidates(0).tolist() == [2, 1]
    out, got = ix.split(0, split_rows, ids[:40], vec[40:], ids[40:], parts[40:], seed=1)
    c = got["new_centroids"]
    assert np.array_equal(c[0], c12[0]) and np.array_equal(c[3], c12[1])
    _, want = sj.split_decisions(ob.l2, cent, 0, c12[0], c12[1], list(split_rows), list(vec[40:]), parts[40:])
    assert np.array_equal(got["dest"], want)
    assert got["dest"][40] == STAYS and got["dest"][41] == 0
    # join: a row equidistant to both candidates takes the first in candidate order
    cj = np.array([[0, 0, 0, 0], [0, 4, 0, 0], [0, -4, 0, 0]], np.float32)
    vj = np.array([[0, 0, 0, 0], [1, 0, 0, 0], [0, 5, 0, 0], [0, -5, 0, 0]], np.float32)
    jx = lb.IvfFlatIndex.from_parts(cj, np.array([0, 0, 1, 2], np.uint32), vj, np.arange(4, dtype=np.uint64), "l2")
    assert jx.reassign_candidates(0).tolist() == [1, 2]
    out, dest = jx.join(0, vj[:2], np.arange(2, dtype=np.uint64))
    assert dest.tolist() == [0, 0]
    ex = out.export()
    assert ex["part_offsets"].tolist() == [0, 3, 4] and ex["row_ids"].tolist() == [2, 0, 1, 3]


@pytest.mark.parametrize("kind", tio.KINDS)
def test_join_with_remap_and_edge_cases(kind):
    n, d, K, seed = 1500, 16, 5, 7
    x = tio._data(n, d, seed=5, k=K)
    ix = tio._build(kind, x, "l2", K=K, seed=3, row_ids=np.arange(n, dtype=np.uint64))
    e = ix.export()
    offs = e["part_offsets"].astype(np.int64)
    part = int(np.argmin(np.diff(offs)))
    ids = np.sort(e["row_ids"][offs[part]:offs[part + 1]])
    # a remap that drops some rows of the joined partition and of another, and rewrites one id
    other = (part + 1) % K
    gone = np.concatenate([ids[:3], e["row_ids"][offs[other]:offs[other] + 2]])
    mapping = {int(i): None for i in gone}
    keep_ids = ids[3:]
    mapping[int(keep_ids[0])] = 10_000_000
    sizes = np.diff(offs) - np.bincount(np.searchsorted(offs, np.flatnonzero(np.isin(e["row_ids"], gone)), "right") - 1,
                                        minlength=K)
    assert ix.partition_to_join(mapping) == sj.should_join(sizes.tolist(), sj.TARGET[kind])
    out, dest = ix.join(part, x[keep_ids.astype(np.int64)], keep_ids, remap=mapping, seed=seed)
    cands, want = sj.join_decisions(ob.l2, e["centroids"], part, list(x[keep_ids.astype(np.int64)]))
    assert np.array_equal(dest, want)
    add = dict(row_ids=keep_ids, **_moved_payload(kind, e, np.delete(e["centroids"], part, 0),
                                                   x[keep_ids.astype(np.int64)], dest, "l2", "f32"))
    pm = np.array([q if q < part else (tio.DROP if q == part else q - 1) for q in range(K)], np.uint32)
    o2, rows, src = tio.merge(e["part_offsets"], tio._rows(kind, e), pm, [], dest, add, K - 1, mapping)
    tio._check_merge(kind, ix, out, e, o2, rows, src, "l2", seed)
    tio._same_search(out, tio._from_parts(kind, out.export(), "l2"), tio._data(8, d, seed=3, k=K))
    # an empty joined partition: only the centroid goes
    out2, d2 = ix.join(part, np.zeros((0, d), np.float32), np.zeros(0, np.uint64))
    assert d2.size == 0 and out2.info()["num_partitions"] == K - 1 and out2.info()["num_rows"] == n - len(ids)


def test_join_two_partitions_into_one():
    x = tio._data(400, 8, seed=9, k=2)
    ix = lb.IvfFlatIndex.build(x, "dot", num_partitions=2, max_iters=5, seed=2, row_ids=np.arange(400, dtype=np.uint64))
    e = ix.export()
    offs = e["part_offsets"].astype(np.int64)
    ids = np.sort(e["row_ids"][offs[0]:offs[1]])
    out, dest = ix.join(0, x[ids.astype(np.int64)], ids)
    assert (dest == 0).all() and out.info()["num_partitions"] == 1 and out.info()["num_rows"] == 400


def test_choice_helpers_at_ivf_flat_thresholds():
    d = 4
    sizes = [16384, 16384, 1024, 1100]
    parts = np.repeat(np.arange(4, dtype=np.uint32), sizes)
    vec = np.random.default_rng(1).normal(size=(parts.size, d)).astype(np.float32)
    ix = lb.IvfFlatIndex.from_parts(np.eye(4, dtype=np.float32), parts, vec, np.arange(parts.size, dtype=np.uint64))
    assert ix.partition_to_split() is None                            # 16384 is not above 4 x 4096
    assert ix.partition_to_split(np.array([1], np.uint32)) == 1
    assert ix.partition_to_split(np.array([1, 0], np.uint32)) == 0    # equal sizes: the first
    assert ix.partition_to_join() is None                             # 1024 is not below 25% of 4096
    start = int(np.cumsum([0] + sizes)[2])
    assert ix.partition_to_join({start: None}) == 2
    assert ix.partition_to_join({start: None, start + 1024: None, start + 1025: None}) == 2   # 1023 vs 1098
    one = lb.IvfFlatIndex.from_parts(np.eye(4, dtype=np.float32)[:1], np.zeros(3, np.uint32), vec[:3])
    assert one.partition_to_join() is None


def test_refusals():
    x = tio._data(2000, 16, seed=1, k=6)
    ix = tio._build("pq", x, "l2", K=6, seed=2, row_ids=np.arange(2000, dtype=np.uint64))
    e = ix.export()
    offs = e["part_offsets"].astype(np.int64)
    part = int(np.argmax(np.diff(offs)))
    _, v, r, cv, cr, cp = _split_inputs(ix, e, x, part)
    with pytest.raises(lb.LanceB200Error):                            # a bad part
        ix.split(6, v, r)
    with pytest.raises(lb.LanceB200Error):                            # unsorted row ids
        ix.split(part, v[::-1], r[::-1])
    with pytest.raises(lb.LanceB200Error):                            # a row outside its stated partition
        ids = np.concatenate([r, cr[:1]])
        o = np.argsort(ids)
        ix.split(part, np.concatenate([v, cv[:1]])[o], ids[o])
    with pytest.raises(lb.LanceB200Error):                            # a candidate row stated for the wrong partition
        bad = cp.copy()
        bad[-1] = part
        ix.split(part, v, r, cv, cr, bad)
    with pytest.raises(lb.LanceB200Error):                            # one row
        ix.split(part, v[:1], r[:1])
    with pytest.raises(lb.LanceB200Error) as ei:                      # an add list without its row ids
        ix.split(part, v, r, cv, cr, cp, add_vectors=x[:20])
    assert ei.value.status == lb._lib.INVALID_ARG
    from lance_b200._lib import OptimizeParams, SplitParams
    import ctypes as C
    pm = np.arange(6, dtype=np.uint32)
    for field, val in (("part_map", pm.ctypes.data), ("new_centroids", e["centroids"].ctypes.data)):
        op = OptimizeParams()
        op.new_k = 6
        setattr(op, field, val)
        sp = SplitParams(part, v.ctypes.data, r.ctypes.data, len(r), None, None, None, 0, op, None, None)
        h = C.c_void_p()
        assert lb._lib.lib().lb2_index_split(ix._h, C.byref(sp), C.byref(h)) == lb._lib.INVALID_ARG
    xn = v.copy()
    xn[0, 0] = np.nan
    with pytest.raises(lb.LanceB200Error):                            # a row the transform would drop
        ix.split(part, xn, r)
    u8 = tio._build("flat", x, "l2", K=6, seed=2, dt="u8")
    with pytest.raises(lb.LanceB200Error) as ei:                      # the reference cannot split u8 columns
        u8.reassign_candidates(0)
    assert ei.value.status == lb._lib.UNSUPPORTED


@pytest.mark.parametrize("metric", ["l2", "cosine"])
def test_split_decisions_with_the_table_streamed_in_chunks(metric):
    """d = 1024: 67 centroid slots do not fit shared memory at once, the decision kernel streams them"""
    n, d, K, seed = 3000, 1024, 70, 12
    x = tio._data(n, d, seed=4, k=K)
    ix = lb.IvfFlatIndex.build(x, metric, num_partitions=K, max_iters=4, seed=3, row_ids=np.arange(n, dtype=np.uint64))
    e = ix.export()
    part = int(np.argmax(np.diff(e["part_offsets"]).astype(np.int64)))
    cands, v, r, cv, cr, cp = _split_inputs(ix, e, x, part)
    assert len(cands) == 64
    out, got = ix.split(part, v, r, cv, cr, cp, seed=seed)
    c12 = _new_centroids(v, metric, "f32", seed)
    _, want = sj.split_decisions(_dist(metric, "f32"), e["centroids"], part, c12[0], c12[1], list(v), list(cv), cp)
    assert np.array_equal(got["dest"], want)


def test_split_of_a_partition_without_raw_rows_changes_only_the_optimize():
    x = tio._data(1500, 16, seed=6, k=5)
    ix = tio._build("sq", x, "l2", K=5, seed=2, row_ids=np.arange(1500, dtype=np.uint64))
    e = ix.export()
    xa = tio._data(50, 16, seed=7, k=5)
    out, got = ix.split(1, np.zeros((0, 16), np.float32), np.zeros(0, np.uint64), add_vectors=xa,
                        add_row_ids=np.arange(1500, 1550, dtype=np.uint64), remove_row_ids=[3, 4])
    want = ix.optimize(add_vectors=xa, add_row_ids=np.arange(1500, 1550, dtype=np.uint64), remove_row_ids=[3, 4])
    a, b = out.export(), want.export()
    assert got["dest"].size == 0 and np.array_equal(got["new_centroids"], e["centroids"])
    for k in ("part_offsets", "codes", "row_ids"):
        assert np.array_equal(a[k], b[k]), k


def test_refuses_a_moved_row_the_transform_drops():
    """finite elements whose L2 sums overflow: no finite distance to any new centroid, so the transform drops the row"""
    x = tio._data(2000, 16, seed=1, k=2)
    ix = tio._build("pq", x, "l2", K=2, seed=2, row_ids=np.arange(2000, dtype=np.uint64))
    e = ix.export()
    part = int(np.argmax(np.diff(e["part_offsets"]).astype(np.int64)))
    _, v, r, cv, cr, cp = _split_inputs(ix, e, x, part)
    assert len(r) > 512                                               # the last row is not in the k-means sample
    v = v.copy()
    v[-1] = 3e19
    with pytest.raises(lb.LanceB200Error) as ei:
        ix.split(part, v, r, cv, cr, cp)
    assert ei.value.status == lb._lib.INVALID_ARG
