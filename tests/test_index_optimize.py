"""lb2_index_transform and lb2_index_optimize for every index kind, against numpy restatements of the merge
(build_partitions / take_partition_batches, rust/lance/src/index/vector/builder.rs:685-935), of storage.remap
(lance-index/src/vector/pq/storage.rs:499-540) and of the unchanged-partition rule of include/lance_b200.h, and
against the graph restatements of tests/hnsw_reference.py, hnsw_pq_reference.py and hnsw_flat_reference.py."""
import numpy as np
import pytest

import lance_b200 as lb
import hnsw_flat_reference as hf
import hnsw_pq_reference as pr
import hnsw_reference as hr

NONE = np.uint64(0xFFFFFFFFFFFFFFFF)
DROP = np.uint32(0xFFFFFFFF)
HNSW = dict(max_level=4, m=6, ef_construction=24)


# ---- numpy restatements (no GPU) ------------------------------------------------------------------------------------
def storage_remap(row_ids, mapping):
    """storage.remap: (keep mask, new ids) in the same order; ids mapped to None dropped, ids mapped to a value
    rewritten, ids not in the mapping unchanged"""
    keep = np.ones(len(row_ids), bool)
    out = np.array(row_ids, np.uint64, copy=True)
    for i, r in enumerate(row_ids):
        r = int(r)
        if r in mapping:
            if mapping[r] is None:
                keep[i] = False
            else:
                out[i] = mapping[r]
    return keep, out


def merge(old_offsets, old_rows, part_map, removed, add_part, add_rows, new_k, mapping=None):
    """the merge of lb2_index_optimize over row records (any per-row arrays in a dict, "row_ids" among them) ->
    (new offsets, rows in the new storage order, src): src[p] = the old partition whose graph p keeps, or -1"""
    offs = np.asarray(old_offsets, np.int64)
    ok = len(offs) - 1
    pm = np.arange(ok, dtype=np.int64) if part_map is None else np.asarray(part_map, np.int64)
    old_part = np.repeat(np.arange(ok), np.diff(offs))
    newp = pm[old_part] if len(old_part) else np.zeros(0, np.int64)
    keep_old = (newp != int(DROP)) & ~np.isin(old_rows["row_ids"], np.asarray(removed, np.uint64))
    parts = np.concatenate([newp, np.asarray(add_part, np.int64)])
    keep = np.concatenate([keep_old, np.ones(len(add_part), bool)])
    rows = {k: np.concatenate([old_rows[k], add_rows[k]]) for k in old_rows}
    if mapping:
        km, rows["row_ids"] = storage_remap(rows["row_ids"], mapping)
        keep &= km
    order = np.argsort(np.where(keep, parts, new_k), kind="stable")[:int(keep.sum())]
    counts = np.bincount(parts[keep], minlength=new_k)
    new_offs = np.concatenate([[0], np.cumsum(counts)]).astype(np.uint64)
    out = {k: v[order] for k, v in rows.items()}
    # the unchanged rule: q lost no row (removed, dropped with its partition or remapped to None), nothing was
    # added to p = part_map[q], and p holds exactly q's rows
    lost = np.bincount(old_part[~keep[:len(old_part)]], minlength=ok)
    added = np.bincount(np.asarray(add_part, np.int64), minlength=new_k)
    src = np.full(new_k, -1, np.int64)
    for q in range(ok):
        p, rows_q = int(pm[q]), int(offs[q + 1] - offs[q])
        if p == int(DROP) or rows_q == 0 or lost[q] or added[p] or counts[p] != rows_q:
            continue
        src[p] = q
    return new_offs, out, src


def graph_slice(g, offs, p):
    """partition p's rows of a graph in the device layout: (levels, counts0, neighbors0, dists0, counts_up,
    neighbors_up, dists_up)"""
    a, b = int(offs[p]), int(offs[p + 1])
    up = np.concatenate([[0], np.cumsum(np.asarray(g["levels"], np.int64) - 1)])
    ua, ub = int(up[a]), int(up[b])
    return (g["levels"][a:b], g["counts0"][a:b], g["neighbors0"][a:b], g["dists0"][a:b], g["counts_up"][ua:ub],
            g["neighbors_up"][ua:ub], g["dists_up"][ua:ub])


def assemble(new_offs, src, rebuilt, old_graph, old_offs):
    """the graph of a merge: kept partitions from old_graph, the others from `rebuilt` (a full graph over the new
    storage)"""
    keys = ("levels", "counts0", "neighbors0", "dists0", "counts_up", "neighbors_up", "dists_up")
    parts = []
    for p in range(len(new_offs) - 1):
        parts.append(graph_slice(old_graph, old_offs, src[p]) if src[p] >= 0 else graph_slice(rebuilt, new_offs, p))
    out = {k: np.concatenate([s[i] for s in parts]) for i, k in enumerate(keys)}
    for k in ("max_level", "m", "ef_construction"):
        out[k] = rebuilt[k]
    return out


def test_storage_remap_restatement():
    ids = np.array([5, 3, 9, 7, 1], np.uint64)
    keep, out = storage_remap(ids, {3: 30, 9: None, 4: 40})
    assert keep.tolist() == [True, True, False, True, True]
    assert out[keep].tolist() == [5, 30, 7, 1]


def test_merge_restatement_and_unchanged_rule():
    offs = np.array([0, 3, 5, 5, 8], np.uint64)          # partitions of 3, 2, 0 and 3 rows
    rows = dict(row_ids=np.arange(8, dtype=np.uint64) * 10)
    add = dict(row_ids=np.array([100, 101], np.uint64))
    # join: old 2 (empty) dropped, old 3 -> 2; remove row 10 (partition 0); add two rows to partition 1
    pm = np.array([0, 1, DROP, 2], np.uint32)
    new_offs, out, src = merge(offs, rows, pm, [10], [1, 1], add, 3)
    assert new_offs.tolist() == [0, 2, 6, 9]
    assert out["row_ids"].tolist() == [0, 20, 30, 40, 100, 101, 50, 60, 70]
    assert src.tolist() == [-1, -1, 3]                     # only the moved, untouched partition keeps its graph
    # a remap that only rewrites ids keeps every graph; one that drops a row of partition 1 rebuilds it alone
    _, out, src = merge(offs, rows, None, [], [], dict(row_ids=np.zeros(0, np.uint64)), 4, {0: 7, 60: 61})
    assert src.tolist() == [0, 1, -1, 3] and out["row_ids"].tolist() == [7, 10, 20, 30, 40, 50, 61, 70]
    _, out, src = merge(offs, rows, None, [], [], dict(row_ids=np.zeros(0, np.uint64)), 4, {40: None})
    assert src.tolist() == [0, -1, -1, 3] and 40 not in out["row_ids"].tolist()
    # two old partitions into one new: only an empty partner leaves the other's graph in place
    pm = np.array([0, 0, 1, 1], np.uint32)
    _, _, src = merge(offs, rows, pm, [], [], dict(row_ids=np.zeros(0, np.uint64)), 2)
    assert src.tolist() == [-1, 3]


# ---- indexes of every kind -------------------------------------------------------------------------------------------
KINDS = ["pq", "flat", "sq", "rq", "hnsw_sq", "hnsw_pq", "hnsw_flat"]
GRAPH = {"hnsw_sq", "hnsw_pq", "hnsw_flat"}


def _data(n, d, seed, k=6):
    rng = np.random.default_rng(seed)
    c = rng.normal(0, 3, (k, d)).astype(np.float32)
    return (c[rng.integers(0, k, n)] + rng.normal(0, 1, (n, d))).astype(np.float32)


def _typed(x, dt):
    if dt == "f16":
        return x.astype(np.float16), {}
    if dt == "u8":
        return np.clip(x * 20 + 128, 0, 255).astype(np.uint8), {}
    return x, {}


def _build(kind, x, metric, K=6, seed=5, row_ids=None, dt="f32"):
    x, kw = _typed(x, dt)
    rid = np.arange(len(x), dtype=np.uint64) if row_ids is None else row_ids
    hp = lb.HnswBuildParams(**HNSW)
    pq = lb.IvfBuildParams(num_partitions=K, num_sub_vectors=4, max_iters=8, pq_max_iters=4, seed=seed)
    if kind == "pq":
        return lb.IvfPqIndex.build(x, metric, pq, row_ids=rid)
    if kind == "hnsw_pq":
        return lb.IvfHnswPqIndex.build(x, metric, pq, hp, row_ids=rid)
    args = dict(num_partitions=K, max_iters=8, seed=seed, row_ids=rid, **kw)
    return {"flat": lambda: lb.IvfFlatIndex.build(x, metric, **args),
            "sq": lambda: lb.IvfSqIndex.build(x, metric, **args),
            "rq": lambda: lb.IvfRqIndex.build(x, metric, **args),
            "hnsw_sq": lambda: lb.IvfHnswSqIndex.build(x, metric, hnsw_params=hp, **args),
            "hnsw_flat": lambda: lb.IvfHnswFlatIndex.build(x, metric, hnsw_params=hp, **args)}[kind]()


def _payload_key(kind):
    return "vectors" if kind.endswith("flat") else "codes"


def _rows(kind, e):
    """the per-row arrays of an export, in storage order"""
    r = dict(row_ids=e["row_ids"], payload=e[_payload_key(kind)])
    if kind == "rq":
        r["add"], r["scale"] = e["add_factors"], e["scale_factors"]
    return r


def _t_rows(kind, t, row_ids):
    ok = t["valid"]
    r = dict(row_ids=np.asarray(row_ids, np.uint64)[ok], payload=t["payload"][ok])
    if kind == "rq":
        r["add"], r["scale"] = t["add_factors"][ok], t["scale_factors"][ok]
    return r, t["part_ids"][ok]


def _graph_of(kind, e, metric, seed, dt="f32"):
    """the restatement's graph over an export's storage (dt: the column's element type)"""
    kw = dict(m=HNSW["m"], max_level=HNSW["max_level"], efc=HNSW["ef_construction"], seed=seed)
    if kind == "hnsw_sq":
        return hr.build(e["codes"], e["part_offsets"], e["bounds"], "dot" if metric == "dot" else "l2", **kw)
    if kind == "hnsw_pq":
        return pr.build(e["codes"], e["part_offsets"], e["codebook"], 8, metric, dt, **kw)
    return hf.build(e["vectors"], e["part_offsets"], metric, dt, **kw)


def _assert_graph_equal(a, b):
    for k in ("max_level", "m", "ef_construction"):
        assert a[k] == b[k], k
    for k in ("levels", "counts0", "neighbors0", "dists0", "counts_up", "neighbors_up", "dists_up"):
        assert np.array_equal(np.asarray(a[k]).view(np.uint8), np.asarray(b[k]).view(np.uint8)), k


def _check_merge(kind, old, new, old_e, offs, rows, src, metric, seed, dt="f32"):
    """new's export against the restated storage (and graphs)"""
    e = new.export()
    assert np.array_equal(e["part_offsets"], offs)
    assert np.array_equal(e["row_ids"], rows["row_ids"])
    assert np.array_equal(np.asarray(e[_payload_key(kind)]).view(np.uint8), np.asarray(rows["payload"]).view(np.uint8))
    if kind == "rq":
        assert np.array_equal(e["add_factors"].view(np.uint32), rows["add"].view(np.uint32))
        assert np.array_equal(e["scale_factors"].view(np.uint32), rows["scale"].view(np.uint32))
    if kind in GRAPH:
        want = assemble(offs, src, _graph_of(kind, e, metric, seed, dt), old_e["graph"], old_e["part_offsets"])
        _assert_graph_equal(e["graph"], want)
    return e


def _from_parts(kind, e, metric):
    """an index opened from an export (graph included): the same storage loaded from scratch"""
    sizes = np.diff(e["part_offsets"]).astype(np.int64)
    part = np.repeat(np.arange(len(sizes), dtype=np.uint32), sizes)
    if kind == "pq":
        return lb.IvfPqIndex.from_parts(e["centroids"], e["codebook"], part, e["codes"], e["row_ids"], metric)
    if kind == "hnsw_pq":
        return lb.IvfHnswPqIndex.from_parts(e["centroids"], e["codebook"], part, e["codes"], e["row_ids"], metric,
                                            graph=e["graph"])
    if kind in ("flat", "hnsw_flat"):
        cls = lb.IvfFlatIndex if kind == "flat" else lb.IvfHnswFlatIndex
        extra = dict(graph=e["graph"]) if kind in GRAPH else {}
        return cls.from_parts(e["centroids"], part, e["vectors"], e["row_ids"], metric, **extra)
    if kind in ("sq", "hnsw_sq"):
        cls = lb.IvfSqIndex if kind == "sq" else lb.IvfHnswSqIndex
        extra = dict(graph=e["graph"]) if kind in GRAPH else {}
        return cls.from_parts(e["centroids"], e["bounds"], part, e["codes"], e["row_ids"], metric, **extra)
    return lb.IvfRqIndex.from_parts(e["centroids"], e["rotation"], part, e["codes"], e["add_factors"],
                                    e["scale_factors"], e["row_ids"], metric)


def _same_search(a, b, q, nprobes=3):
    for x, y in ((a.search(q, k=10, nprobes=nprobes), b.search(q, k=10, nprobes=nprobes)),):
        assert np.array_equal(x[0], y[0]) and np.array_equal(x[1].view(np.uint32), y[1].view(np.uint32))
    n = a.info()["num_rows"]
    allow = np.flatnonzero(np.arange(n) % 3 != 0)
    bm_a = a.row_mask(allow_row_ids=a.export()["row_ids"][allow])
    bm_b = b.row_mask(allow_row_ids=b.export()["row_ids"][allow])
    x, y = a.search_ex(q, k=10, nprobes=nprobes, allow_bitmap=bm_a), b.search_ex(q, k=10, nprobes=nprobes, allow_bitmap=bm_b)
    assert np.array_equal(x[0], y[0]) and np.array_equal(x[1].view(np.uint32), y[1].view(np.uint32))
    x, y = a.search_probed(q, 10, minimum_nprobes=2), b.search_probed(q, 10, minimum_nprobes=2)
    assert all(np.array_equal(np.asarray(u).view(np.uint8), np.asarray(v).view(np.uint8)) for u, v in zip(x, y))


# ---- 1. transform ----------------------------------------------------------------------------------------------------
TRANSFORM_CASES = [(k, m, "f32") for k in ("pq", "flat", "sq", "rq", "hnsw_sq") for m in ("l2", "cosine", "dot")] + \
    [("flat", "l2", "u8"), ("flat", "cosine", "f16"), ("sq", "dot", "u8"), ("sq", "cosine", "f16"),
     ("hnsw_flat", "cosine", "f32"), ("hnsw_pq", "l2", "f32")]


@pytest.mark.gpu
@pytest.mark.parametrize("kind,metric,dt", TRANSFORM_CASES)
def test_transform_equals_the_build_storage(kind, metric, dt):
    x = _data(900, 16, seed=11)
    x[7] = np.nan if dt != "u8" else x[7]                  # a row every build drops
    ix = _build(kind, x, metric, dt=dt)
    e = ix.export()
    t = ix.transform(_typed(x, dt)[0])
    ok = t["valid"]
    assert ok.sum() == ix.info()["num_rows"]
    rid = e["row_ids"].astype(np.int64)
    assert ok[rid].all()
    part = np.repeat(np.arange(len(e["part_offsets"]) - 1), np.diff(e["part_offsets"]).astype(np.int64))
    assert np.array_equal(t["part_ids"][rid], part)
    assert np.array_equal(np.asarray(t["payload"][rid]).view(np.uint8), np.asarray(e[_payload_key(kind)]).view(np.uint8))
    if kind == "pq":
        p, c, v = lb.ivfpq_transform(e["centroids"], e["codebook"], x, metric)
        assert np.array_equal(v, ok) and np.array_equal(p[v], t["part_ids"][ok]) and np.array_equal(c[v], t["payload"][ok])
    if kind == "rq":
        assert np.array_equal(t["add_factors"][rid].view(np.uint32), e["add_factors"].view(np.uint32))
        r = lb.RabitQuantizer(16, 1, e["rotation"]).transform(e["centroids"], x, metric)
        assert np.array_equal(r["valid"], ok)
        for a, b in (("part_ids", "part_ids"), ("codes", "payload"), ("add_factors", "add_factors"),
                     ("scale_factors", "scale_factors")):
            assert np.array_equal(np.asarray(r[a])[ok].view(np.uint8), np.asarray(t[b])[ok].view(np.uint8)), a


# ---- 2. append -------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_append_equals_the_concatenated_storage(kind):
    metric = "cosine" if kind in ("flat", "hnsw_pq") else "l2"
    x = _data(1200, 16, seed=21)
    ix = _build(kind, x[:800], metric)
    old = ix.export()
    y_ids = np.arange(800, 1200, dtype=np.uint64) + np.uint64(5000)
    new = ix.optimize(add_vectors=x[800:], add_row_ids=y_ids, seed=77)
    add, add_part = _t_rows(kind, ix.transform(x[800:]), y_ids)
    offs, rows, src = merge(old["part_offsets"], _rows(kind, old), None, [], add_part, add, ix.info()["num_partitions"])
    e = _check_merge(kind, ix, new, old, offs, rows, src, metric, 77)
    _same_search(new, _from_parts(kind, e, metric), x[:16] + np.float32(0.1))


# ---- 3. remove, join and new centroids -------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["pq", "flat", "sq", "rq", "hnsw_sq"])
def test_remove_join_and_new_centroids(kind):
    metric = "l2"
    rng = np.random.default_rng(31)
    x = _data(1500, 16, seed=31)
    K = 6
    ix = _build(kind, x, metric, K=K, row_ids=np.arange(1500, dtype=np.uint64) * 2)
    old = ix.export()
    old_rows = _rows(kind, old)
    removed = rng.choice(old["row_ids"], 150, replace=False)
    pm = np.arange(K, dtype=np.uint32)
    pm[3] = DROP
    pm[4:] -= 1
    cent2 = np.delete(old["centroids"], 3, axis=0)
    a, b = int(old["part_offsets"][3]), int(old["part_offsets"][4])
    moved = {k: v[a:b] for k, v in old_rows.items()}       # the joined partition's rows re-enter via the add list
    moved["row_ids"] = moved["row_ids"] + np.uint64(1)
    mp = rng.integers(0, K - 1, b - a).astype(np.uint32)
    factors = (moved["add"], moved["scale"]) if kind == "rq" else None
    new = ix.optimize(new_centroids=cent2, part_map=pm, remove_row_ids=removed, add_part_ids=mp,
                      add_payload=moved["payload"], add_factors=factors, add_row_ids=moved["row_ids"], seed=9)
    assert new.info()["num_partitions"] == K - 1
    offs, rows, src = merge(old["part_offsets"], old_rows, pm, removed, mp, moved, K - 1)
    e = _check_merge(kind, ix, new, old, offs, rows, src, metric, 9)
    assert np.array_equal(e["centroids"], cent2)
    _same_search(new, _from_parts(kind, e, metric), x[:16] + np.float32(0.05))
    if kind == "pq":   # lb2_index_update gives the same bytes
        up = ix.update(new_centroids=cent2, part_map=pm, remove_row_ids=removed, add_part_ids=mp,
                       add_codes=moved["payload"], add_row_ids=moved["row_ids"])
        u = up.export()
        for key in u:
            assert np.array_equal(u[key], e[key]), key


# ---- 4. remap --------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["pq", "flat", "rq", "hnsw_flat"])
def test_remap_keeps_order_and_rewrites_ids(kind):
    rng = np.random.default_rng(41)
    x = _data(1000, 16, seed=41)
    ix = _build(kind, x[:800], "l2")
    old = ix.export()
    ids = old["row_ids"]
    pick = rng.permutation(len(ids))
    mapping = {int(i): int(i) + 100000 for i in ids[pick[:200]]}
    mapping.update({int(i): None for i in ids[pick[200:260]]})
    mapping.update({100000000 + j: 5 for j in range(10)})   # ids that are not in the index
    mapping[900] = 7000                                     # an added row is remapped too
    y_ids = np.arange(800, 1000, dtype=np.uint64)
    new = ix.optimize(add_vectors=x[800:], add_row_ids=y_ids, remap=mapping, seed=3)
    add, add_part = _t_rows(kind, ix.transform(x[800:]), y_ids)
    offs, rows, src = merge(old["part_offsets"], _rows(kind, old), None, [], add_part, add, 6, mapping)
    e = _check_merge(kind, ix, new, old, offs, rows, src, "l2", 3)
    q = x[:16] + np.float32(0.05)
    got = new.search(q, k=10, nprobes=6)
    want = _from_parts(kind, e, "l2").search(q, k=10, nprobes=6)
    assert np.array_equal(got[0], want[0])
    assert not np.isin(got[0], [int(i) for i, v in mapping.items() if v is None]).any()
    # the same mapping as two arrays
    o = np.array(sorted(mapping), np.uint64)
    nw = np.array([NONE if mapping[int(i)] is None else mapping[int(i)] for i in o], np.uint64)
    e2 = ix.optimize(add_vectors=x[800:], add_row_ids=y_ids, remap=(o, nw), seed=3).export()
    assert np.array_equal(e2["row_ids"], e["row_ids"])
    for bad in ((o[::-1].copy(), nw[::-1].copy()), (np.array([3, 3], np.uint64), np.array([1, 2], np.uint64))):
        with pytest.raises(lb.LanceB200Error) as err:
            ix.optimize(remap=bad)
        assert err.value.status == lb._lib.INVALID_ARG


# ---- 5. graphs: only the changed partitions are rebuilt --------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["hnsw_sq", "hnsw_pq", "hnsw_flat"])
def test_only_changed_partitions_are_rebuilt(kind):
    metric = "l2"
    x = _data(1400, 16, seed=51)
    K = 6
    ix = _build(kind, x[:1000], metric, K=K, seed=5)
    old = ix.export()
    old_rows = _rows(kind, old)
    t = ix.transform(x[1000:])
    ok = t["valid"] & np.isin(t["part_ids"], [1, 4])        # adds to partitions 1 and 4 only
    y_ids = np.arange(1000, 1400, dtype=np.uint64)
    add = dict(row_ids=y_ids[ok], payload=t["payload"][ok])
    new = ix.optimize(add_part_ids=t["part_ids"][ok], add_payload=add["payload"], add_row_ids=add["row_ids"], seed=99)
    offs, rows, src = merge(old["part_offsets"], old_rows, None, [], t["part_ids"][ok], add, K)
    assert sorted(np.flatnonzero(src < 0).tolist()) == [1, 4]
    _check_merge(kind, ix, new, old, offs, rows, src, metric, 99)
    # a join: partition 2 dropped, its rows re-enter partition 0; partitions 3.. move down one id and keep their graphs
    pm = np.arange(K, dtype=np.uint32)
    pm[2] = DROP
    pm[3:] -= 1
    a, b = int(old["part_offsets"][2]), int(old["part_offsets"][3])
    moved = {k: v[a:b] for k, v in old_rows.items()}
    mp = np.zeros(b - a, np.uint32)
    cent2 = np.delete(old["centroids"], 2, axis=0)
    j = ix.optimize(new_centroids=cent2, part_map=pm, add_part_ids=mp, add_payload=moved["payload"],
                    add_row_ids=moved["row_ids"], seed=99)
    offs, rows, src = merge(old["part_offsets"], old_rows, pm, [], mp, moved, K - 1)
    assert src.tolist() == [-1, 1, 3, 4, 5]
    _check_merge(kind, ix, j, old, offs, rows, src, metric, 99)
    # a graph loaded with from_parts (no seed): a remap that only rewrites ids gives it back unchanged
    g = _graph_of(kind, old, metric, 1234)
    lo = _from_parts(kind, dict(old, graph=g), metric)
    ids = old["row_ids"]
    srt = np.sort(ids)
    r = lo.optimize(remap=(srt, srt + np.uint64(10 ** 6)), seed=7).export()
    _assert_graph_equal(r["graph"], g)
    assert np.array_equal(r["row_ids"], ids + np.uint64(10 ** 6))
    # drop one row of partition p: only p changes
    p = 3
    one = int(ids[int(old["part_offsets"][p]) + 2])
    d1 = lo.optimize(remove_row_ids=[one], seed=7)
    offs, rows, src = merge(old["part_offsets"], old_rows, None, [one], [], {k: v[:0] for k, v in old_rows.items()}, K)
    assert np.flatnonzero(src < 0).tolist() == [p]
    _check_merge(kind, lo, d1, dict(old, graph=g), offs, rows, src, metric, 7)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["hnsw_sq", "hnsw_pq", "hnsw_flat"])
def test_graph_edge_cases(kind):
    metric = "l2"
    x = _data(900, 16, seed=61)
    K = 6
    ix = _build(kind, x[:700], metric, K=K, seed=5)
    old = ix.export()
    old_rows = _rows(kind, old)
    offs0 = old["part_offsets"].astype(np.int64)
    sizes = np.diff(offs0)
    empty = {k: v[:0] for k, v in old_rows.items()}
    ids = old["row_ids"]
    # partition 0 emptied, partition 1 left with one row
    gone = np.concatenate([ids[offs0[0]:offs0[1]], ids[offs0[1] + 1:offs0[2]]])
    e1 = ix.optimize(remove_row_ids=gone, seed=8)
    offs, rows, src = merge(old["part_offsets"], old_rows, None, gone, [], empty, K)
    assert np.diff(offs)[:2].tolist() == [0, 1]
    _check_merge(kind, ix, e1, old, offs, rows, src, metric, 8)
    # partition 5 grows past the old largest partition; then rows added to the emptied partition 0
    t = ix.transform(x[700:])
    ok = t["valid"]
    n_add = int(ok.sum())
    big = np.full(n_add, 5, np.uint32)
    add = dict(row_ids=np.arange(n_add, dtype=np.uint64) + np.uint64(9000), payload=t["payload"][ok])
    assert sizes[5] + n_add > sizes.max()
    e2 = ix.optimize(add_part_ids=big, add_payload=add["payload"], add_row_ids=add["row_ids"], seed=8)
    offs, rows, src = merge(old["part_offsets"], old_rows, None, [], big, add, K)
    _check_merge(kind, ix, e2, old, offs, rows, src, metric, 8)
    old1 = e1.export()
    zero = np.zeros(n_add, np.uint32)
    e3 = e1.optimize(add_part_ids=zero, add_payload=add["payload"], add_row_ids=add["row_ids"], seed=8)
    offs, rows, src = merge(old1["part_offsets"], _rows(kind, old1), None, [], zero, add, K)
    _check_merge(kind, e1, e3, old1, offs, rows, src, metric, 8)
    # an old index with no rows
    e0 = ix.optimize(remove_row_ids=ids, seed=8)
    assert e0.info()["num_rows"] == 0
    old0 = e0.export()
    e4 = e0.optimize(add_part_ids=t["part_ids"][ok], add_payload=add["payload"], add_row_ids=add["row_ids"], seed=8)
    offs, rows, src = merge(old0["part_offsets"], _rows(kind, old0), None, [], t["part_ids"][ok], add, K)
    _check_merge(kind, e0, e4, old0, offs, rows, src, metric, 8)


# ---- 6. refusals -----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_refusals():
    x = _data(600, 16, seed=71)
    rq = _build("rq", x, "l2")
    sq = _build("sq", x, "l2")
    t = rq.transform(x[:4])
    e = sq.transform(x[:4])
    K = rq.info()["num_partitions"]
    cases = [
        lambda: rq.optimize(add_part_ids=t["part_ids"], add_payload=t["payload"], add_row_ids=np.arange(4)),  # missing
        lambda: sq.optimize(add_part_ids=e["part_ids"], add_payload=e["payload"], add_row_ids=np.arange(4),
                            add_factors=(np.zeros(4), np.zeros(4))),                                           # extra
        lambda: sq.optimize(part_map=np.full(K, K, np.uint32)),                                                # part_map
        lambda: sq.optimize(add_part_ids=np.full(4, K, np.uint32), add_payload=e["payload"],
                            add_row_ids=np.arange(4)),                                                         # part ids
    ]
    for call in cases:
        with pytest.raises(lb.LanceB200Error) as err:
            call()
        assert err.value.status == lb._lib.INVALID_ARG
    p = lb._lib.OptimizeParams()
    p.new_k = K + 1                                                                                            # no centroids
    h = lb._lib.C.c_void_p()
    with pytest.raises(lb.LanceB200Error) as err:
        lb._lib.check(lb._lib.lib().lb2_index_optimize(sq._h, lb._lib.C.byref(p), lb._lib.C.byref(h)))
    assert err.value.status == lb._lib.INVALID_ARG
    with pytest.raises(lb.LanceB200Error) as err:
        lb._lib.check(lb._lib.lib().lb2_index_transform(sq._h, None, lb._lib.C.c_uint64(0), None, None,
                                                        lb._lib.C.c_void_p(1), None, None))
    assert err.value.status == lb._lib.INVALID_ARG
