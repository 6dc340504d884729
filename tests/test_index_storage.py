"""lb2_index_export_storage / lb2_index_load_storage: every index kind in the reference's storage layout, against the
restatements of pack_codes / unpack_codes and HNSW::to_batch / load in tests/storage_reference.py."""
import numpy as np
import pytest

import lance_b200 as lb
import storage_reference as sr

HNSW = lb.HnswBuildParams(max_level=4, m=6, ef_construction=24, insert_batch=8)
SIZES = [0, 1, 2, 31, 32, 33, 4200]


# ---- restatements (no GPU) --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [0, 1, 31, 32, 33, 64, 65, 1000])
def test_pack_unpack_round_trip(n):
    c = np.random.default_rng(n).integers(0, 256, (n, 5), dtype=np.uint8)
    p = sr.pack_codes(c)
    assert p.shape == c.shape
    assert np.array_equal(sr.unpack_codes(p), c)


def test_pack_one_block_by_hand():
    # one 32-row block of one byte per row: row r has low nibble r & 15 and high nibble r >> 1
    rows = np.arange(32)
    c = ((rows & 15) | ((rows >> 1) << 4)).astype(np.uint8).reshape(32, 1)
    perm0 = [0, 8, 1, 9, 2, 10, 3, 11, 4, 12, 5, 13, 6, 14, 7, 15]
    want = []
    for j in range(16):  # low nibbles of rows PERM0[j] (bits 0..3) and PERM0[j] + 16 (bits 4..7)
        a, b = perm0[j], perm0[j] + 16
        want.append((a & 15) | ((b & 15) << 4))
    for j in range(16):  # the high nibbles of the same rows
        a, b = perm0[j], perm0[j] + 16
        want.append((a >> 1) | ((b >> 1) << 4))
    assert sr.pack_codes(c).reshape(-1).tolist() == want


def _random_graph(sizes, L=3, m=3, seed=0):
    """a dense-layout graph with valid lists: node 0 of a partition has every level, others a random count"""
    rng = np.random.default_rng(seed)
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    n = int(off[-1])
    levels = np.ones(n, np.uint8)
    for p in range(len(sizes)):
        for i in range(sizes[p]):
            levels[off[p] + i] = L if i == 0 else rng.integers(1, L + 1)
    n_up = int(np.sum(levels.astype(np.int64) - 1))
    g = {"max_level": L, "m": m, "ef_construction": 10, "levels": levels, "counts0": np.zeros(n, np.uint32),
         "neighbors0": np.zeros((n, 2 * m), np.uint32), "dists0": np.zeros((n, 2 * m), np.float32),
         "counts_up": np.zeros(n_up, np.uint32), "neighbors_up": np.zeros((n_up, m), np.uint32),
         "dists_up": np.zeros((n_up, m), np.float32)}
    up = 0
    for p in range(len(sizes)):
        for i in range(sizes[p]):
            r = off[p] + i
            for level in range(int(levels[r])):
                cand = [j for j in range(sizes[p]) if j != i and levels[off[p] + j] > level]
                cap = 2 * m if level == 0 else m
                ids = rng.permutation(cand)[:rng.integers(0, min(cap, len(cand)) + 1)] if cand else []
                ds = rng.random(len(ids)).astype(np.float32)
                if level == 0:
                    g["counts0"][r] = len(ids)
                    g["neighbors0"][r, :len(ids)], g["dists0"][r, :len(ids)] = ids, ds
                else:
                    g["counts_up"][up] = len(ids)
                    g["neighbors_up"][up, :len(ids)], g["dists_up"][up, :len(ids)] = ids, ds
                    up += 1
    return g, off


@pytest.mark.parametrize("sizes", [[5, 0, 1, 7], [1], [0, 0], [3, 1, 1, 0, 9]])
def test_graph_batch_round_trip(sizes):
    g, off = _random_graph(sizes)
    s = sr.to_batch(g, off)
    assert int(s["level_offsets"][:, -1].sum()) == len(s["__vector_id"])
    back = sr.load(s, off)
    for k in ("levels", "counts0", "neighbors0", "dists0", "counts_up", "neighbors_up", "dists_up"):
        assert np.array_equal(back[k], g[k]), k


# ---- device -------------------------------------------------------------------------------------------------------
KINDS = ["pq", "flat", "sq", "rq", "hnsw_pq", "hnsw_flat", "hnsw_sq"]


def _clustered(sizes, d, seed=0):
    """rows in well separated clusters, one per partition, with the given sizes plus what optimize removes"""
    rng = np.random.default_rng(seed)
    centers = rng.normal(0, 50, (len(sizes), d)).astype(np.float32)
    parts = np.repeat(np.arange(len(sizes)), 40)
    return centers, (centers[parts] + rng.normal(0, 1, (len(parts), d))).astype(np.float32)


def _build(kind, data, K, metric, dtype, centroids=None, hnsw=HNSW):
    bf16 = dtype == "bf16"
    x = data
    if dtype == "f16":
        x = data.astype(np.float16)
    elif dtype == "u8":
        x = np.clip(np.rint(data + 128), 0, 255).astype(np.uint8)
    elif bf16:
        x = (data.view(np.uint32) >> 16).astype(np.uint16)
    common = dict(distance_type=metric, num_partitions=K, max_iters=10, sample_rate=1 << 20, centroids=centroids)
    if kind == "pq":
        return lb.IvfPqIndex.build(x, metric, lb.IvfBuildParams(num_partitions=K, num_sub_vectors=4, max_iters=10,
                                                                 pq_max_iters=4, sample_rate=1 << 20,
                                                                 centroids=centroids), bf16=bf16), x
    if kind == "hnsw_pq":
        return lb.IvfHnswPqIndex.build(x, metric, lb.IvfBuildParams(num_partitions=K, num_sub_vectors=4, max_iters=10,
                                                                     pq_max_iters=4, sample_rate=1 << 20,
                                                                     centroids=centroids),
                                       hnsw_params=hnsw, bf16=bf16), x
    if kind == "flat":
        return lb.IvfFlatIndex.build(x, bf16=bf16, **common), x
    if kind == "hnsw_flat":
        return lb.IvfHnswFlatIndex.build(x, bf16=bf16, hnsw_params=hnsw, **common), x
    if kind == "sq":
        return lb.IvfSqIndex.build(x, bf16=bf16, **common), x
    if kind == "hnsw_sq":
        return lb.IvfHnswSqIndex.build(x, bf16=bf16, hnsw_params=hnsw, **common), x
    return lb.IvfRqIndex.build(x, **common), x


def _reopen(kind, ix, st, metric, dtype):
    e = ix.export()
    bf16 = dtype == "bf16"
    npdt = {"f32": np.float32, "f16": np.float16, "bf16": np.float32, "u8": np.uint8}[dtype]
    if kind in ("pq", "hnsw_pq"):
        cls = lb.IvfPqIndex if kind == "pq" else lb.IvfHnswPqIndex
        nbits = 4 if e["codebook"].shape[1] == 16 else 8
        return cls.from_storage(e["centroids"], e["codebook"], st, metric, nbits, npdt, bf16)
    if kind in ("flat", "hnsw_flat"):
        cls = lb.IvfFlatIndex if kind == "flat" else lb.IvfHnswFlatIndex
        return cls.from_storage(e["centroids"], st, metric, npdt, bf16)
    if kind in ("sq", "hnsw_sq"):
        cls = lb.IvfSqIndex if kind == "sq" else lb.IvfHnswSqIndex
        return cls.from_storage(e["centroids"], e["bounds"], st, metric, npdt, bf16)
    return lb.IvfRqIndex.from_storage(e["centroids"], e["rotation"], st, metric)


def _searches(kind, ix, x, q, K):
    """every search path's results, for bit-level comparison"""
    out = []
    n = x.shape[0]
    allow = np.zeros((n + 63) // 64, np.uint64)
    allow[::2] = np.uint64(0xFFFFFFFFFFFFFFFF)
    out += list(ix.search(q, k=10, nprobes=3))
    # a range that cuts: bounds at the 10th and 50th percentiles of the index's own distances to these queries
    d0 = ix.search_ex(q, k=10, nprobes=K)[1]
    fin = d0[np.isfinite(d0)]
    lower, upper = float(np.quantile(fin, 0.1)), float(np.quantile(fin, 0.5))
    out += [np.float32(lower), np.float32(upper)]
    out += list(ix.search_ex(q, k=10, nprobes=K, allow_bitmap=allow, lower_bound=lower, upper_bound=upper))
    out += list(ix.search_ex(q, k=10, nprobes=K, lower_bound=lower, upper_bound=upper))
    out += list(ix.search_probed(q, 10, minimum_nprobes=1, maximum_nprobes=K))
    out += list(ix.search_refine(x, q, k=5, nprobes=2, refine_factor=2))
    if kind.startswith("hnsw"):
        out += list(ix.search(q, k=10, nprobes=K, ef=40))
    return out


def _same(a, b):
    assert len(a) == len(b)
    for u, v in zip(a, b):
        assert np.array_equal(np.atleast_1d(u).view(np.uint8), np.atleast_1d(v).view(np.uint8))


def _sized(kind, metric="l2", dtype="f32", d=32, hnsw=HNSW):
    """an index whose partitions hold SIZES rows: a build over clusters, then optimize removes the extra rows"""
    K = len(SIZES)
    rng = np.random.default_rng(1)
    centers = rng.normal(0, 40, (K, d)).astype(np.float32)
    counts = [s + 3 for s in SIZES]
    parts = np.repeat(np.arange(K), counts)
    data = (centers[parts] + rng.normal(0, 1, (len(parts), d))).astype(np.float32)
    ix, x = _build(kind, data, K, metric, dtype, centroids=centers, hnsw=hnsw)
    e = ix.export()
    off = e["part_offsets"].astype(np.int64)
    have = np.diff(off)
    want = sorted(SIZES)
    order = np.argsort(have, kind="stable")
    remove = []
    for p, s in zip(order, want):
        remove.extend(e["row_ids"][off[p] + s:off[p + 1]].tolist())
    if remove:
        ix = ix.optimize(remove_row_ids=np.array(sorted(remove), np.uint64))
    assert sorted(np.diff(ix.export()["part_offsets"].astype(np.int64)).tolist()) == want
    return ix, x, K


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_round_trip_partition_sizes(kind):
    ix, x, K = _sized(kind)
    st = ix.export_storage()
    assert np.array_equal(st["part_lengths"], np.diff(ix.export()["part_offsets"]))
    back = _reopen(kind, ix, st, "l2", "f32")
    q = x[::97][:16]
    _same(_searches(kind, ix, x, q, K), _searches(kind, back, x, q, K))
    st2 = back.export_storage()
    for k in st:
        assert np.array_equal(np.asarray(st[k]), np.asarray(st2[k])), k


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("metric", ["l2", "cosine", "dot"])
@pytest.mark.parametrize("dtype", ["f32", "f16", "bf16", "u8"])
def test_round_trip_types_and_metrics(kind, metric, dtype):
    if kind == "rq" and dtype != "f32":
        pytest.skip("IVF_RQ takes f32 columns only")
    if kind in ("flat", "hnsw_flat") and dtype == "u8":
        pytest.skip("u8 IVF_FLAT has no storage layout (test_u8_flat_has_no_storage)")
    centers, data = _clustered([0] * 6, 32, seed=3)
    rng = np.random.default_rng(4)
    data = np.concatenate([data, (centers[rng.integers(0, 6, 2000)] + rng.normal(0, 4, (2000, 32)))]).astype(np.float32)
    ix, x = _build(kind, data, 6, metric, dtype)
    st = ix.export_storage()
    back = _reopen(kind, ix, st, metric, dtype)
    q = x[::131][:12]
    _same(_searches(kind, ix, x, q, 6), _searches(kind, back, x, q, 6))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["hnsw_pq", "hnsw_flat", "hnsw_sq"])
def test_one_level_graphs(kind):
    # max_level 1: one level batch per partition; the 4200-row partition spans several 1024-node tiles of the export
    ix, x, K = _sized(kind, hnsw=lb.HnswBuildParams(max_level=1, m=6, ef_construction=24, insert_batch=8))
    e = ix.export()
    st = ix.export_storage()
    assert st["max_level"] == 1 and st["level_offsets"].shape == (K, 2)
    want = sr.to_batch(e["graph"], e["part_offsets"])
    for k in want:
        assert np.array_equal(np.asarray(st[k]), np.asarray(want[k])), k
    back = _reopen(kind, ix, st, "l2", "f32")
    q = x[::97][:16]
    _same(_searches(kind, ix, x, q, K), _searches(kind, back, x, q, K))
    gb = back.export()["graph"]
    for k in ("levels", "counts0", "neighbors0", "dists0"):
        assert np.array_equal(gb[k], e["graph"][k]), k


def test_storage_class_must_match_graph_columns():
    graph = {"part_lengths": np.zeros(1, np.uint64), "level_offsets": np.zeros((1, 2), np.uint64)}
    plain = {"part_lengths": np.zeros(1, np.uint64)}
    c = np.zeros((1, 8), np.float32)
    with pytest.raises(ValueError):
        lb.IvfSqIndex.from_storage(c, (0.0, 1.0), graph)
    with pytest.raises(ValueError):
        lb.IvfHnswSqIndex.from_storage(c, (0.0, 1.0), plain)
    with pytest.raises(ValueError):
        lb.IvfHnswFlatIndex.from_storage(c, plain)
    with pytest.raises(ValueError):
        lb.IvfPqIndex.from_storage(c, np.zeros((4, 256, 2), np.float32), graph)


@pytest.mark.gpu
def test_rq_packed_bytes_match_oracle():
    ix, x, K = _sized("rq")
    e = ix.export()
    st = ix.export_storage()
    assert np.array_equal(st["__rabit_code"], sr.pack_partitions(e["codes"], e["part_offsets"]))
    assert np.array_equal(st["_rowid"], e["row_ids"])
    assert np.array_equal(st["__add_factors"], e["add_factors"])


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["hnsw_pq", "hnsw_flat", "hnsw_sq"])
def test_graph_batches_match_oracle(kind):
    ix, x, K = _sized(kind)
    e = ix.export()
    st = ix.export_storage()
    want = sr.to_batch(e["graph"], e["part_offsets"])
    for k in want:
        assert np.array_equal(np.asarray(st[k]), np.asarray(want[k])), k


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["pq", "hnsw_pq"])
def test_pq_storage_equals_export_partition(kind):
    ix, x, K = _sized(kind)
    st = ix.export_storage()
    off = np.concatenate([[0], np.cumsum(st["part_lengths"].astype(np.int64))])
    flat = st["__pq_code"].reshape(-1)
    cw = st["__pq_code"].shape[1]
    for p in range(K):
        codes_t, rid = ix.export_partition_transposed(p)
        assert np.array_equal(flat[off[p] * cw:off[p + 1] * cw], codes_t.reshape(-1))
        assert np.array_equal(st["_rowid"][off[p]:off[p + 1]], rid)


@pytest.mark.gpu
def test_rq_load_matches_unpacked_load():
    ix, x, K = _sized("rq")
    e = ix.export()
    st = {"part_lengths": np.diff(e["part_offsets"]), "_rowid": e["row_ids"],
          "__rabit_code": sr.pack_partitions(e["codes"], e["part_offsets"]),
          "__add_factors": e["add_factors"], "__scale_factors": e["scale_factors"]}
    a = lb.IvfRqIndex.from_storage(e["centroids"], e["rotation"], st)
    part = np.repeat(np.arange(K, dtype=np.uint32), np.diff(e["part_offsets"]).astype(np.int64))
    b = lb.IvfRqIndex.from_parts(e["centroids"], e["rotation"], part, e["codes"], e["add_factors"],
                                 e["scale_factors"], e["row_ids"])
    ea, eb = a.export(), b.export()
    for k in ea:
        assert np.array_equal(ea[k], eb[k]), k
    q = x[::53][:16]
    _same(_searches("rq", a, x, q, K), _searches("rq", b, x, q, K))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["hnsw_pq", "hnsw_flat", "hnsw_sq"])
def test_graph_load_matches_dense_load(kind):
    ix, x, K = _sized(kind)
    e = ix.export()
    st = ix.export_storage()
    st.update(sr.to_batch(e["graph"], e["part_offsets"]))  # the restated batches, not the device's
    a = _reopen(kind, ix, st, "l2", "f32")
    ga = a.export()["graph"]
    dense = sr.load(st, e["part_offsets"])
    for k in ("levels", "counts0", "neighbors0", "dists0", "counts_up", "neighbors_up", "dists_up"):
        assert np.array_equal(ga[k], dense[k]), k
        assert np.array_equal(ga[k], e["graph"][k]), k
    q = x[::61][:16]
    _same(_searches(kind, ix, x, q, K), _searches(kind, a, x, q, K))


def _first(r):
    return r[0] if isinstance(r, tuple) else r


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_round_trip_after_split_and_join(kind):
    ix, x, K = _sized(kind)
    e = ix.export()
    off = e["part_offsets"].astype(np.int64)
    big = int(np.argmax(np.diff(off)))
    rid = np.sort(e["row_ids"][off[big]:off[big + 1]])
    ix2 = _first(ix.split(big, x[rid.astype(np.int64)], rid))
    e2 = ix2.export()
    off2 = e2["part_offsets"].astype(np.int64)
    small = int(np.argmin(np.where(np.diff(off2) > 0, np.diff(off2), 1 << 30)))
    rid2 = np.sort(e2["row_ids"][off2[small]:off2[small + 1]])
    ix3 = _first(ix2.join(small, x[rid2.astype(np.int64)], rid2))
    for cur in (ix2, ix3):
        k = cur.info()["num_partitions"]
        back = _reopen(kind, cur, cur.export_storage(), "l2", "f32")
        q = x[::89][:16]
        _same(_searches(kind, cur, x, q, k), _searches(kind, back, x, q, k))


def _expect_refusal(ix, kind, st, x, K, before):
    with pytest.raises(lb.LanceB200Error) as err:
        ix._load_storage(st)
    assert err.value.status == 1, str(err.value)
    q = x[::97][:8]
    _same(before, _searches(kind, ix, x, q, K))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["rq", "hnsw_sq"])
def test_refusals_leave_the_index(kind):
    ix, x, K = _sized(kind)
    good = ix.export_storage()
    q = x[::97][:8]
    before = _searches(kind, ix, x, q, K)

    def bad(**over):
        s = {k: (np.array(v, copy=True) if isinstance(v, np.ndarray) else v) for k, v in good.items()}
        for k, v in over.items():
            s[k] = v(s) if callable(v) else v
        _expect_refusal(ix, kind, s, x, K, before)

    lens = good["part_lengths"].copy()
    lens[0] += 1
    bad(part_lengths=lens)
    wrap = good["part_lengths"].copy()  # two lengths above num_rows that sum to num_rows modulo 2^64
    wrap[:2] += np.uint64(1 << 63)
    bad(part_lengths=wrap)
    code = good["__rabit_code"] if kind == "rq" else good["__sq_code"]
    bad(**{("__rabit_code" if kind == "rq" else "__sq_code"): code[:-1]})
    if kind != "hnsw_sq":
        return
    lo = good["level_offsets"]
    L = int(good["max_level"])
    big = int(np.argmax(good["part_lengths"]))
    base = int(np.concatenate([[0], np.cumsum(lo[:, L].astype(np.int64))])[big])

    def with_(key, f):
        def g(s):
            a = np.array(s[key], copy=True)
            f(a)
            return a
        return g

    def swap_ids(a):  # not ascending within level 0
        a[base + 1], a[base + 2] = a[base + 2], a[base + 1]
    bad(__vector_id=with_("__vector_id", swap_ids))

    def id_too_big(a):
        a[base + 1] = good["part_lengths"][big]
    bad(__vector_id=with_("__vector_id", id_too_big))

    def offsets_descend(a):
        a[base + 3] = a[base + 2] - 1 if a[base + 2] else a[base + 4] + 1
    bad(list_offsets=with_("list_offsets", offsets_descend))

    def wrong_end(a):
        a[-1] += 1
    bad(list_offsets=with_("list_offsets", wrong_end))

    def level_offsets_off(a):
        a[big, L] += 1
    bad(level_offsets=with_("level_offsets", level_offsets_off))

    def level_count_above_rows(a):  # level 1 claims more rows than the partition has, and every later level too
        a[big, 2:] += np.uint64(1 << 62)
    bad(level_offsets=with_("level_offsets", level_count_above_rows))

    def entry_one(a):
        a[big] = 1
    bad(entry_point=with_("entry_point", entry_one))

    def degree(s):
        lof = np.array(s["list_offsets"], np.int64)
        nb, ds = list(s["__neighbors"]), list(s["_distance"])
        gr = base  # node 0's level-0 list takes 2m + 1 entries (ids repeat: the degree check comes first)
        extra = 2 * int(good["m"]) + 1 - (lof[gr + 1] - lof[gr])
        nb[lof[gr + 1]:lof[gr + 1]] = [1] * extra
        ds[lof[gr + 1]:lof[gr + 1]] = [0.0] * extra
        lof[gr + 1:] += extra
        s["list_offsets"] = lof.astype(np.uint64)
        s["_distance"] = np.array(ds, np.float32)
        return np.array(nb, np.uint32)
    bad(__neighbors=degree)

    def neighbour_not_at_level(s):
        # a level-1 list of partition `big` naming a node that lacks level 1
        a = np.array(s["__neighbors"], copy=True)
        lof = s["list_offsets"].astype(np.int64)
        l1 = base + int(lo[big, 1])
        ids1 = set(s["__vector_id"][l1:base + int(lo[big, 2])].tolist())
        lacking = next(i for i in range(int(good["part_lengths"][big])) if i not in ids1)
        gr = next(g for g in range(l1, base + int(lo[big, 2])) if lof[g + 1] > lof[g])
        a[lof[gr]] = lacking
        return a
    bad(__neighbors=neighbour_not_at_level)

    def gap(s):
        # node v present at level 2 but not at level 1: rename level 2's last node to a node only at level 0
        a = np.array(s["__vector_id"], copy=True)
        l1, l2, l3 = (base + int(lo[big, i]) for i in (1, 2, 3))
        ids1 = set(a[l1:l2].tolist())
        cand = [i for i in range(int(a[l3 - 1]) + 1, int(good["part_lengths"][big])) if i not in ids1]
        a[l3 - 1] = cand[0]
        return a
    if int(lo[big, 3]) > int(lo[big, 2]):
        bad(__vector_id=gap)


@pytest.mark.gpu
def test_u8_flat_has_no_storage():
    data = np.random.default_rng(0).integers(0, 255, (500, 16)).astype(np.uint8)
    ix = lb.IvfFlatIndex.build(data, "l2", num_partitions=4, max_iters=4)
    with pytest.raises(lb.LanceB200Error) as err:
        ix.export_storage()
    assert err.value.status == 1
