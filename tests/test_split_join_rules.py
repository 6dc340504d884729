"""The split and join decisions of lb2_index_split / lb2_index_join where the per-type distance rules can be told apart:
dimension tails (d % 16 and d % 32 non-zero), every element type and metric, the streamed centroid table down to its
smallest chunk, a resident grid that sweeps its rows several times, and the candidate-ranking and row-set edges.

The expected decisions always come from the oracle's per-pair distances (tests/split_join_reference.py).  The numpy
rules of split_join_reference (LANES16, DOT32 and wrong variants of them) only prove that a case discriminates: every
case built to pin a rule asserts that the wrong rules change at least one of its decisions."""
import math

import numpy as np
import pytest

import lance_b200 as lb
import split_join_reference as sj
import test_index_optimize as tio
import test_partition_split_join as psj

STAYS = sj.STAYS
DIMS = [12, 20, 36, 44, 100]   # IVF_FLAT takes multiples of 4: below 16, and tails of 4 and 12
DTYPES = ["f32", "f16", "bf16"]


def _native(x, dt):
    """f32 values (exact in dt) -> the column as the index reads it (bf16: uint16 bit patterns)"""
    return psj._raw(np.asarray(x, np.float32), dt)


def _oracle_pairs(metric, dt):
    """the oracle's dist(from, to) on native values"""
    return psj._dist(metric, dt)


# ---- 1. the numpy rules against the oracle (CPU) --------------------------------------------------------------------
def _rows_with_big_terms(rng, n, d, dt):
    x = rng.standard_normal((n, d)).astype(np.float32) * np.float32(0.3)
    x[:, [0, d - 1]] += np.float32(1000.0)
    return psj._round(x, dt)


@pytest.mark.parametrize("d", DIMS + [3, 4, 8, 16, 17, 33, 1024, 1536, 4604])
@pytest.mark.parametrize("dt", DTYPES)
def test_rules_equal_the_oracle_bit_for_bit(d, dt):
    rng = np.random.default_rng(d)
    x, y = _rows_with_big_terms(rng, 40, d, dt), _rows_with_big_terms(rng, 40, d, dt)
    for metric in ("l2", "dot"):
        rule = sj.batch_rule(metric, dt)
        got = rule(x, y, metric)
        f = _oracle_pairs(metric, dt)
        want = np.array([f(_native(a, dt), _native(b, dt)) for a, b in zip(x, y)], np.float32)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (metric, dt, d)
    if dt != "f32":   # the other 32-lane rule of the oracle: f32 dot has 16 lanes, 16-bit dot 32
        assert sj.batch_rule("dot", dt) is sj.dot32 and sj.batch_rule("dot", "f32") is sj.lanes16


def _differ(a, b, x, y, metric):
    return int((a(x, y, metric).view(np.uint32) != b(x, y, metric).view(np.uint32)).sum())


def test_which_dimensions_tell_the_rules_apart():
    """LANES16, DOT32, the tail walked into the lanes and DOT32 folded upper half first agree wherever their partial
    sums coincide (d = 4, 8, 16; every rule below 16; LANES16 and DOT32 at 17), and differ at the tails this file
    uses"""
    rng = np.random.default_rng(1)
    for d in (3, 4, 8, 12, 16, 17, 20, 33, 36, 44, 47, 100, 1024):
        x, y = _rows_with_big_terms(rng, 300, d, "f32"), _rows_with_big_terms(rng, 300, d, "f32")
        for metric in ("l2", "dot"):
            swap = _differ(sj.lanes16, sj.dot32, x, y, metric)
            tail = _differ(sj.lanes16, sj.tail_in_lanes, x, y, metric)
            bfirst = _differ(sj.dot32, sj.dot32_b_first, x, y, metric)
            dtail = _differ(sj.dot32, sj.tail_in_lanes, x, y, metric)
            assert (swap > 0) == (d > 17), (d, metric, swap)
            assert (tail > 0) == (d > 16 and d % 16 != 0), (d, metric, tail)
            assert (bfirst > 0) == (d >= 32), (d, metric, bfirst)
            assert (dtail > 0) == (d > 16), (d, metric, dtail)


# ---- cases built to pin the rules -----------------------------------------------------------------------------------
def _tie_case(d, dt, metric, seed, K=8, part=2, n_bc=512, n_a=320, n_c=48, n_stay=0):
    """An index whose distances all share two large terms, one in the 16-lane chunks (element 0) and one in the tail
    (element d - 1), so that they differ only by small terms the large partial sums absorb differently in each order.
    Partition `part` holds n_bc rows that the k = 2 training sees (two groups, so c1 and c2 are far from the rest)
    and then n_a rows near c0, whose candidate scan decides them; each other partition holds n_stay rows that clearly
    stay and then n_c rows between their own centroid and c1.  Returns (centroids, partition of each row, rows) as f32
    values exact in dt, rows grouped by partition in id order."""
    rng = np.random.default_rng(seed)
    P = [0, d - 1]

    def small(n):
        return (rng.standard_normal((n, d)) * 0.3).astype(np.float32)
    cent, bc, a, c = small(K), small(n_bc), small(n_a), small(n_c * (K - 1))
    st = small(n_stay * (K - 1))
    two = np.where(np.arange(n_bc) % 2 == 0, 1.0, 2.0).astype(np.float32)
    if metric == "l2":
        b = np.float32(2000.0)
        cent[:, P] = 0
        cent[part, P] = b
        bc[:, P] = 2 * b
        bc[:, 1] += 3 * (2 * two - 3)      # +-3: two groups
        a[:, P] = b
        a[::2, 1] += 1.5
        c[:, P] = b
        c[:, 1] += 1.5
        st[:, 1] -= 3.0
    else:
        b = np.float32(1000.0)
        for m in (cent, bc, a, c, st):
            m[:, P] = b
        cent[:, 1] = 30.0                  # c0 and every candidate: the same large term in element 1 too
        bc[:, 1] -= 3 * two
        a[:, 1] = 100.0                    # far nearer c0 and the candidates than c1 / c2 (dot k-means splits
        c[:, 1] = 0.0                      # the groups along elements 0 and d - 1)
        st[:, 1] = 6.0
    rows, parts = [np.concatenate([bc, a])], [np.full(n_bc + n_a, part, np.uint32)]
    j = 0
    for q in range(K):
        if q == part:
            continue
        rows.append(np.concatenate([st[j * n_stay:(j + 1) * n_stay], c[j * n_c:(j + 1) * n_c]]))
        parts.append(np.full(n_stay + n_c, q, np.uint32))
        j += 1
    rows = np.concatenate(rows)
    parts = np.concatenate(parts)
    order = np.argsort(parts, kind="stable")
    return psj._round(cent, dt), parts[order], psj._round(rows[order], dt)


def _wrong_rules(metric, dt, d):
    """(name, rule of every distance, rule of the candidate scan) for each wrong rule the decisions must expose"""
    right = sj.batch_rule(metric, dt)
    out = []
    if d > 16 and d % 16:
        out.append(("tail walked into the lanes", right, sj.tail_in_lanes))
    if metric == "dot" and d > 17:
        swap = sj.lanes16 if right is sj.dot32 else sj.dot32
        out.append(("LANES16 / DOT32 swapped", swap, swap))
        if dt != "f32" and d >= 32:
            out.append(("DOT32 folded upper half first", right, sj.dot32_b_first))
    return out


def _assert_discriminates(cent, parts, x, part, metric, dt, c12=None):
    """the right numpy rule gives the oracle's decisions and every wrong rule changes at least one; returns the
    right rule's decisions"""
    d = x.shape[1]
    right = sj.batch_rule(metric, dt)
    D = sj.matrix(right, metric)
    kw = {}
    if c12 is not None:   # a split: the candidates' rows too
        cands = sj.select_reassign_candidates(D(cent[part:part + 1], cent)[0], part)
        kw = dict(c12=c12, cand_rows=np.concatenate([x[parts == q] for q in cands] + [x[:0]]),
                  cand_parts=np.concatenate([parts[parts == q] for q in cands] + [parts[:0]]))
    _, want = sj.decisions(D, cent, part, x[parts == part], **kw)
    for name, w_all, w_scan in _wrong_rules(metric, dt, d):
        _, got = sj.decisions(sj.matrix(w_all, metric), cent, part, x[parts == part], Dc=sj.matrix(w_scan, metric),
                              **kw)
        assert not np.array_equal(got, want), f"{name} changes no decision: the case would not test it"
    return want


@pytest.mark.parametrize("d", [20, 36, 44, 100])
@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("metric", ["l2", "dot"])
def test_constructed_cases_discriminate(d, dt, metric):
    """CPU: the cases of the device tests below tell every wrong rule apart, with c1 and c2 from the oracle's
    k = 2 training, and the right numpy rule decides as the oracle does"""
    cent, parts, x = _tie_case(d, dt, metric, seed=d)
    part = 2
    c12 = psj._new_centroids(_native(x[parts == part], dt), metric, dt, seed=d)
    want = _assert_discriminates(cent, parts, x, part, metric, dt, c12=c12)
    _assert_discriminates(cent, parts, x, part, metric, dt)
    dist = _oracle_pairs(metric, dt)
    cc = lambda a: _native(a, dt) if dt == "bf16" else a  # noqa: E731
    cands = sj.select_reassign_candidates([dist(cc(cent[part]), cc(c)) for c in cent], part)
    cx = np.concatenate([x[parts == q] for q in cands])
    cp = np.concatenate([parts[parts == q] for q in cands])
    _, oracle = sj.split_decisions(dist, cc(cent), part, cc(c12[0]), cc(c12[1]), [cc(r) for r in x[parts == part]],
                                   [cc(r) for r in cx], cp)
    assert np.array_equal(want, oracle)


# ---- device helpers -------------------------------------------------------------------------------------------------
def _flat(cent, parts, x, ids, metric, dt):
    return lb.IvfFlatIndex.from_parts(_native(cent, dt), parts, _native(x, dt), ids, metric, bf16=dt == "bf16")


def _inputs(ix, e, col, ids_all, part):
    """the raw rows the host fetches by row id (ids_all ascending): the partition's, then its candidates' grouped in
    candidate order"""
    offs = e["part_offsets"].astype(np.int64)
    rid = e["row_ids"]

    def rows_of(p):
        ids = np.sort(rid[offs[p]:offs[p + 1]])
        return col[np.searchsorted(ids_all, ids)], ids
    cands = ix.reassign_candidates(part)
    v, r = rows_of(part)
    cv, cr, cp = [col[:0]], [np.zeros(0, np.uint64)], [np.zeros(0, np.uint32)]
    for q in cands:
        a, b = rows_of(int(q))
        cv.append(a), cr.append(b), cp.append(np.full(len(b), q, np.uint32))
    return cands, v, r, np.concatenate(cv), np.concatenate(cr), np.concatenate(cp)


def _cc(dt):
    """model values as the oracle takes them"""
    return (lambda a: psj._bf16_bits(a)) if dt == "bf16" else (lambda a: np.asarray(a))


def _split_and_check(kind, ix, col, ids_all, part, metric, dt, seed, check_index=True):
    """split `part` on the device; candidates, new centroids and every destination against the oracle, and the new
    index against the restated merge.  Returns (dest, c12, split inputs)."""
    e = ix.export()
    K = len(e["part_offsets"]) - 1
    cands, v, r, cv, cr, cp = _inputs(ix, e, col, ids_all, part)
    dist = _oracle_pairs(metric, dt)
    cent = psj._round(e["centroids"], dt)
    cc = _cc(dt)
    assert cands.tolist() == sj.select_reassign_candidates([dist(cc(cent[part]), cc(c)) for c in cent], part)
    out, got = ix.split(part, v, r, cv, cr, cp, seed=seed)
    c12 = psj._new_centroids(v, metric, dt, seed)
    newc = psj._as_f32(got["new_centroids"], dt) if dt == "bf16" else np.asarray(got["new_centroids"], np.float32)
    assert np.array_equal(newc[part].view(np.uint32), c12[0].view(np.uint32))
    assert np.array_equal(newc[K].view(np.uint32), c12[1].view(np.uint32))
    _, want = sj.split_decisions(dist, cc(cent), part, cc(c12[0]), cc(c12[1]), list(v), list(cv), cp)
    assert np.array_equal(got["dest"], want)
    if check_index:
        offs, rows, src = psj._restated_split(kind, ix, e, col, part, newc, cands, v, r, cv, cr, cp, got["dest"],
                                              metric, dt)
        tio._check_merge(kind, ix, out, e, offs, rows, src, metric, seed, dt=dt)
    return got["dest"], c12, (cands, v, r, cv, cr, cp)


def _join_and_check(kind, ix, col, ids_all, part, metric, dt, seed, check_index=True):
    """join `part` on the device; destinations against the oracle and the new index against the restated merge"""
    e = ix.export()
    K = len(e["part_offsets"]) - 1
    offs = e["part_offsets"].astype(np.int64)
    ids = np.sort(e["row_ids"][offs[part]:offs[part + 1]])
    v = col[np.searchsorted(ids_all, ids)]
    out, dest = ix.join(part, v, ids, seed=seed)
    cent = psj._round(e["centroids"], dt)
    cc = _cc(dt)
    _, want = sj.join_decisions(_oracle_pairs(metric, dt), cc(cent), part, list(v))
    assert np.array_equal(dest, want)
    if check_index:
        newc = np.delete(e["centroids"], part, 0)
        add = dict(row_ids=ids, **psj._moved_payload(kind, e, newc, v, dest, metric, dt))
        pm = np.array([q if q < part else (tio.DROP if q == part else q - 1) for q in range(K)], np.uint32)
        o2, rows, src = tio.merge(e["part_offsets"], tio._rows(kind, e), pm, [], dest, add, K - 1)
        tio._check_merge(kind, ix, out, e, o2, rows, src, metric, seed, dt=dt)
    return dest, v


def _cosine_bound(d):
    """the device's cosine is within this of the f64 value (tests/test_linalg_primitives.py, S <= 1), and so is the
    oracle's"""
    return 3.0 * (math.ceil(d / 32) + 5) * 2.0 ** -24 + 2.0 ** -24


def _assert_cosine_margins(dist, cent, part, rows, c12=None, cand_rows=(), cand_parts=()):
    """no comparison a decision makes is closer in the oracle's values than twice the bound of each side: the
    device's cosine (off by at most the bound) then decides every row as the oracle does"""
    d = len(cent[0])
    gap = 4 * _cosine_bound(d)

    def far(a, b):
        return np.all(np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64)) > gap)
    ranking = np.array([dist(cent[part], c) for c in cent], np.float64)
    srt = np.sort(np.delete(ranking, part))
    assert far(srt[1:], srt[:-1]), "two candidates rank within the cosine bound"
    cands = sj.select_reassign_candidates(list(ranking), part)

    def scan(r):
        return np.sort(np.array([dist(r, cent[c]) for c in cands], np.float64))
    for r in rows:
        if c12 is None:
            ds = scan(r)
            assert len(ds) < 2 or far(ds[1], ds[0]), "a joined row's nearest candidates are within the bound"
            continue
        d0, d1, d2 = dist(cent[part], r), dist(c12[0], r), dist(c12[1], r)
        assert far(d0, d1) and far(d0, d2) and far(d1, d2), "a split row's d0 / d1 / d2 are within the bound"
        if d0 <= d1 and d0 <= d2:
            ds = scan(r)
            assert (len(ds) < 2 or far(ds[1], ds[0])) and far(ds[0], d1) and far(ds[0], d2)
    for r, q in zip(cand_rows, cand_parts):
        d0, d1, d2 = dist(cent[q], r), dist(c12[0], r), dist(c12[1], r)
        assert far(d0, d1) and far(d0, d2) and far(d1, d2), "a candidate row's distances are within the bound"


def _cosine_case(d, dt, seed, split, train_seed=0, K=8, part=2, n_part=300, n_c=30):
    """Random clustered rows, partition `part` the largest, the centroids spread in their cosine to c0 so that the
    candidates rank far apart.  The first of seed, seed + 1, .. whose oracle decisions (with c1 and c2 trained with
    train_seed for a split) all clear the cosine bound: (centroids, partition of each row, rows)."""
    for s in range(seed, seed + 20):
        rng = np.random.default_rng(s)
        base = rng.standard_normal((K, d)).astype(np.float32)
        w = np.linspace(0.0, 0.9, K, dtype=np.float32)[rng.permutation(K)][:, None]
        cent = psj._round(w * base[part] + (1 - w) * base, dt)
        sizes = np.full(K, n_c)
        sizes[part] = n_part
        parts = np.repeat(np.arange(K, dtype=np.uint32), sizes)
        x = psj._round(cent[parts] + rng.standard_normal((len(parts), d)).astype(np.float32) * np.float32(0.5), dt)
        col, cc, dist = _native(x, dt), _cc(dt), _oracle_pairs("cosine", dt)
        try:
            if not split:
                _assert_cosine_margins(dist, [cc(c) for c in cent], part, list(col[parts == part]))
                return cent, parts, x
            c12 = psj._new_centroids(col[parts == part], "cosine", dt, train_seed)
            cands = sj.select_reassign_candidates([dist(cc(cent[part]), cc(c)) for c in cent], part)
            _assert_cosine_margins(dist, [cc(c) for c in cent], part, list(col[parts == part]), [cc(c) for c in c12],
                                   [r for q in cands for r in col[parts == q]],
                                   np.concatenate([parts[parts == q] for q in cands]))
            return cent, parts, x
        except AssertionError:
            continue
    raise AssertionError("no seed gives a cosine case whose decisions clear the bound")


# ---- 2. split and join decisions at dimension tails, every element type and metric (IVF_FLAT) -----------------------
CASES = [(d, dt, m) for d in DIMS for dt in DTYPES for m in ("l2", "dot", "cosine")]


@pytest.mark.gpu
@pytest.mark.parametrize("d,dt,metric", CASES)
def test_split_decisions_at_tail_dimensions(d, dt, metric):
    part, seed = 2, d + 1
    if metric == "cosine":   # its margins are asserted where the case is chosen
        cent, parts, x = _cosine_case(d, dt, d, split=True, train_seed=seed)
    else:
        cent, parts, x = _tie_case(d, dt, metric, seed=d)
        c12 = psj._new_centroids(_native(x[parts == part], dt), metric, dt, seed)
        _assert_discriminates(cent, parts, x, part, metric, dt, c12=c12)
    ids = np.arange(len(x), dtype=np.uint64)
    col = _native(x, dt)
    ix = _flat(cent, parts, x, ids, metric, dt)
    _split_and_check("flat", ix, col, ids, part, metric, dt, seed)


@pytest.mark.gpu
@pytest.mark.parametrize("d,dt,metric", CASES)
def test_join_decisions_at_tail_dimensions(d, dt, metric):
    part, seed = 2, d + 2
    if metric == "cosine":
        cent, parts, x = _cosine_case(d, dt, d + 7, split=False)
    else:
        cent, parts, x = _tie_case(d, dt, metric, seed=d)
        _assert_discriminates(cent, parts, x, part, metric, dt)
    ids = np.arange(len(x), dtype=np.uint64)
    ix = _flat(cent, parts, x, ids, metric, dt)
    _join_and_check("flat", ix, _native(x, dt), ids, part, metric, dt, seed)


# ---- 3. every index kind at 16-bit types -----------------------------------------------------------------------------
def _build16(kind, x, metric, dt, K, seed):
    data, bf = _native(x, dt), dt == "bf16"
    rid = np.arange(len(x), dtype=np.uint64)
    hp = lb.HnswBuildParams(**tio.HNSW)
    if kind == "hnsw_pq":
        prm = lb.IvfBuildParams(num_partitions=K, num_sub_vectors=4, max_iters=8, pq_max_iters=4, seed=seed)
        return lb.IvfHnswPqIndex.build(data, metric, prm, hp, row_ids=rid, bf16=bf)
    args = dict(num_partitions=K, max_iters=8, seed=seed, row_ids=rid, bf16=bf)
    if kind == "sq":
        return lb.IvfSqIndex.build(data, metric, **args)
    if kind == "hnsw_sq":
        return lb.IvfHnswSqIndex.build(data, metric, hnsw_params=hp, **args)
    return lb.IvfHnswFlatIndex.build(data, metric, hnsw_params=hp, **args)


KIND16 = ([(k, dt, "l2") for k in ("sq", "hnsw_sq", "hnsw_pq", "hnsw_flat") for dt in ("f16", "bf16")]
          + [("hnsw_flat", "f16", "cosine"), ("hnsw_sq", "bf16", "dot")])


@pytest.mark.gpu
@pytest.mark.parametrize("kind,dt,metric", KIND16)
def test_split_and_join_of_every_kind_at_16_bit_types(kind, dt, metric):
    """d = 20 (a 4-element tail under both lane rules): the moved rows' payload and the rebuilt graphs"""
    n, d, K, seed = 1600, 20, 6, 13
    x = psj._round(tio._data(n, d, seed=17, k=K), dt)
    ids = np.arange(n, dtype=np.uint64)
    col = _native(x, dt)
    ix = _build16(kind, x, metric, dt, K, seed=3)
    part = int(np.argmax(np.diff(ix.export()["part_offsets"]).astype(np.int64)))
    _split_and_check(kind, ix, col, ids, part, metric, dt, seed)
    small = int(np.argmin(np.diff(ix.export()["part_offsets"]).astype(np.int64)))
    _join_and_check(kind, ix, col, ids, small, metric, dt, seed)


# ---- 4. the streamed centroid table at its limits --------------------------------------------------------------------
def _random_index(d, dt, metric, K, n_part, n_other, seed, part=1):
    rng = np.random.default_rng(seed)
    cent = psj._round(rng.standard_normal((K, d)).astype(np.float32), dt)
    sizes = np.full(K, n_other)
    sizes[part] = n_part
    parts = np.repeat(np.arange(K, dtype=np.uint32), sizes)
    x = psj._round(cent[parts] + rng.standard_normal((len(parts), d)).astype(np.float32), dt)
    return cent, parts, x


@pytest.mark.gpu
@pytest.mark.parametrize("dt,metric", [("f32", "l2"), ("bf16", "dot")])
def test_streamed_table_in_chunks_of_three_slots(dt, metric):
    """d = 4604 is the largest d IVF_FLAT takes whose chunk is 3 slots (4605 is the largest at all): c0, c1, c2
    alone in the first chunk, no candidate scan there; the 67 slots stream in 23 chunks, the last holding one.
    bf16 dot: DOT32 with a tail of 28"""
    d, K, part, seed = 4604, 66, 1, 5
    cent, parts, x = _random_index(d, dt, metric, K, 40, 6, seed=d)
    cr = parts != part                 # candidate rows half way to c0: some stay, some go to c1 / c2
    x[cr] = psj._round((x[cr] + cent[part]) * np.float32(0.5), dt)
    ids = np.arange(len(x), dtype=np.uint64)
    col = _native(x, dt)
    ix = _flat(cent, parts, x, ids, metric, dt)
    dest, _, inp = _split_and_check("flat", ix, col, ids, part, metric, dt, seed, check_index=False)
    assert len(inp[0]) == 64
    assert (dest[len(inp[2]):] != STAYS).any() and (dest[len(inp[2]):] == STAYS).any()
    _join_and_check("flat", ix, col, ids, part, metric, dt, seed, check_index=False)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["f16", "bf16"])
def test_streamed_table_under_cosine_at_16_bit(dt):
    """d = 1536: 67 slots in chunks of 24, the cosine sums of the streamed slots"""
    d, K, part, seed = 1536, 70, 1, 6
    cent, parts, x = _cosine_case(d, dt, d, split=True, train_seed=seed, K=K, part=part, n_part=60, n_c=4)
    ids = np.arange(len(x), dtype=np.uint64)
    col = _native(x, dt)
    ix = _flat(cent, parts, x, ids, "cosine", dt)
    _split_and_check("flat", ix, col, ids, part, "cosine", dt, seed)


@pytest.mark.gpu
def test_dimension_past_the_shared_memory_limit_is_unsupported():
    """d = 4608 (past 4605): not even 3 slots fit the decision kernel's shared memory"""
    d = 4608
    cent, parts, x = _random_index(d, "f32", "l2", 4, 20, 5, seed=1)
    ids = np.arange(len(x), dtype=np.uint64)
    ix = _flat(cent, parts, x, ids, "l2", "f32")
    _, v, r, cv, cr, cp = _inputs(ix, ix.export(), x, ids, 1)
    for call in (lambda: ix.split(1, v, r, cv, cr, cp), lambda: ix.join(1, v, r)):
        with pytest.raises(lb.LanceB200Error) as ei:
            call()
        assert ei.value.status == lb._lib.UNSUPPORTED


# ---- 5. many sweeps of the resident grid -----------------------------------------------------------------------------
@pytest.mark.gpu
def test_resident_grid_sweeps_its_rows_several_times():
    """more than 25 344 raw rows (3 x 132 SMs x 8 blocks x 8 warps) at d = 36 under bf16 dot: every warp decides
    several rows, and the moved-row compaction spans many 1024-row blocks, some of which move nothing"""
    d, dt, metric, part, seed = 36, "bf16", "dot", 2, 8
    cent, parts, x = _tie_case(d, dt, metric, seed=9, n_a=10000, n_c=100, n_stay=2100)
    assert len(x) > 25344
    ids = np.arange(len(x), dtype=np.uint64)
    col = _native(x, dt)
    c12 = psj._new_centroids(col[parts == part], metric, dt, seed)
    want = _assert_discriminates(cent, parts, x, part, metric, dt, c12=c12)
    blocks = np.add.reduceat((want != STAYS).astype(np.int64), np.arange(0, len(want), 1024))
    assert (blocks == 0).sum() >= 2 and (blocks > 0).sum() >= 10
    ix = _flat(cent, parts, x, ids, metric, dt)
    dest, _, _ = _split_and_check("flat", ix, col, ids, part, metric, dt, seed)
    assert np.array_equal(dest, want)


# ---- 6. candidate-ranking and row-set edges --------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("K", [65, 66])
def test_candidates_at_65_and_66_partitions(K):
    d, part, seed = 20, 4, 3
    cent, parts, x = _random_index(d, "f32", "l2", K, 200, 5, seed=K, part=part)
    ids = np.arange(len(x), dtype=np.uint64)
    ix = _flat(cent, parts, x, ids, "l2", "f32")
    _, _, inp = _split_and_check("flat", ix, x, ids, part, "l2", "f32", seed)
    assert len(inp[0]) == 64 and part not in inp[0].tolist()
    _join_and_check("flat", ix, x, ids, part, "l2", "f32", seed)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["f32", "bf16"])
def test_dot_partition_outside_its_own_first_65(dt):
    """under dot, 1 - <c0, c0> need not be the smallest distance: centroid `part` is short, 69 others point its
    way and are longer, so it is not among its own first 65 and the 65th nearest is dropped"""
    d, K, part, seed = 36, 70, 5, 4
    rng = np.random.default_rng(11)
    u = np.zeros(d, np.float32)
    u[0] = 1.0
    cent = (u * rng.uniform(2.0, 4.0, (K, 1)) + rng.standard_normal((K, d)) * 0.3).astype(np.float32)
    cent[part] = u * 0.5 + rng.standard_normal(d).astype(np.float32) * 0.05
    cent = psj._round(cent, dt)
    sizes = np.full(K, 5)
    sizes[part] = 120
    parts = np.repeat(np.arange(K, dtype=np.uint32), sizes)
    x = psj._round(cent[parts] + rng.standard_normal((len(parts), d)).astype(np.float32) * 0.3, dt)
    dist = _oracle_pairs("dot", dt)
    cc = _cc(dt)
    dd = [dist(cc(cent[part]), cc(c)) for c in cent]
    first65 = sorted(range(K), key=lambda j: (sj._total_key(dd[j]), j))[:65]
    assert part not in first65
    assert sj.select_reassign_candidates(dd, part) == first65[:64]
    ids = np.arange(len(x), dtype=np.uint64)
    col = _native(x, dt)
    ix = _flat(cent, parts, x, ids, "dot", dt)
    _split_and_check("flat", ix, col, ids, part, "dot", dt, seed)
    _join_and_check("flat", ix, col, ids, part, "dot", dt, seed)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", ["f16", "bf16"])
@pytest.mark.parametrize("which", ["first", "last"])
def test_join_of_the_first_and_last_partition_at_16_bit(dt, which):
    d, K, seed = 36, 7, 2
    part = 0 if which == "first" else K - 1
    cent, parts, x = _random_index(d, dt, "dot", K, 150, 30, seed=21, part=part)
    ids = np.arange(len(x), dtype=np.uint64)
    ix = _flat(cent, parts, x, ids, "dot", dt)
    dest, _ = _join_and_check("flat", ix, _native(x, dt), ids, part, "dot", dt, seed)
    assert dest.max() <= K - 2 and len(np.unique(dest)) > 1


@pytest.mark.gpu
def test_empty_and_one_row_candidates_with_fragment_row_ids():
    """candidate partitions with no row and with one row, and Lance row ids (fragment << 32) | offset over several
    fragments"""
    d, K, part, seed = 20, 6, 1, 12
    rng = np.random.default_rng(5)
    cent = rng.standard_normal((K, d)).astype(np.float32)
    sizes = np.array([30, 700, 0, 1, 25, 0])
    parts = np.repeat(np.arange(K, dtype=np.uint32), sizes)
    x = (cent[parts] + rng.standard_normal((len(parts), d)).astype(np.float32)).astype(np.float32)
    pos = np.arange(len(x))
    ids = ((pos // 97).astype(np.uint64) << np.uint64(32)) | (pos % 97 * 3 + 1).astype(np.uint64)
    assert len(np.unique(ids >> np.uint64(32))) >= 8 and np.all(np.diff(ids.astype(np.float64)) > 0)
    ix = _flat(cent, parts, x, ids, "l2", "f32")
    cands = ix.reassign_candidates(part).tolist()
    assert 2 in cands and 3 in cands and 5 in cands
    dest, _, inp = _split_and_check("flat", ix, x, ids, part, "l2", "f32", seed)
    assert inp[4].max() > np.uint64(1 << 32)
    _join_and_check("flat", ix, x, ids, part, "l2", "f32", seed)
    for empty in (2, 5):   # a partition without rows joins without raw rows
        out, dd = ix.join(empty, np.zeros((0, d), np.float32), np.zeros(0, np.uint64))
        assert dd.size == 0 and out.info()["num_partitions"] == K - 1 and out.info()["num_rows"] == len(x)
