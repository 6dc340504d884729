"""IVF_RQ restated from the reference for the tests (no product code).

Everything is f32 element-wise arithmetic, which numpy performs exactly as the reference's Rust does (each product and
sum rounded on its own, no contraction), in the reference's order:
  - rotation: `dot(R[j, :d], x)` (lance-linalg/src/distance/dot.rs:30-58, the CPU oracle's lo_dot_f32) for the query
    side (bq/storage.rs:130-156); the data side is defined the same way (the reference's ndarray GEMM has no
    specified summation order), with a sequential sum of |rot| (codes_res_dot_dists, bq/builder.rs:100-141);
  - transform: RQTransformer::transform (bq/transform.rs:70-220) after IvfTransformer::with_rq (ivf.rs:281-328);
  - distances: RabitDistCalculator (bq/storage.rs:160-445): the lowbit-chain table, its u8 quantisation, the 16-bit
    sums of the x86 kernels (which wrap mod 2^16, dist_table.rs:96-160 and dist_table.c), the exact f32 pair sums
    of the last n % 32 rows, and the f32 epilogue.
The search is FlatIndex::search (flat/index.rs:82-177) through the CPU oracle's restated heap (oracle/binding.py
flat_topk), and the global merge by (_distance, _rowid) (rust/lance/src/dataset/scanner.rs:3450-3466).
"""
import numpy as np

from oracle import binding as ob

PERM0 = (0, 8, 1, 9, 2, 10, 3, 11, 4, 12, 5, 13, 6, 14, 7, 15)   # bq/storage.rs:40


def dot16(X, R):
    """Y[m][j] = dot(R[j], X[m]): the d % 16 tail summed first, 16 lane sums over the 16-wide chunks folded 0..15,
    then tail + fold (the oracle's lo_dot_f32)."""
    X = np.ascontiguousarray(X, np.float32)
    R = np.ascontiguousarray(R, np.float32)
    m, d = X.shape
    J = R.shape[0]
    assert R.shape[1] == d
    out = np.empty((m, J), np.float32)
    n16 = d // 16 * 16
    step = max(1, (1 << 22) // max(1, 16 * J))
    for a in range(0, m, step):
        x = X[a:a + step]
        s = np.zeros((x.shape[0], J), np.float32)
        for i in range(n16, d):
            s = s + x[:, i:i + 1] * R[None, :, i]
        lanes = np.zeros((16, x.shape[0], J), np.float32)
        for c in range(0, n16, 16):
            lanes += x[:, c:c + 16].T[:, :, None] * R[:, c:c + 16].T[:, None, :]
        t = np.zeros((x.shape[0], J), np.float32)
        for lane in range(16):
            t = t + lanes[lane]
        out[a:a + step] = s + t
    return out


def seq_sum(a, axis=-1, start=0.0):
    """a left fold of f32 adds along `axis` from `start` (Rust's iterator `sum`)"""
    a = np.moveaxis(np.asarray(a, np.float32), axis, 0)
    s = np.full(a.shape[1:], start, np.float32)
    for v in a:
        s = s + v
    return s


def pack_signs(rot):
    """bit j = rot[j].is_sign_positive(), LSB-first bytes (BitVec<u8, Lsb0>, bq/builder.rs:170-173)"""
    return np.packbits(~np.signbit(np.asarray(rot, np.float32)), axis=-1, bitorder="little")


def rq_transform(centroids, rotation, vectors, metric="l2", num_bits=1):
    """-> part_ids, codes [n][code_dim / 8], add, scale, valid (rows with valid False have zero outputs)"""
    cent = np.ascontiguousarray(centroids, np.float32)
    x = np.ascontiguousarray(vectors, np.float32)
    n, d = x.shape
    cd = d * num_bits
    if metric == "cosine":
        x = ob.normalize_rows(x)                                   # NormalizeTransformer, then L2 everywhere
    m = "dot" if metric == "dot" else "l2"
    with np.errstate(all="ignore"):
        finite = np.isfinite(x).all(axis=1)                        # KeepFiniteVectors
        part, dist, ok = ob.compute_membership(cent, np.where(finite[:, None], x, 0), metric=m)
    valid = finite & ok
    part = np.where(valid, part, 0).astype(np.uint32)
    res = np.where(valid[:, None], x - cent[part], 0).astype(np.float32)
    rot = dot16(res, np.ascontiguousarray(rotation, np.float32)[:, :d])
    codes = pack_signs(rot)
    sqrt_d = np.sqrt(np.float32(d) * np.float32(num_bits))
    ip = seq_sum(np.abs(rot), axis=1) / sqrt_d
    with np.errstate(all="ignore"):
        if m == "l2":
            rns = dist
            add = rns.copy()
            scale = np.where(ip == 0, np.float32(0), (np.float32(-2.0) * rns) / ip).astype(np.float32)
        else:
            rns = seq_sum(res * res, axis=1)                         # norm_squared_fsl
            cn = seq_sum(cent * cent, axis=1)
            add = (dist + cn[part]).astype(np.float32)
            scale = -np.where(ip == 0, np.float32(0), rns / ip).astype(np.float32)
    codes[~valid] = 0
    add = np.where(valid, add, 0).astype(np.float32)
    scale = np.where(valid, scale, 0).astype(np.float32)
    assert codes.shape == (n, cd // 8)
    return part, codes, add, scale, valid


def dist_table(rq):
    """build_dist_table_direct (bq/storage.rs:210-245): [code_dim / 4][16], t[j] = t[j - lowbit(j)] + rq[4s + ctz(j)]"""
    sub = np.asarray(rq, np.float32).reshape(-1, 4)
    t = np.zeros((sub.shape[0], 16), np.float32)
    for j in range(1, 16):
        lb = j & -j
        t[:, j] = t[:, j - lb] + sub[:, lb.bit_length() - 1]
    return t


def _total_key(d):
    b = np.asarray(d, np.float32).view(np.int32).astype(np.int64)
    return np.where(b < 0, b ^ 0x7FFFFFFF, b)


def quantize_table(t):
    """quantize_dist_table (bq/storage.rs:249-267) -> (qmin, qmax, u8 table)"""
    flat = np.asarray(t, np.float32).ravel()
    k = _total_key(flat)
    qmin, qmax = flat[np.argmin(k)], flat[np.argmax(k)]
    if qmin == qmax:
        return qmin, qmax, np.zeros(t.shape, np.uint8)
    factor = np.float32(255.0) / (qmax - qmin)
    v = (np.asarray(t, np.float32) - qmin) * factor
    fl = np.floor(v)
    r = np.where(v - fl >= 0.5, fl + 1, fl)                       # f32::round: half away from zero (v >= 0)
    r = np.where(np.isnan(r), 0, r)                                # `as u8`: NaN -> 0, saturating
    return qmin, qmax, np.clip(r, 0, 255).astype(np.uint8)


def rq_distances(rq, codes, add, scale, q_factor, exact_all=False):
    """RabitDistCalculator::distance_all (exact_all False) or per-row distance (True) over one partition's rows"""
    rq = np.asarray(rq, np.float32)
    codes = np.asarray(codes, np.uint8)
    n, cb = codes.shape
    t = dist_table(rq)
    # the fold from -0.0: -0.0 + a0 == a0, so it equals numpy's accumulate, which adds strictly left to right
    sum_q = np.add.accumulate(rq, dtype=np.float32)[-1] if rq.size else np.float32(-0.0)
    sqrt_d = np.sqrt(np.float32(rq.size))
    lo, hi = (codes & 15).astype(np.int64), (codes >> 4).astype(np.int64)
    i2 = np.arange(cb)
    nq = 0 if exact_all else n - n % 32
    dist = np.empty(n, np.float32)
    pairs = t[2 * i2, lo[nq:]] + t[2 * i2 + 1, hi[nq:]]             # [n - nq][cb] f32
    dist[nq:] = seq_sum(pairs, axis=1, start=-0.0 if exact_all else 0.0)
    if nq:
        qmin, qmax, qt = quantize_table(t)
        qt = qt.astype(np.int64)
        qs = (qt[2 * i2, lo[:nq]] + qt[2 * i2 + 1, hi[:nq]]).sum(axis=1) & 0xFFFF   # u16 lanes that wrap
        rng = (qmax - qmin) / np.float32(255.0)
        sum_min = np.float32(t.shape[0]) * qmin
        dist[:nq] = qs.astype(np.float32) * rng + sum_min
    dvq = (np.float32(2.0) * dist - sum_q) / sqrt_d
    return ((dvq * np.asarray(scale, np.float32)) + np.asarray(add, np.float32)) + np.float32(q_factor)


def ivfrq_search(centroids, rotation, part_offsets, codes, add, scale, row_ids, queries, k, nprobes, metric="l2",
                 allow=None, block=None, lower=None, upper=None):
    """IVFIndex::search over an IVF_RQ index held as CSR-by-partition arrays -> ([nq][k] ids, dists, counts).
    With a mask every selected row is scored by DistCalculator::distance and unselected rows never reach the heap
    (flat/index.rs:129-165)."""
    cent = np.ascontiguousarray(centroids, np.float32)
    K, d = cent.shape
    R = np.ascontiguousarray(rotation, np.float32)[:, :d]
    offs = np.asarray(part_offsets, np.int64)
    codes = np.asarray(codes, np.uint8)
    add, scale = np.asarray(add, np.float32), np.asarray(scale, np.float32)
    row_ids = np.asarray(row_ids, np.uint64)
    queries = np.ascontiguousarray(queries, np.float32)
    if metric == "cosine":
        queries = ob.normalize_rows(queries)                      # knn.rs:497-499
    cmetric = "dot" if metric == "dot" else "l2"
    masked = allow is not None or block is not None
    allow_set = None if allow is None else set(np.asarray(allow, np.uint64).tolist())
    block_set = set() if block is None else set(np.asarray(block, np.uint64).tolist())
    nq = queries.shape[0]
    oi = np.full((nq, k), np.iinfo(np.uint64).max, np.uint64)
    od = np.full((nq, k), np.inf, np.float32)
    oc = np.zeros(nq, np.uint32)
    for qi in range(nq):
        q = queries[qi]
        pids, pd = ob.find_partitions(cent, q, min(nprobes, K), metric=cmetric)
        rqs = dot16(q[None, :] - cent[pids], R)                   # v2.rs:316-332, storage.rs:130-156
        cid, cd = [], []
        for p, dqc, rq in zip(pids, pd, rqs):
            a, b = offs[p], offs[p + 1]
            if a == b:
                continue
            qf = dqc if metric == "l2" else np.float32(dqc) - np.float32(1.0)   # storage.rs:427-434
            rid = row_ids[a:b]
            dist = rq_distances(rq, codes[a:b], add[a:b], scale[a:b], qf, exact_all=masked)
            if masked:
                sel = np.array([(allow_set is None or r in allow_set) and r not in block_set for r in rid.tolist()],
                               dtype=bool)
                dist, rid = dist[sel], rid[sel]
            ids, ds = ob.flat_topk(dist, rid, k, lower, upper)
            cid.append(ids)
            cd.append(ds)
        if not cid:
            continue
        ids, ds = np.concatenate(cid), np.concatenate(cd)
        order = np.lexsort((ids, _total_key(ds)))[:k]
        oi[qi, :order.size], od[qi, :order.size], oc[qi] = ids[order], ds[order], order.size
    return oi, od, oc


def pack_codes_block(codes32):
    """pack_codes (bq/storage.rs:477-544) of one block of 32 rows [32][code_len] -> the x86 kernels' layout"""
    codes32 = np.asarray(codes32, np.uint8)
    code_len = codes32.shape[1]
    out = np.zeros(32 * code_len, np.uint8)
    for i in range(code_len):
        col = codes32[:, i]
        c0, c1 = col & 0xF, col >> 4
        for j in range(16):
            out[i * 32 + j] = c0[PERM0[j]] | (c0[PERM0[j] + 16] << 4)
            out[i * 32 + j + 16] = c1[PERM0[j]] | (c1[PERM0[j] + 16] << 4)
    return out
