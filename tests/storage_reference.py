"""numpy restatements of the reference's storage layouts, written from reading the reference (nothing copied):

- pack_codes / unpack_codes (lance-index/src/vector/bq/storage.rs:477-601): RaBitQ codes of one partition in 32-row
  blocks in PERM0 nibble order (lance-linalg/src/simd/dist_table.rs:10), the last n % 32 rows transposed;
- HNSW::to_batch / HNSW::load (lance-index/src/vector/hnsw/builder.rs:579-640,788-833) with HnswMetadata's
  level_offsets (:283-303), over the device's dense graph layout (include/lance_b200.h, IVF_HNSW_SQ section), every
  partition's batch back to back as lb2_index_export_storage writes them."""
import numpy as np

PERM0 = [0, 8, 1, 9, 2, 10, 3, 11, 4, 12, 5, 13, 6, 14, 7, 15]
BATCH = 32


def pack_codes(codes):
    """codes [n][code_len] u8 -> the packed values buffer [n][code_len] (one partition)"""
    codes = np.asarray(codes, np.uint8)
    n, cl = codes.shape
    out = np.zeros(n * cl, np.uint8)
    full = n // BATCH * BATCH
    for row in range(0, full, BATCH):
        for i in range(cl):
            col = codes[row:row + BATCH, i]
            lo, hi = col & 0xF, col >> 4
            at = row // BATCH * cl * BATCH + i * BATCH
            for j in range(16):
                out[at + j] = lo[PERM0[j]] | (lo[PERM0[j] + 16] << 4)
                out[at + j + 16] = hi[PERM0[j]] | (hi[PERM0[j] + 16] << 4)
    out[full * cl:] = codes[full:].T.reshape(-1)
    return out.reshape(n, cl)


def unpack_codes(packed):
    """the inverse of pack_codes"""
    packed = np.asarray(packed, np.uint8)
    n, cl = packed.shape
    flat = packed.reshape(-1)
    out = np.zeros((n, cl), np.uint8)
    full = n // BATCH * BATCH
    for b in range(n // BATCH):
        for i in range(cl):
            blk = flat[b * cl * BATCH + i * BATCH:][:BATCH]
            for j in range(16):
                v0, v1 = int(blk[j]), int(blk[j + 16])
                out[b * BATCH + PERM0[j], i] = (v0 & 0xF) | ((v1 & 0xF) << 4)
                out[b * BATCH + PERM0[j] + 16, i] = (v0 >> 4) | ((v1 >> 4) << 4)
    rem = n - full
    if rem:
        out[full:] = flat[full * cl:].reshape(cl, rem).T
    return out


def pack_partitions(codes, part_offsets):
    """pack_codes restarted at every partition (merge_partitions writes each partition's storage on its own)"""
    codes = np.asarray(codes, np.uint8)
    off = np.asarray(part_offsets, np.int64)
    return np.concatenate([pack_codes(codes[off[p]:off[p + 1]]) for p in range(len(off) - 1)]
                          + [np.zeros((0, codes.shape[1]), np.uint8)])


def _lists(g, off, m):
    """{(row, level): (ids, dists)} of the dense layout g (export()["graph"])"""
    out, up = {}, 0
    for r in range(int(off[-1])):
        c = int(g["counts0"][r])
        out[r, 0] = (g["neighbors0"][r][:c], g["dists0"][r][:c])
        for level in range(1, int(g["levels"][r])):
            c = int(g["counts_up"][up])
            out[r, level] = (g["neighbors_up"][up][:c], g["dists_up"][up][:c])
            up += 1
    return out


def to_batch(g, part_offsets):
    """HNSW::to_batch of every partition, back to back: for each level 0 .. max_level - 1 a row per node that has the
    level, ascending node id -> the graph columns of lb2_index_export_storage"""
    off = np.asarray(part_offsets, np.int64)
    K, L, m = len(off) - 1, int(g["max_level"]), int(g["m"])
    lists = _lists(g, off, m)
    vid, lens, nbr, dst = [], [], [], []
    level_offsets = np.zeros((K, L + 1), np.uint64)
    for p in range(K):
        rows = 0
        for level in range(L):
            level_offsets[p, level] = rows
            for i in range(int(off[p + 1] - off[p])):
                r = int(off[p]) + i
                if level < int(g["levels"][r]):
                    ids, ds = lists[r, level]
                    vid.append(i)
                    lens.append(len(ids))
                    nbr.extend(int(x) for x in ids)
                    dst.extend(float(x) for x in ds)
                    rows += 1
        level_offsets[p, L] = rows
    return {"max_level": L, "m": m, "ef_construction": int(g.get("ef_construction", 0)),
            "entry_point": np.zeros(K, np.uint32), "level_offsets": level_offsets,
            "__vector_id": np.array(vid, np.uint32),
            "list_offsets": np.concatenate([[0], np.cumsum(lens, dtype=np.int64)]).astype(np.uint64),
            "__neighbors": np.array(nbr, np.uint32), "_distance": np.array(dst, np.float32)}


def load(s, part_offsets):
    """HNSW::load of every partition's batch into the dense layout: a node has the levels whose batches hold it
    (HNSW::load gives every node all levels, the upper ones of nodes absent there empty, which no list reaches)"""
    off = np.asarray(part_offsets, np.int64)
    K, L, m = len(off) - 1, int(s["max_level"]), int(s["m"])
    n = int(off[-1])
    lo, lof = np.asarray(s["level_offsets"], np.int64), np.asarray(s["list_offsets"], np.int64)
    levels = np.zeros(n, np.uint8)
    lists = {}
    base = 0
    for p in range(K):
        for level in range(L):
            for gr in range(base + lo[p, level], base + lo[p, level + 1]):
                r = int(off[p]) + int(s["__vector_id"][gr])
                lists[r, level] = (s["__neighbors"][lof[gr]:lof[gr + 1]], s["_distance"][lof[gr]:lof[gr + 1]])
                levels[r] = max(levels[r], level + 1)
        base += int(lo[p, L])
    n_up = int(np.sum(np.maximum(levels.astype(np.int64) - 1, 0)))
    g = {"max_level": L, "m": m, "ef_construction": int(s.get("ef_construction", 0)), "levels": levels,
         "counts0": np.zeros(n, np.uint32), "neighbors0": np.zeros((n, 2 * m), np.uint32),
         "dists0": np.zeros((n, 2 * m), np.float32), "counts_up": np.zeros(n_up, np.uint32),
         "neighbors_up": np.zeros((n_up, m), np.uint32), "dists_up": np.zeros((n_up, m), np.float32)}
    up = 0
    for r in range(n):
        for level in range(int(levels[r])):
            ids, ds = lists[r, level]
            if level == 0:
                g["counts0"][r] = len(ids)
                g["neighbors0"][r, :len(ids)], g["dists0"][r, :len(ids)] = ids, ds
            else:
                g["counts_up"][up] = len(ids)
                g["neighbors_up"][up, :len(ids)], g["dists_up"][up, :len(ids)] = ids, ds
                up += 1
    return g
