// storage.cu -- every index kind in the reference's storage layout (the columns merge_partitions writes,
// rust/lance/src/index/vector/builder.rs:938-1079; include/lance_b200.h, lb2_index_storage): IVF_PQ's transposed
// codes, IVF_RQ's packed codes and the HNSW graphs' level batches, converted to and from the device layout by kernels.
#include <algorithm>
#include <memory>

#include "hnsw.cuh"
#include "index.cuh"

namespace lb2 {
namespace {

// ---- IVF_PQ: the codes column-major per partition ----------------------------------------------------------------
// row-major codes [n_p][cw] of the partitions off[0 .. K] -> the reference's storage layout, each partition
// column-major [cw][n_p] (pq/storage.rs:430-450), or back (to_rows); `in` and `out` start at partition 0's first byte
__global__ void transpose_codes_kernel(const uint8_t* __restrict__ in, const uint64_t* __restrict__ off, int K, int cw,
                                       uint64_t total, int to_rows, uint8_t* __restrict__ out) {
  for (uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t o0 = off[0], G = o0 * cw + g;
    const int p = segment_of(off, K, G / cw);
    const uint64_t o = off[p], n = off[p + 1] - o, l = G - o * cw;
    const uint64_t row = (o - o0 + l % n) * cw + l / n;
    if (to_rows) out[row] = in[g];
    else out[g] = in[row];
  }
}
static void transpose_codes(const uint8_t* in, const uint64_t* off, int K, int cw, uint64_t rows, bool to_rows,
                            uint8_t* out) {
  const uint64_t total = rows * cw;
  if (total)
    LB2_LAUNCH("transpose_codes", transpose_codes_kernel, (unsigned)std::min<uint64_t>(cdiv(total, 256), 64ull * ctx().num_sms),
               256, 0, in, off, K, cw, total, to_rows ? 1 : 0, out);
}

// ---- IVF_RQ: the codes packed per partition -----------------------------------------------------------------------
// pack_codes / unpack_codes (bq/storage.rs:477-601), restarted at every partition.  Byte g of the packed column
// belongs to the partition of row g / cl (a partition's packed bytes are its own rows' bytes); inside it, with nb
// full 32-row blocks, byte b * 32 * cl + i * 32 + j (j < 16) holds the low nibbles of byte i of rows 32b + PERM0[j]
// (bits 0..3) and 32b + PERM0[j] + 16 (bits 4..7), byte j + 16 their high nibbles; the n_p % 32 tail rows follow
// column-major [cl][tail].  PERM0[j] = j / 2 + (j % 2) * 8 (lance-linalg/src/simd/dist_table.rs:10).
// One thread per output byte: every byte is written once and read from at most two input bytes.
__global__ void rq_pack_kernel(const uint8_t* __restrict__ codes, const uint64_t* __restrict__ off, int K, int cl,
                               uint64_t total, uint8_t* __restrict__ packed) {
  for (uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (uint64_t)gridDim.x * blockDim.x) {
    const int p = segment_of(off, K, g / cl);
    const uint64_t o = off[p], np = off[p + 1] - o, full = np / 32 * 32;
    const uint64_t l = g - o * cl;  // byte within the partition
    const uint8_t* c = codes + o * cl;
    uint8_t v;
    if (l < full * cl) {
      const uint64_t b = l / (32ull * cl);
      const int i = (int)(l / 32 % cl), j = (int)(l % 32), jj = j & 15;
      const uint64_t r0 = b * 32 + (jj >> 1) + (jj & 1) * 8;  // PERM0[jj]
      const int sh = j < 16 ? 0 : 4;
      v = (uint8_t)(((c[r0 * cl + i] >> sh) & 0xF) | (((c[(r0 + 16) * cl + i] >> sh) & 0xF) << 4));
    } else {
      const uint64_t t = l - full * cl, rem = np - full;
      v = c[(full + t % rem) * cl + t / rem];
    }
    packed[g] = v;
  }
}

// the inverse: byte g of the row-major codes from the packed column
__global__ void rq_unpack_kernel(const uint8_t* __restrict__ packed, const uint64_t* __restrict__ off, int K, int cl,
                                 uint64_t total, uint8_t* __restrict__ codes) {
  for (uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t row = g / cl;
    const int i = (int)(g % cl);
    const int p = segment_of(off, K, row);
    const uint64_t o = off[p], np = off[p + 1] - o, full = np / 32 * 32, r = row - o;
    const uint8_t* c = packed + o * cl;
    uint8_t v;
    if (r < full) {
      const uint64_t base = r / 32 * 32 * cl + (uint64_t)i * 32;
      const int t = (int)(r % 32), h = t >> 4, u = t & 15;
      const int j = (u & 7) * 2 + (u >> 3);  // PERM0[j] == u
      const int sh = h ? 4 : 0;
      v = (uint8_t)(((c[base + j] >> sh) & 0xF) | (((c[base + j + 16] >> sh) & 0xF) << 4));
    } else {
      const uint64_t rem = np - full;
      v = c[full * cl + (uint64_t)i * rem + (r - full)];
    }
    codes[g] = v;
  }
}

// pack_codes (unpack = false) or unpack_codes (unpack = true) of every partition of the part_offsets [K + 1] (device)
// at once: n rows of cl = code_dim / 8 bytes, `codes` and `packed` in partition order
void rq_pack(const uint8_t* codes, const uint64_t* part_offsets, int K, uint64_t n, int cl, uint8_t* packed, bool unpack) {
  const uint64_t total = n * cl;
  if (!total) return;
  const unsigned grid = (unsigned)std::min<uint64_t>(cdiv(total, 256), 64ull * ctx().num_sms);
  if (unpack) LB2_LAUNCH("rq_unpack", rq_unpack_kernel, grid, 256, 0, codes, part_offsets, K, cl, total, packed);
  else LB2_LAUNCH("rq_pack", rq_pack_kernel, grid, 256, 0, codes, part_offsets, K, cl, total, packed);
}

// ---- the reference's storage layout of the graphs (HNSW::to_batch / HNSW::load, builder.rs:283-303,579-640,788-833)
// One record batch per partition: level 0 .. max_level - 1, a row per node that has the level, ascending node id.

// out[0] = 0, out[i + 1] = in[0] + .. + in[i]: a block-local scan of 1024-element tiles, the tile sums scanned by one
// block, then added back
__device__ __forceinline__ uint64_t block_exclusive_scan(uint64_t v, uint64_t* warp_sums, uint64_t* total) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  uint64_t x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint64_t y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warp_sums[w] = x;
  __syncthreads();
  uint64_t before = 0, all = 0;
  for (int i = 0; i < nw; ++i) {
    if (i < w) before += warp_sums[i];
    all += warp_sums[i];
  }
  __syncthreads();
  *total = all;
  return before + x - v;
}

__global__ void scan_tiles_kernel(const uint64_t* __restrict__ in, uint64_t n, uint64_t* __restrict__ tile_sums) {
  __shared__ uint64_t ws[32];
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  uint64_t t;
  block_exclusive_scan(i < n ? in[i] : 0, ws, &t);
  if (threadIdx.x == 0) tile_sums[blockIdx.x] = t;
}

__global__ void scan_sums_kernel(uint64_t* __restrict__ sums, uint64_t nt) {
  __shared__ uint64_t ws[32];
  uint64_t carry = 0;
  for (uint64_t b = 0; b < nt; b += blockDim.x) {
    const uint64_t i = b + threadIdx.x;
    const uint64_t v = i < nt ? sums[i] : 0;
    uint64_t t;
    const uint64_t e = block_exclusive_scan(v, ws, &t);
    if (i < nt) sums[i] = carry + e;
    carry += t;
  }
  if (threadIdx.x == 0) sums[nt] = carry;
}

__global__ void scan_apply_kernel(const uint64_t* __restrict__ in, uint64_t n, const uint64_t* __restrict__ tile_sums,
                                  uint64_t* __restrict__ out) {
  __shared__ uint64_t ws[32];
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  uint64_t t;
  const uint64_t e = block_exclusive_scan(i < n ? in[i] : 0, ws, &t);
  if (i < n) out[i] = tile_sums[blockIdx.x] + e;
  if (i == 0) out[n] = tile_sums[gridDim.x];
}

void scan_u64(const uint64_t* in, uint64_t n, uint64_t* out) {
  if (n == 0) {
    LB2_CUDA(cudaMemsetAsync(out, 0, sizeof(uint64_t), ctx().stream));
    return;
  }
  const uint64_t nt = cdiv(n, 1024);
  DevBuf<uint64_t> sums(nt + 1);
  LB2_LAUNCH("storage_scan", scan_tiles_kernel, (unsigned)nt, 1024, 0, in, n, sums.p);
  LB2_LAUNCH("storage_scan", scan_sums_kernel, 1, 1024, 0, sums.p, nt);
  LB2_LAUNCH("storage_scan", scan_apply_kernel, (unsigned)nt, 1024, 0, in, n, sums.p, out);
}

// per partition: level_offsets (lo[p][l + 1] - lo[p][l] = nodes with more than l levels) and its batch's rows
__global__ void graph_level_offsets_kernel(const uint8_t* __restrict__ nlev, const uint64_t* __restrict__ off, int L,
                                           uint64_t* __restrict__ lo, uint64_t* __restrict__ rows) {
  __shared__ unsigned long long hist[64];
  const int p = blockIdx.x;
  for (int l = threadIdx.x; l < L; l += blockDim.x) hist[l] = 0;
  __syncthreads();
  for (uint64_t r = off[p] + threadIdx.x; r < off[p + 1]; r += blockDim.x) atomicAdd(&hist[nlev[r] - 1], 1ull);
  __syncthreads();
  if (threadIdx.x == 0) {
    uint64_t at_least = 0;  // nodes with more than l levels, from the top down
    for (int l = L - 1; l >= 0; --l) {
      at_least += hist[l];
      hist[l] = at_least;
    }
    uint64_t acc = 0;
    uint64_t* o = lo + (uint64_t)p * (L + 1);
    for (int l = 0; l < L; ++l) {
      o[l] = acc;
      acc += hist[l];
    }
    o[L] = acc;
    rows[p] = acc;
  }
}

// per partition, in tiles of nodes: the rank of each (node, level) among the level's nodes -> its row of the batches
// (gb[p] + lo[p][l] + rank): the node id, the list length and where the list lives in the dense layout
__global__ void graph_rows_kernel(GraphDev g, const uint64_t* __restrict__ off, const uint64_t* __restrict__ gb,
                                  const uint64_t* __restrict__ lo, uint64_t n, uint32_t* __restrict__ vid,
                                  uint64_t* __restrict__ len, uint64_t* __restrict__ slot) {
  __shared__ uint64_t ws[32];
  __shared__ uint64_t run[64];
  const int p = blockIdx.x, L = g.max_level;
  const uint64_t o = off[p], np = off[p + 1] - o;
  const uint64_t* lp = lo + (uint64_t)p * (L + 1);
  for (int l = threadIdx.x; l < L; l += blockDim.x) run[l] = 0;
  __syncthreads();
  for (uint64_t base = 0; base < np; base += blockDim.x) {
    const uint64_t i = base + threadIdx.x;
    const int lv = i < np ? g.nlev[o + i] : 0;
    for (int l = 0; l < L; ++l) {
      uint64_t t;
      // run[l] is read only after the scan's barriers: thread 0 wrote it after the previous tile's last barrier, and
      // with max_level 1 no other barrier lies between that write and this read
      const uint64_t e = block_exclusive_scan(lv > l ? 1 : 0, ws, &t);
      const uint64_t rank = run[l] + e;
      if (lv > l) {
        const uint64_t gr = gb[p] + lp[l] + rank, r = o + i;
        vid[gr] = (uint32_t)i;
        len[gr] = *list_of(g, r, l).cnt;
        slot[gr] = l == 0 ? r : n + g.up_base[r] + (l - 1);
      }
      __syncthreads();
      if (threadIdx.x == 0) run[l] += t;
    }
  }
}

// one warp per batch row: its list, in ranked order, from the dense layout to the concatenated list values
__global__ void graph_edges_out_kernel(GraphDev g, uint64_t rows, const uint64_t* __restrict__ slot, uint64_t n,
                                       const uint64_t* __restrict__ loff, uint32_t* __restrict__ nbr,
                                       float* __restrict__ dst) {
  const uint64_t gr = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (gr >= rows) return;
  const uint64_t s = slot[gr], a = loff[gr], c = loff[gr + 1] - a;
  const uint32_t* sn = s < n ? g.nbr0 + s * 2 * g.m : g.nbru + (s - n) * g.m;
  const float* sd = s < n ? g.dst0 + s * 2 * g.m : g.dstu + (s - n) * g.m;
  for (uint64_t j = lane; j < c; j += 32) {
    if (nbr) nbr[a + j] = sn[j];
    if (dst) dst[a + j] = sd[j];
  }
}

__global__ void sum_counts_kernel(const uint32_t* __restrict__ a, uint64_t n, unsigned long long* __restrict__ out) {
  unsigned long long s = 0;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) s += a[i];
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0 && s) atomicAdd(out, s);
}

// The graphs as every partition's level batches back to back (include/lance_b200.h, lb2_index_storage).
// hnsw_storage_edges: the number of list entries.  hnsw_to_storage: every output a device pointer or NULL;
// level_offsets [K][max_level + 1], vector_id [rows], list_offsets [rows + 1] (global), neighbors / distances [edges],
// rows = n + g.n_up.
uint64_t hnsw_storage_edges(const HnswGraph& g, uint64_t n) {
  DevBuf<unsigned long long> e(1);
  e.zero();
  const unsigned grid = (unsigned)std::max<uint64_t>(1, std::min<uint64_t>(cdiv(std::max(n, g.n_up), 256), 1024));
  if (n) LB2_LAUNCH("hnsw_to_storage", sum_counts_kernel, grid, 256, 0, g.cnt0.p, n, e.p);
  if (g.n_up) LB2_LAUNCH("hnsw_to_storage", sum_counts_kernel, grid, 256, 0, g.cntu.p, g.n_up, e.p);
  unsigned long long h = 0;
  d2h(&h, e.p, 1);
  sync_stream();
  return h;
}

void hnsw_to_storage(const HnswGraph& g, const uint64_t* part_offsets, int K, uint64_t n, uint64_t* level_offsets,
                     uint32_t* vector_id, uint64_t* list_offsets, uint32_t* neighbors, float* distances) {
  const int L = g.max_level;
  const uint64_t rows = n + g.n_up;
  DevBuf<uint64_t> lo((size_t)K * (L + 1)), prow(K), gb(K + 1), len(std::max<uint64_t>(rows, 1)),
      slot(std::max<uint64_t>(rows, 1)), loff(rows + 1);
  DevBuf<uint32_t> vid(std::max<uint64_t>(rows, 1));
  LB2_LAUNCH("hnsw_to_storage", graph_level_offsets_kernel, K, 256, 0, g.nlev.p, part_offsets, L, lo.p, prow.p);
  scan_u64(prow.p, K, gb.p);
  if (rows) LB2_LAUNCH("hnsw_to_storage", graph_rows_kernel, K, 1024, 0, dev_view(g), part_offsets, gb.p, lo.p, n,
                       vid.p, len.p, slot.p);
  scan_u64(len.p, rows, loff.p);
  if (rows && (neighbors || distances))
    LB2_LAUNCH("hnsw_to_storage", graph_edges_out_kernel, cdiv(rows * 32, 256), 256, 0, dev_view(g), rows, slot.p, n,
               loff.p, neighbors, distances);
  cudaStream_t st = ctx().stream;
  if (level_offsets) LB2_CUDA(cudaMemcpyAsync(level_offsets, lo.p, 8 * lo.n, cudaMemcpyDeviceToDevice, st));
  if (vector_id && rows) LB2_CUDA(cudaMemcpyAsync(vector_id, vid.p, 4 * rows, cudaMemcpyDeviceToDevice, st));
  if (list_offsets) LB2_CUDA(cudaMemcpyAsync(list_offsets, loff.p, 8 * (rows + 1), cudaMemcpyDeviceToDevice, st));
  sync_stream();
}

// the checks of hnsw_from_storage, in the order they are reported
enum : uint32_t {
  SE_LEVEL_OFFSETS = 1, SE_LEVEL0, SE_ENTRY, SE_VECTOR_ID, SE_ASCENDING, SE_LIST_OFFSETS, SE_DEGREE, SE_GAP
};
__device__ __forceinline__ void storage_error(uint64_t* err, uint32_t code, uint64_t where) {
  if (atomicCAS(reinterpret_cast<unsigned long long*>(err), 0ull, (unsigned long long)code) == 0) err[1] = where;
}

// per partition: level_offsets start at 0 and ascend by at most n_p per level, level 0 holds every row of the
// partition, the entry point is node 0; rows[p] = the batch's rows
__global__ void storage_check_parts_kernel(const uint64_t* __restrict__ off, int K, int L, const uint64_t* __restrict__ lo,
                                           const uint32_t* __restrict__ entry, uint64_t* __restrict__ rows,
                                           uint64_t* __restrict__ err) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= K) return;
  const uint64_t* o = lo + (uint64_t)p * (L + 1);
  const uint64_t np = off[p + 1] - off[p];
  bool mono = o[0] == 0;
  for (int l = 0; l < L; ++l) mono = mono && o[l + 1] >= o[l] && o[l + 1] - o[l] <= np;
  if (!mono) storage_error(err, SE_LEVEL_OFFSETS, p);
  else if (o[1] != np) storage_error(err, SE_LEVEL0, p);
  if (entry[p] != 0) storage_error(err, SE_ENTRY, p);
  rows[p] = mono ? o[L] : 0;
}

// the partition p and level l of batch row gr, and its position i in the level
struct BatchRow {
  int p, l;
  uint64_t i;
};
__device__ __forceinline__ BatchRow batch_row(const uint64_t* gb, int K, const uint64_t* lo, int L, uint64_t gr) {
  BatchRow b;
  b.p = segment_of(gb, K, gr);
  const uint64_t* o = lo + (uint64_t)b.p * (L + 1);
  const uint64_t t = gr - gb[b.p];
  b.l = segment_of(o, L, t);
  b.i = t - o[b.l];
  return b;
}

// one thread per batch row: the id is a node of the partition, ascending in its level; the list offsets ascend and
// the list fits the level's degree; the node's level mask gains bit l
__global__ void storage_check_rows_kernel(const uint64_t* __restrict__ off, int K, const uint64_t* __restrict__ gb,
                                          const uint64_t* __restrict__ lo, int L, int m, uint64_t rows,
                                          const uint32_t* __restrict__ vid, const uint64_t* __restrict__ loff,
                                          unsigned long long* __restrict__ mask, uint64_t* __restrict__ err) {
  const uint64_t gr = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (gr >= rows) return;
  const BatchRow b = batch_row(gb, K, lo, L, gr);
  const uint64_t np = off[b.p + 1] - off[b.p];
  const uint32_t v = vid[gr];
  if (v >= np) { storage_error(err, SE_VECTOR_ID, gr); return; }
  if (b.i > 0 && vid[gr - 1] >= v) { storage_error(err, SE_ASCENDING, gr); return; }
  if (loff[gr + 1] < loff[gr]) { storage_error(err, SE_LIST_OFFSETS, gr); return; }
  if (loff[gr + 1] - loff[gr] > (uint64_t)(b.l == 0 ? 2 * m : m)) { storage_error(err, SE_DEGREE, gr); return; }
  atomicOr(&mask[off[b.p] + v], 1ull << b.l);
}

// one thread per node: its levels are 0 .. L - 1 without a gap -> nlev, and its L - 1 upper rows
__global__ void storage_node_levels_kernel(const unsigned long long* __restrict__ mask, uint64_t n,
                                           uint8_t* __restrict__ nlev, uint64_t* __restrict__ nup,
                                           uint64_t* __restrict__ err) {
  const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const unsigned long long k = mask[r];
  if (k == 0 || (k & (k + 1)) != 0) storage_error(err, SE_GAP, r);
  const int L = __popcll(k);
  nlev[r] = (uint8_t)L;
  nup[r] = L ? L - 1 : 0;
}

// one warp per batch row: its list into the dense layout (level 0 row r, upper row up[r] + l - 1)
__global__ void storage_edges_in_kernel(const uint64_t* __restrict__ off, int K, const uint64_t* __restrict__ gb,
                                        const uint64_t* __restrict__ lo, int L, int m, uint64_t rows,
                                        const uint32_t* __restrict__ vid, const uint64_t* __restrict__ loff,
                                        const uint32_t* __restrict__ nbr, const float* __restrict__ dst,
                                        const uint64_t* __restrict__ up, uint32_t* __restrict__ cnt0,
                                        uint32_t* __restrict__ nbr0, float* __restrict__ dst0,
                                        uint32_t* __restrict__ cntu, uint32_t* __restrict__ nbru,
                                        float* __restrict__ dstu) {
  const uint64_t gr = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (gr >= rows) return;
  const BatchRow b = batch_row(gb, K, lo, L, gr);
  const uint64_t r = off[b.p] + vid[gr], a = loff[gr], c = loff[gr + 1] - a;
  uint32_t* on;
  float* od;
  if (b.l == 0) {
    on = nbr0 + r * 2 * m;
    od = dst0 + r * 2 * m;
    if (lane == 0) cnt0[r] = (uint32_t)c;
  } else {
    const uint64_t u = up[r] + (b.l - 1);
    on = nbru + u * m;
    od = dstu + u * m;
    if (lane == 0) cntu[u] = (uint32_t)c;
  }
  for (uint64_t j = lane; j < c; j += 32) {
    on[j] = nbr[a + j];
    od[j] = dst[a + j];
  }
}

// the inverse into g (its parameters set by the caller; device inputs): the storage checks on the device, then
// hnsw_load of the dense layout.  LB2_INVALID_ARG on malformed input, before g is filled.
void hnsw_from_storage(HnswGraph& g, const uint64_t* part_offsets, int K, uint64_t n, const uint32_t* entry_point,
                       const uint64_t* level_offsets, const uint32_t* vector_id, const uint64_t* list_offsets,
                       const uint32_t* neighbors, const float* distances, uint64_t rows, uint64_t edges) {
  const int L = g.max_level, m = g.m;
  DevBuf<uint64_t> err(2), prow(K), gb(K + 1), nup(std::max<uint64_t>(n, 1)), up(n + 1);
  err.zero();
  LB2_LAUNCH("hnsw_from_storage", storage_check_parts_kernel, cdiv(K, 256), 256, 0, part_offsets, K, L, level_offsets,
             entry_point, prow.p, err.p);
  scan_u64(prow.p, K, gb.p);
  uint64_t h[3], e[2];
  d2h(h, gb.p + K, 1);
  d2h(h + 1, list_offsets, 1);
  d2h(h + 2, list_offsets + rows, 1);
  d2h(e, err.p, 2);
  sync_stream();
  auto report = [&](uint64_t code, uint64_t at) {
    switch (code) {
      case SE_LEVEL_OFFSETS: fail(LB2_INVALID_ARG, "%s: level_offsets of partition %llu do not start at 0 and ascend by at most the partition's rows per level", g.kind, (unsigned long long)at);
      case SE_LEVEL0: fail(LB2_INVALID_ARG, "%s: level 0 of partition %llu does not hold every row of the partition", g.kind, (unsigned long long)at);
      case SE_ENTRY: fail(LB2_INVALID_ARG, "%s: the entry point of partition %llu is not node 0", g.kind, (unsigned long long)at);
      case SE_VECTOR_ID: fail(LB2_INVALID_ARG, "%s: __vector_id of batch row %llu is not a node of its partition", g.kind, (unsigned long long)at);
      case SE_ASCENDING: fail(LB2_INVALID_ARG, "%s: __vector_id of batch row %llu does not ascend within its level", g.kind, (unsigned long long)at);
      case SE_LIST_OFFSETS: fail(LB2_INVALID_ARG, "%s: the list offsets of batch row %llu descend", g.kind, (unsigned long long)at);
      case SE_DEGREE: fail(LB2_INVALID_ARG, "%s: batch row %llu has more neighbours than its level allows (2m at level 0, m above)", g.kind, (unsigned long long)at);
      case SE_GAP: fail(LB2_INVALID_ARG, "%s: row %llu is present at a level but absent at the level below", g.kind, (unsigned long long)at);
    }
  };
  report(e[0], e[1]);
  LB2_REQUIRE(h[0] == rows, "%s: level_offsets give %llu batch rows, the storage has %llu", g.kind,
              (unsigned long long)h[0], (unsigned long long)rows);
  LB2_REQUIRE(h[1] == 0 && h[2] == edges, "%s: the list offsets run from %llu to %llu, not from 0 to the %llu edges",
              g.kind, (unsigned long long)h[1], (unsigned long long)h[2], (unsigned long long)edges);
  DevBuf<unsigned long long> mask(std::max<uint64_t>(n, 1));
  DevBuf<uint8_t> nlev(std::max<uint64_t>(n, 1));
  mask.zero();
  if (rows)
    LB2_LAUNCH("hnsw_from_storage", storage_check_rows_kernel, cdiv(rows, 256), 256, 0, part_offsets, K, gb.p,
               level_offsets, L, m, rows, vector_id, list_offsets, mask.p, err.p);
  if (n) LB2_LAUNCH("hnsw_from_storage", storage_node_levels_kernel, cdiv(n, 256), 256, 0, mask.p, n, nlev.p, nup.p, err.p);
  d2h(e, err.p, 2);
  sync_stream();
  report(e[0], e[1]);
  scan_u64(nup.p, n, up.p);
  uint64_t n_up = 0;
  d2h(&n_up, up.p + n, 1);
  sync_stream();
  DevBuf<uint32_t> cnt0(std::max<uint64_t>(n, 1)), nbr0(std::max<uint64_t>(n * 2 * m, 1)),
      cntu(std::max<uint64_t>(n_up, 1)), nbru(std::max<uint64_t>(n_up * m, 1));
  DevBuf<float> dst0(std::max<uint64_t>(n * 2 * m, 1)), dstu(std::max<uint64_t>(n_up * m, 1));
  cnt0.zero(); nbr0.zero(); dst0.zero(); cntu.zero(); nbru.zero(); dstu.zero();
  if (rows)
    LB2_LAUNCH("hnsw_from_storage", storage_edges_in_kernel, cdiv(rows * 32, 256), 256, 0, part_offsets, K, gb.p,
               level_offsets, L, m, rows, vector_id, list_offsets, neighbors, distances, up.p, cnt0.p, nbr0.p, dst0.p,
               cntu.p, nbru.p, dstu.p);
  // the neighbour checks and the attachment are lb2_index_load_hnsw_*'s
  hnsw_load(g, part_offsets, K, nlev.p, cnt0.p, nbr0.p, dst0.p, cntu.p, nbru.p, dstu.p);
}

}  // namespace
}  // namespace lb2

using namespace lb2;

__global__ void part_lengths_kernel(const uint64_t* __restrict__ off, int K, uint64_t* __restrict__ len) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p < K) len[p] = off[p + 1] - off[p];
}
// a length above n would let the u64 sum of the lengths wrap to n with offsets that are not ascending
__global__ void lengths_above_kernel(const uint64_t* __restrict__ len, int K, uint64_t n, uint32_t* __restrict__ bad) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p < K && len[p] > n) atomicMax(bad, (uint32_t)p + 1);
}
__global__ void part_ids_kernel(const uint64_t* __restrict__ off, int K, uint64_t n, uint32_t* __restrict__ part) {
  const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r < n) part[r] = (uint32_t)segment_of(off, K, r);
}
// u8 IVF_FLAT rows are held as f32; the reference's u8 flat storage is the Hamming one (include/lance_b200.h)
static void storage_kind_check(const lb2_index* index, const char* what) {
  LB2_REQUIRE(!(index->kind == IndexKind::FLAT && index->dtype == LB2_U8),
              "%s: an IVF_FLAT index over u8 rows has no storage layout (the reference stores u8 columns only in its "
              "binary Hamming storage)", what);
}

extern "C" {

lb2_status lb2_index_export_partition(const lb2_index* index, uint32_t partition, uint8_t* codes_transposed_out,
                                      uint64_t* row_ids_out, uint64_t* num_rows_out) {
  LB2_API_BEGIN
  LB2_REQUIRE(index && index->kind == IndexKind::PQ, "not an IVF_PQ index");
  LB2_REQUIRE(partition < (uint32_t)index->K, "partition %u out of range (the index has %d)", partition, index->K);
  uint64_t off[2];
  d2h(off, index->part_offsets.p + partition, 2);
  sync_stream();
  const uint64_t np = off[1] - off[0];
  const int cw = (int)index->row_bytes();
  if (num_rows_out) *num_rows_out = np;
  if (np && codes_transposed_out) {
    OutArg<uint8_t> o(codes_transposed_out, (size_t)np * cw);
    transpose_codes(index->codes.p + off[0] * cw, index->part_offsets.p + partition, 1, cw, np, false, o.get());
    o.commit();
  }
  if (np && row_ids_out)
    LB2_CUDA(cudaMemcpyAsync(row_ids_out, index->row_ids.p + off[0], sizeof(uint64_t) * np, cudaMemcpyDefault, ctx().stream));
  sync_stream();
  LB2_API_END
}

lb2_status lb2_index_export_storage(const lb2_index* index, lb2_index_storage* out) {
  LB2_API_BEGIN
  LB2_REQUIRE(index && out, "null argument");
  storage_kind_check(index, "index_export_storage");
  const uint64_t n = index->n;
  const int K = index->K;
  const size_t rb = index->row_bytes();
  const HnswGraph* g = index->hnsw.get();
  out->num_partitions = (uint32_t)K;
  out->num_rows = n;
  out->num_bytes = n * rb;
  out->max_level = g ? (uint32_t)g->max_level : 0;
  out->m = g ? (uint32_t)g->m : 0;
  out->ef_construction = g ? (uint32_t)g->ef_construction : 0;
  out->num_graph_rows = g ? n + g->n_up : 0;
  out->num_edges = g ? hnsw_storage_edges(*g, n) : 0;
  cudaStream_t s = ctx().stream;
  const uint64_t* off = index->part_offsets.p;
  OutArg<uint64_t> len(out->part_lengths, K);
  if (len.get()) LB2_LAUNCH("storage_export", part_lengths_kernel, cdiv(K, 256), 256, 0, off, K, len.get());
  len.commit();
  if (out->row_ids && n)
    LB2_CUDA(cudaMemcpyAsync(out->row_ids, index->row_ids.p, sizeof(uint64_t) * n, cudaMemcpyDefault, s));
  OutArg<uint8_t> pay(out->payload, n * rb);
  if (pay.get()) {
    if (index->kind == IndexKind::PQ) transpose_codes(index->codes.p, off, K, (int)rb, n, false, pay.get());
    else if (index->kind == IndexKind::RQ) rq_pack(index->codes.p, off, K, n, (int)rb, pay.get(), false);
    else d2d(pay.get(), index->payload().p, n * rb);
  }
  pay.commit();
  if (index->kind == IndexKind::RQ && n) {
    if (out->add_factors)
      LB2_CUDA(cudaMemcpyAsync(out->add_factors, index->rq_add.p, sizeof(float) * n, cudaMemcpyDefault, s));
    if (out->scale_factors)
      LB2_CUDA(cudaMemcpyAsync(out->scale_factors, index->rq_scale.p, sizeof(float) * n, cudaMemcpyDefault, s));
  }
  if (g) {
    const uint64_t rows = out->num_graph_rows, e = out->num_edges;
    OutArg<uint32_t> ep(out->entry_point, K);
    if (ep.get()) LB2_CUDA(cudaMemsetAsync(ep.get(), 0, sizeof(uint32_t) * K, s));
    ep.commit();
    OutArg<uint64_t> lo(out->level_offsets, (size_t)K * (g->max_level + 1)), lof(out->list_offsets, rows + 1);
    OutArg<uint32_t> vid(out->vector_id, rows), nbr(out->neighbors, e);
    OutArg<float> dst(out->distances, e);
    if (lo.get() || vid.get() || lof.get() || nbr.get() || dst.get())
      hnsw_to_storage(*g, off, K, n, lo.get(), vid.get(), lof.get(), nbr.get(), dst.get());
    lo.commit(); lof.commit(); vid.commit(); nbr.commit(); dst.commit();
    sync_stream();
  }
  sync_stream();
  LB2_API_END
}

lb2_status lb2_index_load_storage(lb2_index* index, const lb2_index_storage* st) {
  LB2_API_BEGIN
  LB2_REQUIRE(index && st, "null argument");
  storage_kind_check(index, "index_load_storage");
  const int K = index->K;
  const uint64_t n = st->num_rows;
  const size_t rb = index->row_bytes();
  const bool rq = index->kind == IndexKind::RQ;
  LB2_REQUIRE(st->num_partitions == (uint32_t)K, "index_load_storage: %u partitions, the index has %d",
              st->num_partitions, K);
  LB2_REQUIRE(n < 0xffffffffull, "more than 2^32-1 rows per index shard");
  LB2_REQUIRE(st->num_bytes == n * rb, "index_load_storage: %llu payload bytes, %llu rows of %zu bytes need %llu",
              (unsigned long long)st->num_bytes, (unsigned long long)n, rb, (unsigned long long)(n * rb));
  LB2_REQUIRE(st->part_lengths && (n == 0 || (st->payload && st->row_ids)), "null argument");
  LB2_REQUIRE(rq ? n == 0 || (st->add_factors && st->scale_factors) : !st->add_factors && !st->scale_factors,
              "index_load_storage: add / scale factors are IVF_RQ's columns, required there and only there");
  LB2_REQUIRE(st->max_level == 0 || !rq, "index_load_storage: IVF_RQ has no graph");
  if (index->kind == IndexKind::FLAT)
    LB2_REQUIRE(index->d % 4 == 0, "IVF_FLAT needs a dimension that is a multiple of 4");
  InArg<uint64_t> len(st->part_lengths, K);
  std::unique_ptr<lb2_index> ix = make_index(index->kind, K, index->d, index->metric, index->dtype);
  copy_model(index, ix.get());
  DevBuf<uint64_t> off(K + 1);
  DevBuf<uint32_t> bad(1);
  bad.zero();
  LB2_LAUNCH("storage_load", lengths_above_kernel, cdiv(K, 256), 256, 0, len.get(), K, n, bad.p);
  scan_u64(len.get(), K, off.p);
  uint64_t total = 0;
  uint32_t above = 0;
  d2h(&total, off.p + K, 1);
  d2h(&above, bad.p, 1);
  sync_stream();
  LB2_REQUIRE(above == 0, "index_load_storage: part_lengths[%u] is above num_rows %llu", above - 1,
              (unsigned long long)n);
  LB2_REQUIRE(total == n, "index_load_storage: part_lengths sum to %llu, num_rows is %llu", (unsigned long long)total,
              (unsigned long long)n);
  // the rows in partition order with their partition ids: the loads' own grouping keeps that order
  DevBuf<uint32_t> part(std::max<uint64_t>(n, 1));
  if (n) LB2_LAUNCH("storage_load", part_ids_kernel, cdiv(n, 256), 256, 0, off.p, K, n, part.p);
  InArg<uint64_t> rid(st->row_ids, n);
  if (index->kind == IndexKind::FLAT) {
    Source src(st->payload, n, index->d, index->dtype);
    src.start_resident_copy();
    index_load_flat_src(ix.get(), part.p, src, rid.get(), nullptr, /*normalize=*/false);
  } else {
    InArg<uint8_t> pay(st->payload, n * rb);
    InArg<float> a(st->add_factors, n), sc(st->scale_factors, n);
    DevBuf<uint8_t> rows;
    const uint8_t* codes = pay.get();
    if (index->kind != IndexKind::SQ && n) {
      rows.alloc(n * rb);
      if (rq) rq_pack(pay.get(), off.p, K, n, (int)rb, rows.p, true);
      else transpose_codes(pay.get(), off.p, K, (int)rb, n, true, rows.p);
      codes = rows.p;
    }
    index_load_dev(ix.get(), part.p, codes, rid.get(), n, nullptr, a.get(), sc.get());
  }
  if (st->max_level) {
    const uint64_t rows = st->num_graph_rows, e = st->num_edges;
    std::unique_ptr<HnswGraph> g = new_graph(index->kind, st->max_level, st->m, st->ef_construction);
    LB2_REQUIRE(st->entry_point && st->level_offsets && st->list_offsets && (rows == 0 || st->vector_id) &&
                    (e == 0 || (st->neighbors && st->distances)),
                "null argument");
    InArg<uint32_t> ep(st->entry_point, K), vid(st->vector_id, rows), nbr(st->neighbors, e);
    InArg<uint64_t> lo(st->level_offsets, (size_t)K * (st->max_level + 1)), lof(st->list_offsets, rows + 1);
    InArg<float> dst(st->distances, e);
    hnsw_from_storage(*g, ix->part_offsets.p, K, n, ep.get(), lo.get(), vid.get(), lof.get(), nbr.get(), dst.get(),
                      rows, e);
    ix->hnsw = std::move(g);
  }
  sync_stream();
  ix->pi_mode = index->pi_mode;  // the centroids are unchanged, so the partition rule and its graph carry over
  ix->pi_seed = index->pi_seed;
  ix->pi_batch = index->pi_batch;
  ix->pidx = std::move(index->pidx);
  *index = std::move(*ix);
  LB2_API_END
}

}  // extern "C"
