// split.cu -- the partition split and join of an optimize, on the device (SURVEY 8f-4): which partition to split or
// join, its reassign candidates, k = 2 training, every row's decision, the moved rows' payload and the merge.
//
// Replaces  IvfIndexBuilder::should_split / split_partition_impl   rust/lance/src/index/vector/builder.rs:1152-1333
//           IvfIndexBuilder::should_join / join_partition_impl     builder.rs:1343-1530
//           assign_vectors / reassign_vectors                      builder.rs:1690-1785
//           select_reassign_candidates_impl                        builder.rs:1788-1814
//           build_assign_batch (the moved rows' transform)         builder.rs:1534-1650
// The host keeps what only it can do: loading a partition's raw rows by row id (load_partition_raw_vectors,
// builder.rs:1118-1147).
#include <algorithm>
#include <memory>
#include <vector>

#include "build.cuh"
#include "comm.cuh"
#include "index.cuh"
#include "kmeans.cuh"
#include "probe.cuh"
#include "row_distance.cuh"

namespace lb2 {
namespace {

constexpr uint32_t NONE = 0xffffffffu;
constexpr uint64_t NONE64 = ~0ull;
constexpr int REASSIGN_RANGE = 64;           // builder.rs:60
constexpr uint64_t MAX_PARTITION_SIZE_FACTOR = 4;   // lance-index/src/lib.rs:52
constexpr uint64_t MIN_PARTITION_SIZE_PERCENT = 25;
constexpr int DECIDE_WARPS = 8;

// IndexType::target_partition_size (lance-index/src/lib.rs:284-295)
uint64_t target_partition_size(const lb2_index* ix) {
  if (ix->hnsw) return 1024 * 1024;
  return ix->kind == IndexKind::FLAT ? 4096 : 8192;
}

void check_kind(const lb2_index* ix, const char* what) {
  if (comm_nranks() > 1) fail(LB2_UNSUPPORTED, "%s: an index over more than one rank is not implemented", what);
  // arrow_batch_func dispatches on the f32 model centroid and cannot downcast u8 rows to it (l2.rs:205-231,
  // cosine.rs:315-336, dot.rs:218-240): the reference cannot split or join a u8 column
  if (ix->dtype == LB2_U8) fail(LB2_UNSUPPORTED, "%s: the reference's distances cannot take u8 rows", what);
}

__device__ __forceinline__ int part_of_pos(const uint64_t* __restrict__ offsets, int K, uint64_t i) {
  int lo = 0, hi = K;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (offsets[mid] <= i) lo = mid; else hi = mid;
  }
  return lo;
}

// ---- the rule of one (from, to) distance, as lb2_distance_batch computes it ------------------------------------
// COSINE: the warp's cos32 sums; 16-bit dot: DOT32; everything else (f32, 16-bit L2): LANES16.  LANES16 and DOT32 are
// symmetric in their operands, cosine is not (the norm of `from` is taken first).
template <int METRIC, class T>
constexpr int batch_rule() {
  return METRIC == METRIC_COSINE ? RULE_COSINE
         : (METRIC == METRIC_DOT && !std::is_same<T, float>::value) ? RULE_DOT32
                                                                     : RULE_LANES16;
}

// One warp per row.  Centroid table slots: 0 = c0 (the split partition's old centroid), 1 = c1, 2 = c2, 3 + j = the
// old centroid of candidate j.  Rows [0, n_a) are the split (or joined) partition's, rows [n_a, n_a + n_b) the
// candidate partitions' (cand_rank[cand_part[i]] = j).
//   split row:     d0 / d1 / d2 = batch(c, row); d0 <= d1 && d0 <= d2 -> reassign_vectors(Some(d1, d2)) over
//                  batch(row, candidates): the first minimum by total_cmp goes if it is <= d1 and <= d2; otherwise
//                  c1 when d1 <= d2, else c2 (assign_vectors with deleted_original_partition = true, :1690-1749)
//   candidate row: d0 = batch(own centroid, row); d0 minimal -> stays (NONE); otherwise c1 / c2 as above
//   join row:      the first minimum over the candidates (:1476-1530), ids above `part` shifted down by one
// A row with a non-finite element, or a zero row under cosine, is one the transform would drop: bad[0].
// Each row is read from memory once, into the warp's f32 row buffer (the conversion is exact).  The few distances of
// c0 / c1 / c2 and a candidate row's own centroid take a half-warp each (row_distance), the two halves on two
// centroids at once; the candidate scan of a split or join row takes one lane per candidate (thread_distance,
// cos32_sum_thread), the table's slots padded to a stride of d + 1 floats so that the 32 lanes read 32 banks.
struct DecideArgs {
  const void* rows_a;
  uint64_t n_a;
  const void* rows_b;
  uint64_t n_b;
  int d, ld;  // ld: the table's slot stride in shared memory
  const uint32_t* cand_part;
  const uint32_t* cand_rank;
  const float* table;
  int S, chunk;
  const uint32_t* cand_ids;
  uint32_t part, k_old;
  int join;
  uint32_t* dest;
  uint32_t* bad;
};

struct RowState {
  bool live = false, ok = false, split_row = false, want_cand = false;
  int own = 0;
  float rr = 0.0f;  // <row, row> (cosine)
};

// row i into the warp's buffer xr, its kind, and whether the transform would keep it
template <int RULE, class T>
__device__ __forceinline__ RowState row_begin(const DecideArgs& a, uint64_t i, float* xr, int lane) {
  RowState st;
  st.live = true;
  const T* row = i < a.n_a ? static_cast<const T*>(a.rows_a) + i * a.d
                           : static_cast<const T*>(a.rows_b) + (i - a.n_a) * a.d;
  st.split_row = i < a.n_a && !a.join;
  if (i >= a.n_a) {
    const uint32_t r = a.cand_rank[a.cand_part[i - a.n_a]];
    st.own = r == NONE ? -1 : 3 + (int)r;
  }
  bool ok = st.own >= 0;
  for (int e = lane; e < a.d; e += 32) {
    const float v = ldf<T>(row, e);
    xr[e] = v;
    ok = ok && isfinite(v);
  }
  ok = __all_sync(0xffffffffu, ok);
  if constexpr (RULE == RULE_COSINE) {
    st.rr = cos32_sum(row, row, a.d, lane);
    ok = ok && st.rr != 0.0f;
  }
  if (!ok && lane == 0) atomicOr(a.bad, 1u);
  st.ok = ok;
  st.want_cand = ok && a.join;
  __syncwarp();
  return st;
}

// batch(c, row) for up to 3 slots (list; the distances go to wd[out[t]]): under the 16-lane rules two slots at a time,
// one per half-warp; under cosine one slot at a time on the whole warp
template <int RULE, int METRIC>
__device__ __forceinline__ void few_distances(const DecideArgs& a, const RowState& st, const float* tab, const float* cn,
                                              int s0, const float* xr, const int* list, const int* out, int cnt,
                                              float* wd, int lane) {
  if constexpr (RULE == RULE_COSINE) {
    for (int t = 0; t < cnt; ++t) {
      const int c = list[t] - s0;
      const float v = cos32_finish(cos32_sum(tab + (size_t)c * a.ld, xr, a.d, lane), cn[c], st.rr);
      if (lane == 0) wd[out[t]] = v;
    }
  } else {
    const int l = lane & 15, half = lane >> 4;
    const unsigned hmask = 0xffffu << (16 * half);
    for (int r = 0; r < cnt; r += 2) {
      const int t = min(r + half, cnt - 1);  // an idle half repeats its partner's slot and writes nothing
      const float v = row_distance<RULE, METRIC, float>(tab + (size_t)(list[t] - s0) * a.ld, xr, a.d, l, hmask, 0.0f);
      if (l == 0 && r + half < cnt) wd[out[t]] = v;
    }
  }
}

// the distances one row needs from table slots [s0, s0 + cs) (tab: those slots, cn: their <c, c> under cosine)
template <int RULE, int METRIC>
__device__ __forceinline__ void row_chunk(const DecideArgs& a, RowState& st, const float* tab, const float* cn,
                                          int s0, int cs, const float* xr, float* wd, int lane) {
  const int d = a.d;
  if (s0 == 0 && st.split_row) {  // d0, d1, d2: slots 0..2 are in the first chunk (chunk >= 3)
    const int list[3] = {0, 1, 2};
    few_distances<RULE, METRIC>(a, st, tab, cn, 0, xr, list, list, 3, wd, lane);
    __syncwarp();
    st.want_cand = wd[0] <= wd[1] && wd[0] <= wd[2];
  }
  if (st.split_row || a.join) {
    if (!st.want_cand) return;
    for (int c = max(3 - s0, 0) + lane; c < cs; c += 32) {  // batch(row, candidate), one lane per candidate
      const float* cv = tab + (size_t)c * a.ld;
      float v;
      if constexpr (RULE == RULE_COSINE) v = cos32_finish(cos32_sum_thread(xr, cv, d), st.rr, cn[c]);
      else v = thread_distance<RULE, METRIC, float>(cv, xr, d);
      wd[s0 + c] = v;
    }
    return;
  }
  int list[3], out[3], cnt = 0;  // a candidate row: batch(c, row) for c1, c2 and its own centroid
  const int want[3] = {1, 2, st.own}, slot[3] = {1, 2, 0};
  for (int t = 0; t < 3; ++t)
    if (want[t] >= s0 && want[t] < s0 + cs) {
      list[cnt] = want[t];
      out[cnt++] = slot[t];
    }
  few_distances<RULE, METRIC>(a, st, tab, cn, s0, xr, list, out, cnt, wd, lane);
}

__device__ __forceinline__ void row_end(const DecideArgs& a, const RowState& st, const float* wd, uint64_t i) {
  uint32_t out = NONE;
  if (!st.ok) {
  } else if (!st.split_row && !a.join) {
    const float d0 = wd[0], d1 = wd[1], d2 = wd[2];
    out = (d0 <= d1 && d0 <= d2) ? NONE : (d1 <= d2 ? a.part : a.k_old);
  } else {
    int best = -1;
    int32_t bk = 0;
    if (st.want_cand)
      for (int s = 3; s < a.S; ++s) {  // position_min_by(total_cmp): the first minimum
        const int32_t k = total_order_key(wd[s]);
        if (best < 0 || k < bk) { best = s; bk = k; }
      }
    if (a.join) {
      const uint32_t id = best < 0 ? NONE : a.cand_ids[best - 3];
      out = id == NONE ? NONE : (id > a.part ? id - 1 : id);
    } else {
      const float d1 = wd[1], d2 = wd[2];
      if (best >= 0 && wd[best] <= d1 && wd[best] <= d2) out = a.cand_ids[best - 3];
      else out = d1 <= d2 ? a.part : a.k_old;
    }
  }
  a.dest[i] = out;
}

// the table's slots [s0, s0 + cs) into shared memory at stride ld, and <c, c> of each under cosine
template <int RULE>
__device__ __forceinline__ void load_chunk(const DecideArgs& a, float* tab, float* cn, int s0, int cs, int w, int lane) {
  const int d = a.d;
  for (int t = threadIdx.x; t < cs * d; t += blockDim.x) tab[(size_t)(t / d) * a.ld + t % d] = a.table[(size_t)s0 * d + t];
  __syncthreads();
  if constexpr (RULE == RULE_COSINE) {
    for (int c = w; c < cs; c += DECIDE_WARPS) {
      const float v = cos32_sum(tab + (size_t)c * a.ld, tab + (size_t)c * a.ld, d, lane);
      if (lane == 0) cn[c] = v;
    }
    __syncthreads();
  }
}

// shared memory of the decision kernel: the table chunk [chunk][ld], <c, c> [chunk], per warp the distances
// [3 + REASSIGN_RANGE] and the row [d]
inline size_t decide_smem(int chunk, int d) {
  return sizeof(float) * ((size_t)chunk * (d + 1) + chunk + (size_t)DECIDE_WARPS * (3 + REASSIGN_RANGE + d));
}

// The whole table fits shared memory (S <= chunk): loaded once per block, the warps walk the rows grid-stride.
// Otherwise one row per warp, the table streamed through shared memory `chunk` slots at a time.
template <int METRIC, class T>
__global__ void __launch_bounds__(DECIDE_WARPS * 32) split_decide_kernel(DecideArgs a) {
  constexpr int RULE = batch_rule<METRIC, T>();
  extern __shared__ float sm[];
  float* tab = sm;
  float* cn = tab + (size_t)a.chunk * a.ld;
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* wd = cn + a.chunk + w * (3 + REASSIGN_RANGE);
  float* xr = cn + a.chunk + DECIDE_WARPS * (3 + REASSIGN_RANGE) + (size_t)w * a.d;
  const uint64_t n = a.n_a + a.n_b;
  if (a.S <= a.chunk) {
    load_chunk<RULE>(a, tab, cn, 0, a.S, w, lane);
    for (uint64_t i = (uint64_t)blockIdx.x * DECIDE_WARPS + w; i < n; i += (uint64_t)gridDim.x * DECIDE_WARPS) {
      RowState st = row_begin<RULE, T>(a, i, xr, lane);
      if (st.ok) row_chunk<RULE, METRIC>(a, st, tab, cn, 0, a.S, xr, wd, lane);
      __syncwarp();
      if (lane == 0) row_end(a, st, wd, i);
      __syncwarp();
    }
    return;
  }
  const uint64_t i = (uint64_t)blockIdx.x * DECIDE_WARPS + w;
  RowState st;
  if (i < n) st = row_begin<RULE, T>(a, i, xr, lane);
  for (int s0 = 0; s0 < a.S; s0 += a.chunk) {
    const int cs = min(a.chunk, a.S - s0);
    __syncthreads();
    load_chunk<RULE>(a, tab, cn, s0, cs, w, lane);
    if (st.ok) row_chunk<RULE, METRIC>(a, st, tab, cn, s0, cs, xr, wd, lane);
  }
  __syncwarp();
  if (st.live && lane == 0) row_end(a, st, wd, i);
}

// the raw rows' order: ids strictly ascending within a group, candidate groups in candidate order (bad[1])
__global__ void check_groups_kernel(const uint64_t* __restrict__ ids_a, uint64_t n_a, const uint64_t* __restrict__ ids_b,
                                    const uint32_t* __restrict__ part_b, const uint32_t* __restrict__ cand_rank,
                                    uint64_t n_b, uint32_t* __restrict__ bad) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i + 1 < n_a && ids_a[i] >= ids_a[i + 1]) atomicOr(bad + 1, 1u);
  if (i + 1 < n_b) {
    const uint32_t r0 = cand_rank[part_b[i]], r1 = cand_rank[part_b[i + 1]];
    if (r0 > r1 || (r0 == r1 && ids_b[i] >= ids_b[i + 1])) atomicOr(bad + 1, 1u);
  }
}

// ---- the rows of the partitions a split or join reads: an open-addressing set of (row id -> partition) ----------
__device__ __forceinline__ uint64_t hash_id(uint64_t x) {
  x ^= x >> 33;
  x *= 0xff51afd7ed558ccdull;
  x ^= x >> 33;
  return x;
}
__device__ __forceinline__ void rowset_insert(unsigned long long* __restrict__ keys, uint32_t* __restrict__ vals,
                                              uint64_t mask, unsigned long long id, uint32_t p) {
  for (uint64_t h = hash_id(id) & mask;; h = (h + 1) & mask) {
    const unsigned long long prev = atomicCAS(&keys[h], (unsigned long long)NONE64, id);
    if (prev == NONE64) { vals[h] = p; return; }
    if (prev == id) return;
  }
}
// the stored rows of the involved partitions: segment j is seg_part[j]'s rows, storage positions seg_start[j] ..,
// rows seg_prefix[j] .. seg_prefix[j + 1] of the launch
__global__ void rowset_insert_old_kernel(unsigned long long* __restrict__ keys, uint32_t* __restrict__ vals,
                                         uint64_t mask, const uint64_t* __restrict__ row_ids,
                                         const uint64_t* __restrict__ seg_prefix, const uint64_t* __restrict__ seg_start,
                                         const uint32_t* __restrict__ seg_part, int nseg) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= seg_prefix[nseg]) return;
  const int j = part_of_pos(seg_prefix, nseg, i);
  rowset_insert(keys, vals, mask, row_ids[seg_start[j] + (i - seg_prefix[j])], seg_part[j]);
}
// the added rows of the involved partitions
__global__ void rowset_insert_add_kernel(unsigned long long* __restrict__ keys, uint32_t* __restrict__ vals,
                                         uint64_t mask, const uint64_t* __restrict__ ids, const uint32_t* __restrict__ part,
                                         uint64_t n, const uint8_t* __restrict__ involved) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && involved[part[i]]) rowset_insert(keys, vals, mask, ids[i], part[i]);
}
// bad[2]: a raw row that is not a row of the partition it is passed for
__global__ void rowset_check_kernel(const unsigned long long* __restrict__ keys, const uint32_t* __restrict__ vals,
                                    uint64_t mask, const uint64_t* __restrict__ ids, uint64_t n, uint32_t part_a,
                                    uint64_t n_a, const uint32_t* __restrict__ part_b, uint32_t* __restrict__ bad) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long id = ids[i];
  const uint32_t want = i < n_a ? part_a : part_b[i - n_a];
  for (uint64_t h = hash_id(id) & mask;; h = (h + 1) & mask) {
    const unsigned long long k = keys[h];
    if (k == id) {
      if (vals[h] != want) atomicOr(bad + 2, 1u);
      return;
    }
    if (k == NONE64) {
      atomicOr(bad + 2, 1u);
      return;
    }
  }
}

__global__ void fill_u64_kernel(unsigned long long* __restrict__ p, uint64_t n, unsigned long long v) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

__global__ void fill_moved_kernel(const uint32_t* __restrict__ dest, uint64_t n, uint8_t* __restrict__ moved) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) moved[i] = dest[i] != NONE;
}

// An ordered stream compaction of the moved rows (dest != NONE) in blocks of 1024 rows: the rows each block moves,
// then (after an exclusive scan of those counts) each moved row's position, so the moved rows keep the add-op order
constexpr int COMPACT_BLOCK = 1024;
__global__ void __launch_bounds__(COMPACT_BLOCK) moved_count_kernel(const uint32_t* __restrict__ dest, uint64_t n,
                                                                    uint32_t* __restrict__ block_counts) {
  const uint64_t i = (uint64_t)blockIdx.x * COMPACT_BLOCK + threadIdx.x;
  const int c = __syncthreads_count(i < n && dest[i] != NONE);
  if (threadIdx.x == 0) block_counts[blockIdx.x] = (uint32_t)c;
}
__global__ void __launch_bounds__(COMPACT_BLOCK) moved_compact_kernel(const uint32_t* __restrict__ dest, uint64_t n,
                                                                      const uint32_t* __restrict__ block_base,
                                                                      uint32_t* __restrict__ members) {
  __shared__ uint32_t wbase[COMPACT_BLOCK / 32];
  const uint64_t i = (uint64_t)blockIdx.x * COMPACT_BLOCK + threadIdx.x;
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool moved = i < n && dest[i] != NONE;
  const unsigned bal = __ballot_sync(0xffffffffu, moved);
  if (lane == 0) wbase[w] = __popc(bal);
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t run = 0;
    for (int k = 0; k < COMPACT_BLOCK / 32; ++k) {
      const uint32_t t = wbase[k];
      wbase[k] = run;
      run += t;
    }
  }
  __syncthreads();
  if (moved) members[block_base[blockIdx.x] + wbase[w] + __popc(bal & ((1u << lane) - 1))] = (uint32_t)i;
}

// 1 in *flag when some v[i] is 0
__global__ void any_zero_kernel(const uint8_t* __restrict__ v, uint64_t n, uint32_t* __restrict__ flag) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && !v[i]) atomicOr(flag, 1u);
}

// moved row t (members[t], in add-op order) -> contiguous rows, ids, destinations, and whether it left a
// candidate partition
__global__ void gather_moved_kernel(const uint32_t* __restrict__ members, uint64_t cnt, const uint8_t* __restrict__ rows_a,
                                    uint64_t n_a, const uint8_t* __restrict__ rows_b, size_t row_bytes,
                                    const uint64_t* __restrict__ ids_a, const uint64_t* __restrict__ ids_b,
                                    const uint32_t* __restrict__ dest, uint8_t* __restrict__ out_rows,
                                    uint64_t* __restrict__ out_ids, uint32_t* __restrict__ out_dest,
                                    uint8_t* __restrict__ out_cand) {
  const uint64_t t = blockIdx.x;
  if (t >= cnt) return;
  const uint64_t i = members[t];
  const uint8_t* src = i < n_a ? rows_a + i * row_bytes : rows_b + (i - n_a) * row_bytes;
  for (size_t b = threadIdx.x; b < row_bytes; b += blockDim.x) out_rows[t * row_bytes + b] = src[b];
  if (threadIdx.x == 0) {
    out_ids[t] = i < n_a ? ids_a[i] : ids_b[i - n_a];
    out_dest[t] = dest[i];
    out_cand[t] = i >= n_a;
  }
}

// the user's added rows that stay: not of the split partition, not moved out of a candidate partition
__global__ void add_keep_kernel(const uint32_t* __restrict__ part, const uint64_t* __restrict__ ids, uint64_t n,
                                uint32_t split_part, const uint64_t* __restrict__ moved, uint64_t n_moved,
                                uint8_t* __restrict__ keep) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) keep[i] = part[i] != split_part && !(n_moved && sorted_contains(moved, n_moved, ids[i]));
}

// rows per partition of an optimize's add list, and the old rows not mapped to None
__global__ void count_u32_kernel(const uint32_t* __restrict__ part, uint64_t n, int K, uint32_t* __restrict__ counts,
                                 uint32_t* __restrict__ bad) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (part[i] >= (uint32_t)K) atomicOr(bad, 1u);
  else atomicAdd(&counts[part[i]], 1u);
}
__global__ void count_unmapped_kernel(const uint64_t* __restrict__ offsets, int K, const uint64_t* __restrict__ ids,
                                      uint64_t n, const uint64_t* __restrict__ old_ids,
                                      const uint64_t* __restrict__ new_ids, uint64_t n_remap,
                                      uint32_t* __restrict__ counts) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint64_t id = ids[i];
  uint64_t lo = 0, hi = n_remap;
  while (lo < hi) {
    const uint64_t mid = (lo + hi) >> 1;
    if (old_ids[mid] < id) lo = mid + 1; else hi = mid;
  }
  if (lo < n_remap && old_ids[lo] == id && new_ids[lo] == NONE64) return;
  atomicAdd(&counts[part_of_pos(offsets, K, i)], 1u);
}

// batch(from, to[j]) for j < K under the index rule: one warp per row of `to`, for the candidate ranking
template <int METRIC, class T>
__global__ void centroid_row_kernel(const float* __restrict__ from, const float* __restrict__ to, int K, int d,
                                    float* __restrict__ out) {
  constexpr int RULE = batch_rule<METRIC, T>();
  const int j = (int)(((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (j >= K) return;
  const float* y = to + (size_t)j * d;
  float v;
  if constexpr (RULE == RULE_COSINE) {
    float xx, xy, yy;
    cos32_sums(from, y, d, lane, xx, xy, yy);
    v = cos32_finish(xy, xx, yy);
  } else {
    v = row_distance<RULE, METRIC, float>(from, y, d, lane & 15, 0xffffu << (16 * (lane >> 4)), 0.0f);
  }
  if (lane == 0) out[j] = v;
}

template <class F>
void dispatch_split(int metric, lb2_dtype dt, F&& f) {
  auto by_elem = [&](auto m) {
    if (dt == LB2_F16) f(m, type_tag<__half>{});
    else if (dt == LB2_BF16) f(m, type_tag<__nv_bfloat16>{});
    else f(m, type_tag<float>{});
  };
  if (metric == METRIC_DOT) by_elem(std::integral_constant<int, METRIC_DOT>{});
  else if (metric == METRIC_COSINE) by_elem(std::integral_constant<int, METRIC_COSINE>{});
  else by_elem(std::integral_constant<int, METRIC_L2>{});
}

// select_reassign_candidates_impl (builder.rs:1788-1814): batch(c0, centroids), the first min(65, K) by (distance,
// id) (rank_probes' order), `part` dropped, min(65, K) - 1 kept
std::vector<uint32_t> reassign_candidates(const lb2_index* ix, uint32_t part) {
  const int K = ix->K, d = ix->d;
  const int L = std::min(REASSIGN_RANGE + 1, K);
  DevBuf<float> row(K), pd(L);
  DevBuf<uint32_t> ids(L);
  dispatch_split(ix->metric, ix->dtype, [&](auto m, auto e) {
    using T = typename decltype(e)::type;
    LB2_LAUNCH("split_candidates", (centroid_row_kernel<decltype(m)::value, T>), cdiv((uint64_t)K * 32, 256), 256, 0,
               ix->centroids.p + (size_t)part * d, ix->centroids.p, K, d, row.p);
  });
  rank_probes(row.p, 1, K, L, ids.p, pd.p);
  std::vector<uint32_t> h(L), out;
  d2h(h.data(), ids.p, L);
  sync_stream();
  for (uint32_t id : h)
    if (id != part && (int)out.size() < L - 1) out.push_back(id);
  return out;
}

// centroids [k][d] (f32 holding model-type values) in the model type, on the device (what index_merge reads)
DevBuf<uint8_t> model_centroids(const float* c, size_t count, lb2_dtype dt) {
  const lb2_dtype md = model_dtype(dt);
  DevBuf<uint8_t> out(count * dtype_size(md));
  if (md == LB2_F32) d2d(reinterpret_cast<float*>(out.p), c, count);
  else LB2_LAUNCH("convert_from_f32", from_f32_kernel, cdiv(count, 256), 256, 0, c, (int)md, count, (void*)out.p);
  return out;
}

// what a split or join does with its raw rows: the decisions, and the moved rows as an add list of the new model
struct Moved {
  uint64_t cnt = 0;
  DevBuf<uint32_t> dest_all;  // [n_a + n_b]
  DevBuf<uint32_t> part;
  DevBuf<uint8_t> payload, is_cand;
  DevBuf<uint64_t> ids;
  DevBuf<float> fa, fs;
};

void decide_and_transform(const lb2_index* old, const char* what, uint32_t part, const float* c0c1c2 /*[3][d] or null*/,
                          const std::vector<uint32_t>& cands, const void* va, const uint64_t* ia, uint64_t n_a,
                          const void* vb, const uint64_t* ib, const uint32_t* pb, uint64_t n_b,
                          const uint64_t* add_ids, const uint32_t* add_part, uint64_t n_add, bool join,
                          const lb2_index* model, Moved& mv) {
  const int K = old->K, d = old->d;
  const uint64_t n_all = n_a + n_b;
  const size_t rbytes = (size_t)d * dtype_size(old->dtype);
  // candidate ranks per old partition
  std::vector<uint32_t> rank_h(K, NONE);
  for (size_t j = 0; j < cands.size(); ++j) rank_h[cands[j]] = (uint32_t)j;
  DevBuf<uint32_t> rank(K), cid(std::max<size_t>(1, cands.size())), bad(3);
  h2d(rank.p, rank_h.data(), K);
  if (!cands.empty()) h2d(cid.p, cands.data(), cands.size());
  bad.zero();
  // the table: c0, c1, c2 (split) and the candidates' old centroids
  const int S = 3 + (int)cands.size();
  DevBuf<float> table((size_t)S * d);
  table.zero();
  if (c0c1c2) d2d(table.p, c0c1c2, (size_t)3 * d);
  for (size_t j = 0; j < cands.size(); ++j) d2d(table.p + (3 + j) * d, old->centroids.p + (size_t)cands[j] * d, (size_t)d);
  // which raw rows are rows of their partitions: a set of the stored and added rows of `part` and the candidates,
  // sized by those rows alone
  std::vector<uint32_t> involved(1, part);
  involved.insert(involved.end(), cands.begin(), cands.end());
  std::vector<uint8_t> inv_h(K, 0);
  for (uint32_t p : involved) inv_h[p] = 1;
  DevBuf<uint8_t> inv(K);
  h2d(inv.p, inv_h.data(), K);
  std::vector<uint64_t> off(K + 1);
  std::vector<uint32_t> add_cnt(K, 0);
  d2h(off.data(), old->part_offsets.p, (size_t)K + 1);
  DevBuf<uint32_t> acnt(K), range(1);  // (the add list's ids are in range: check_part_ids)
  acnt.zero();
  range.zero();
  if (n_add) {
    LB2_LAUNCH("split_count_added", count_u32_kernel, cdiv(n_add, 256), 256, 0, add_part, n_add, K, acnt.p, range.p);
    d2h(add_cnt.data(), acnt.p, K);
  }
  sync_stream();
  const int nseg = (int)involved.size();
  std::vector<uint64_t> seg_prefix(nseg + 1, 0), seg_start(nseg);
  uint64_t n_add_inv = 0;
  for (int j = 0; j < nseg; ++j) {
    const uint32_t p = involved[j];
    seg_start[j] = off[p];
    seg_prefix[j + 1] = seg_prefix[j] + (off[p + 1] - off[p]);
    n_add_inv += add_cnt[p];
  }
  const uint64_t n_old_inv = seg_prefix[nseg];
  uint64_t cap = 1024;
  while (cap < 2 * (n_old_inv + n_add_inv)) cap <<= 1;
  DevBuf<uint64_t> ids_all(std::max<uint64_t>(1, n_all));
  if (n_a) d2d(ids_all.p, ia, n_a);
  if (n_b) d2d(ids_all.p + n_a, ib, n_b);
  {
    DevBuf<unsigned long long> keys(cap);
    DevBuf<uint32_t> vals(cap);
    DevBuf<uint64_t> dpre(nseg + 1), dstart(nseg);
    DevBuf<uint32_t> dpart(nseg);
    h2d(dpre.p, seg_prefix.data(), nseg + 1);
    h2d(dstart.p, seg_start.data(), nseg);
    h2d(dpart.p, involved.data(), nseg);
    LB2_LAUNCH("split_rowset_fill", fill_u64_kernel, cdiv(cap, 256), 256, 0, keys.p, cap, (unsigned long long)NONE64);
    if (n_old_inv)
      LB2_LAUNCH("split_rowset_insert", rowset_insert_old_kernel, cdiv(n_old_inv, 256), 256, 0, keys.p, vals.p, cap - 1,
                 (const uint64_t*)old->row_ids.p, dpre.p, dstart.p, dpart.p, nseg);
    if (n_add_inv)
      LB2_LAUNCH("split_rowset_insert", rowset_insert_add_kernel, cdiv(n_add, 256), 256, 0, keys.p, vals.p, cap - 1,
                 add_ids, add_part, n_add, inv.p);
    if (n_all)
      LB2_LAUNCH("split_rowset_check", rowset_check_kernel, cdiv(n_all, 256), 256, 0, keys.p, vals.p, cap - 1,
                 ids_all.p, n_all, part, n_a, pb, bad.p);
    sync_stream();  // the set is freed on return
  }
  if (n_all)
    LB2_LAUNCH("split_check_groups", check_groups_kernel, cdiv(std::max(n_a, n_b), 256), 256, 0, ia, n_a, ib, pb,
               rank.p, n_b, bad.p);
  // the decisions
  mv.dest_all.alloc(std::max<uint64_t>(1, n_all));
  if (n_all) {
    int chunk = S;
    while (chunk >= 3 && decide_smem(chunk, d) > 200 * 1024) --chunk;
    if (chunk < 3) fail(LB2_UNSUPPORTED, "%s: d = %d is too large for the decision kernel's shared memory", what, d);
    const size_t smem = decide_smem(chunk, d);
    DecideArgs da{va, n_a, vb, n_b, d, d + 1, pb, rank.p, table.p, S, chunk, cid.p, part, (uint32_t)K, join ? 1 : 0,
                  mv.dest_all.p, bad.p};
    dispatch_split(old->metric, old->dtype, [&](auto m, auto e) {
      using T = typename decltype(e)::type;
      auto kern = split_decide_kernel<decltype(m)::value, T>;
      set_smem(kern, smem);
      unsigned grid = cdiv(n_all, DECIDE_WARPS);
      if (S <= chunk) {  // resident blocks walk the rows
        int per_sm = 0, sms = 0, dev = 0;
        LB2_CUDA(cudaGetDevice(&dev));
        LB2_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
        LB2_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, DECIDE_WARPS * 32, smem));
        grid = std::min<unsigned>(grid, (unsigned)std::max(1, per_sm * sms));
      }
      LB2_LAUNCH("split_decide", kern, grid, DECIDE_WARPS * 32, smem, da);
    });
  }
  uint32_t hb[3];
  d2h(hb, bad.p, 3);
  sync_stream();
  if (hb[1]) fail(LB2_INVALID_ARG, "%s: raw row ids must ascend within a partition, candidate partitions in candidate order", what);
  if (hb[2]) fail(LB2_INVALID_ARG, "%s: a raw row is not a row of the partition it is passed for", what);
  if (hb[0]) fail(LB2_INVALID_ARG, "%s: a raw row the index's transform would drop (rows in an index are finite)", what);
  if (n_all == 0) return;
  // the moved rows in add-op order: the split (or joined) rows, then the candidates' in candidate order
  const unsigned nblk = cdiv(n_all, COMPACT_BLOCK);
  DevBuf<uint32_t> bcount(nblk), members(n_all);
  LB2_LAUNCH("split_moved_count", moved_count_kernel, nblk, COMPACT_BLOCK, 0, mv.dest_all.p, n_all, bcount.p);
  std::vector<uint32_t> bc(nblk);
  d2h(bc.data(), bcount.p, nblk);
  sync_stream();
  uint32_t cnt = 0;
  for (auto& c : bc) {
    const uint32_t t = c;
    c = cnt;
    cnt += t;
  }
  mv.cnt = cnt;
  if (!cnt) return;
  h2d(bcount.p, bc.data(), nblk);
  LB2_LAUNCH("split_moved_compact", moved_compact_kernel, nblk, COMPACT_BLOCK, 0, mv.dest_all.p, n_all, bcount.p,
             members.p);
  DevBuf<uint8_t> rows((size_t)cnt * rbytes);
  mv.ids.alloc(cnt);
  mv.part.alloc(cnt);
  mv.is_cand.alloc(cnt);
  LB2_LAUNCH("split_gather_moved", gather_moved_kernel, cnt, 128, 0, members.p, (uint64_t)cnt, (const uint8_t*)va, n_a,
             (const uint8_t*)vb, rbytes, ia, ib, mv.dest_all.p, rows.p, mv.ids.p, mv.part.p, mv.is_cand.p);
  // build_assign_batch: the new model's transform, PART_ID given (IVF_PQ residuals to the decided partition; IVF_RQ
  // recomputes its partition for the codes and factors, ivf.rs:301-304)
  const bool rq = old->kind == IndexKind::RQ;
  mv.payload.alloc((size_t)cnt * old->row_bytes());
  if (rq) {
    mv.fa.alloc(cnt);
    mv.fs.alloc(cnt);
  }
  Source src(rows.p, cnt, d, old->dtype);
  DevBuf<uint8_t> tvalid(cnt);
  index_transform_rows(model, src, mv.part.p, nullptr, mv.payload.p, mv.fa.p, mv.fs.p, tvalid.p);
  // a moved row the new model's transform drops (no finite distance to any centroid) cannot enter the index
  bad.zero();
  LB2_LAUNCH("split_check_transform", any_zero_kernel, cdiv(cnt, 256), 256, 0, tvalid.p, (uint64_t)cnt, bad.p);
  uint32_t tb = 0;
  d2h(&tb, bad.p, 1);
  sync_stream();
  if (tb) fail(LB2_INVALID_ARG, "%s: a moved row the index's transform drops (no finite distance to a centroid)", what);
}

}  // namespace
}  // namespace lb2

using namespace lb2;

extern "C" {

lb2_status lb2_index_partition_to_split(const lb2_index* ix, const uint32_t* new_part_ids, uint64_t n_new,
                                        uint32_t* part) {
  LB2_API_BEGIN
  LB2_REQUIRE(ix && part && (new_part_ids || n_new == 0), "null argument");
  const int K = ix->K;
  DevBuf<uint32_t> cnt(K), bad(1);
  cnt.zero();
  bad.zero();
  InArg<uint32_t> np(new_part_ids, n_new);
  if (n_new) LB2_LAUNCH("split_count_new", count_u32_kernel, cdiv(n_new, 256), 256, 0, np.get(), n_new, K, cnt.p, bad.p);
  std::vector<uint32_t> c(K);
  std::vector<uint64_t> off(K + 1);
  uint32_t hb = 0;
  d2h(c.data(), cnt.p, K);
  d2h(off.data(), ix->part_offsets.p, (size_t)K + 1);
  d2h(&hb, bad.p, 1);
  sync_stream();
  if (hb) fail(LB2_INVALID_ARG, "partition_to_split: a partition id is out of range (the index has %d)", K);
  // should_split (builder.rs:1152-1176): the largest, strictly above 4 x the target; the first of equal sizes
  const uint64_t limit = MAX_PARTITION_SIZE_FACTOR * target_partition_size(ix);
  uint64_t best = 0;
  *part = NONE;
  for (int p = 0; p < K; ++p) {
    const uint64_t rows = off[p + 1] - off[p] + c[p];
    if (rows > best && rows > limit) {
      best = rows;
      *part = (uint32_t)p;
    }
  }
  LB2_API_END
}

lb2_status lb2_index_partition_to_join(const lb2_index* ix, const uint64_t* remap_old, const uint64_t* remap_new,
                                       uint64_t n_remap, uint32_t* part) {
  LB2_API_BEGIN
  LB2_REQUIRE(ix && part && (n_remap == 0 || (remap_old && remap_new)), "null argument");
  *part = NONE;
  const int K = ix->K;
  if (K <= 1) return LB2_OK;  // at least one partition stays
  DevBuf<uint32_t> cnt(K);
  cnt.zero();
  InArg<uint64_t> ro(remap_old, n_remap), rn(remap_new, n_remap);
  if (ix->n)
    LB2_LAUNCH("join_count", count_unmapped_kernel, cdiv(ix->n, 256), 256, 0, ix->part_offsets.p, K,
               (const uint64_t*)ix->row_ids.p, ix->n, ro.get(), rn.get(), n_remap, cnt.p);
  std::vector<uint32_t> c(K);
  d2h(c.data(), cnt.p, K);
  sync_stream();
  // should_join (builder.rs:1343-1394): the smallest, strictly below 25% of the target; the first of equal sizes
  const uint64_t limit = MIN_PARTITION_SIZE_PERCENT * target_partition_size(ix) / 100;
  uint64_t best = ~0ull;
  for (int p = 0; p < K; ++p)
    if (c[p] < best && c[p] < limit) {
      best = c[p];
      *part = (uint32_t)p;
    }
  LB2_API_END
}

lb2_status lb2_index_reassign_candidates(const lb2_index* ix, uint32_t part, uint32_t* ids_out, uint32_t* count) {
  LB2_API_BEGIN
  LB2_REQUIRE(ix && ids_out && count, "null argument");
  check_kind(ix, "reassign_candidates");
  LB2_REQUIRE(part < (uint32_t)ix->K, "reassign_candidates: partition %u out of range (the index has %d)", part, ix->K);
  const std::vector<uint32_t> c = reassign_candidates(ix, part);
  for (size_t j = 0; j < c.size(); ++j) ids_out[j] = c[j];
  *count = (uint32_t)c.size();
  LB2_API_END
}

lb2_status lb2_index_split(const lb2_index* old, const lb2_split_params* sp, lb2_index** out) {
  LB2_API_BEGIN
  LB2_REQUIRE(old && sp && out, "null argument");
  const char* what = "lb2_index_split";
  check_kind(old, what);
  const lb2_optimize_params& op = sp->opt;
  LB2_REQUIRE(!op.new_centroids && !op.part_map && op.n_remap == 0,
              "%s: new_centroids, part_map and the remap of the embedded optimize are the split's own", what);
  const int K = old->K, d = old->d;
  const uint32_t part = sp->part;
  LB2_REQUIRE(part < (uint32_t)K, "%s: partition %u out of range (the index has %d)", what, part, K);
  const uint64_t n_a = sp->n, n_b = sp->n_cand;
  LB2_REQUIRE((n_a == 0 || (sp->vectors && sp->row_ids)) && (n_b == 0 || (sp->cand_vectors && sp->cand_row_ids && sp->cand_part_ids)),
              "%s: null raw rows", what);
  if (n_a == 0) {  // split_partition without raw rows: the centroids stay (builder.rs:1184-1189)
    LB2_REQUIRE(n_b == 0, "%s: candidate rows without rows of the split partition", what);
    lb2_optimize_params mp = op;
    mp.new_k = K;
    std::unique_ptr<lb2_index> ix = index_merge(old, mp, what);
    if (sp->new_centroids_out) {
      VecOut o(sp->new_centroids_out, (size_t)K * d, model_dtype(old->dtype));
      d2d(o.get(), ix->centroids.p, (size_t)K * d);
      o.commit();
    }
    sync_stream();
    *out = ix.release();
    return LB2_OK;
  }
  // train_kmeans rejects fewer rows than centroids (kmeans.rs:1320-1326)
  LB2_REQUIRE(n_a >= 2, "%s: KMeans: can not train 2 centroids with %llu vectors", what, (unsigned long long)n_a);
  const bool rq = old->kind == IndexKind::RQ;
  const uint64_t n_add = op.n_add;
  LB2_REQUIRE(n_add == 0 || (op.add_payload && op.add_row_ids && op.add_part_ids),
              "%s: added rows need partition ids, payload and row ids", what);
  if (rq)
    LB2_REQUIRE(n_add == 0 || (op.add_rq_add && op.add_rq_scale), "%s: IVF_RQ rows need their add and scale factors", what);
  else
    LB2_REQUIRE(!op.add_rq_add && !op.add_rq_scale, "%s: add and scale factors are for IVF_RQ indexes only", what);
  LB2_REQUIRE(op.n_remove == 0 || op.remove_row_ids, "%s: null remove list", what);
  const lb2_dtype dt = old->dtype;
  const size_t es = dtype_size(dt);
  InArg<uint8_t> va(sp->vectors, (size_t)n_a * d * es), vb(sp->cand_vectors, (size_t)n_b * d * es);
  InArg<uint64_t> ia(sp->row_ids, n_a), ib(sp->cand_row_ids, n_b);
  InArg<uint32_t> pb(sp->cand_part_ids, n_b);
  InArg<uint32_t> ap(op.add_part_ids, op.n_add);
  InArg<uint64_t> ar(op.add_row_ids, op.n_add);
  if (n_b) check_part_ids(pb.get(), n_b, K, what);
  if (op.n_add) check_part_ids(ap.get(), op.n_add, K, what);
  // split_partition_impl (builder.rs:1234-1264): k = 2 on the partition's rows (normalised under cosine, trained with
  // L2), max_iters 50, redos 1, tolerance 1e-4, no balance factor, the first 2 x 256 rows
  DevBuf<float> c012((size_t)3 * d);
  {
    TagScope tg("split_train");
    const uint64_t rows = std::min<uint64_t>(n_a, 512);
    DevBuf<float> x((size_t)rows * d);
    if (dt == LB2_F32)
      d2d(x.p, reinterpret_cast<const float*>(va.get()), (size_t)rows * d);
    else
      LB2_LAUNCH("convert_to_f32", to_f32_kernel, cdiv((uint64_t)rows * d, 256), 256, 0, va.get(), (int)dt,
                 (size_t)rows * d, x.p);
    if (old->metric == METRIC_COSINE) {
      normalize_rows(x.p, rows, d, x.p);
      round_model(x.p, (size_t)rows * d, dt);
    }
    lb2_kmeans_params kp;
    lb2_kmeans_params_default(&kp);
    kp.seed = op.seed;
    std::vector<double> loss;
    std::vector<uint32_t> iters;
    train_kmeans(x.p, rows, d, 2, old->metric == METRIC_DOT ? METRIC_DOT : METRIC_L2, kp, nullptr, c012.p + d, &loss,
                 &iters);
    round_model(c012.p + d, (size_t)2 * d, dt);
    d2d(c012.p, old->centroids.p + (size_t)part * d, (size_t)d);
  }
  // c1 replaces centroid `part`, c2 becomes centroid K
  const uint32_t new_k = K + 1;
  DevBuf<float> newc((size_t)new_k * d);
  d2d(newc.p, old->centroids.p, (size_t)K * d);
  d2d(newc.p + (size_t)part * d, c012.p + d, (size_t)d);
  d2d(newc.p + (size_t)K * d, c012.p + 2 * d, (size_t)d);
  DevBuf<uint8_t> newc_model = model_centroids(newc.p, (size_t)new_k * d, dt);
  std::unique_ptr<lb2_index> model = make_index(old->kind, new_k, d, old->metric, dt);
  copy_model(old, model.get(), newc_model.p);
  if (old->kind == IndexKind::RQ)  // IVF_RQ's moved rows take their nearest new centroid by the index's rule
    set_partition_index(model.get(), old->pi_mode, old->pi_seed, old->pi_batch);
  const std::vector<uint32_t> cands = reassign_candidates(old, part);
  Moved mv;
  decide_and_transform(old, what, part, c012.p, cands, va.get(), ia.get(), n_a, vb.get(), ib.get(), pb.get(), n_b,
                       ar.get(), ap.get(), op.n_add, false, model.get(), mv);
  // the rows that leave a candidate partition are removed from it (AssignOp::Remove), with the caller's removals
  std::vector<uint64_t> removed;
  if (mv.cnt) {
    std::vector<uint64_t> ids(mv.cnt);
    std::vector<uint8_t> cand(mv.cnt);
    d2h(ids.data(), mv.ids.p, mv.cnt);
    d2h(cand.data(), mv.is_cand.p, mv.cnt);
    sync_stream();
    for (uint64_t t = 0; t < mv.cnt; ++t)
      if (cand[t]) removed.push_back(ids[t]);
    std::sort(removed.begin(), removed.end());
  }
  DevBuf<uint64_t> moved_dev(std::max<size_t>(1, removed.size()));
  if (!removed.empty()) h2d(moved_dev.p, removed.data(), removed.size());
  std::vector<uint64_t> rm_all(removed);
  if (op.n_remove) {
    InArg<uint64_t> rm(op.remove_row_ids, op.n_remove);
    std::vector<uint64_t> u(op.n_remove);
    d2h(u.data(), rm.get(), op.n_remove);
    sync_stream();
    std::vector<uint64_t> merged;
    std::merge(u.begin(), u.end(), removed.begin(), removed.end(), std::back_inserter(merged));
    rm_all.swap(merged);
  }
  DevBuf<uint64_t> rm_dev(std::max<size_t>(1, rm_all.size()));
  if (!rm_all.empty()) h2d(rm_dev.p, rm_all.data(), rm_all.size());
  // the add list: the caller's rows that stay, then the moved rows
  const size_t rb = old->row_bytes();
  const uint64_t n_tot = n_add + mv.cnt;
  DevBuf<uint32_t> apart(std::max<uint64_t>(1, n_tot));
  DevBuf<uint8_t> apay(std::max<uint64_t>(1, n_tot * rb)), akeep(std::max<uint64_t>(1, n_tot));
  DevBuf<uint64_t> aid(std::max<uint64_t>(1, n_tot));
  DevBuf<float> afa, afs;
  if (rq) {
    afa.alloc(std::max<uint64_t>(1, n_tot));
    afs.alloc(std::max<uint64_t>(1, n_tot));
  }
  if (n_add) {
    InArg<uint8_t> apl(op.add_payload, (size_t)n_add * rb);
    d2d(apart.p, ap.get(), n_add);
    d2d(apay.p, apl.get(), (size_t)n_add * rb);
    d2d(aid.p, ar.get(), n_add);
    if (rq) {
      InArg<float> fa(op.add_rq_add, n_add), fs(op.add_rq_scale, n_add);
      d2d(afa.p, fa.get(), n_add);
      d2d(afs.p, fs.get(), n_add);
    }
    LB2_LAUNCH("split_add_keep", add_keep_kernel, cdiv(n_add, 256), 256, 0, ap.get(), ar.get(), n_add, part,
               moved_dev.p, (uint64_t)removed.size(), akeep.p);
  }
  if (mv.cnt) {
    d2d(apart.p + n_add, mv.part.p, mv.cnt);
    d2d(apay.p + n_add * rb, mv.payload.p, mv.cnt * rb);
    d2d(aid.p + n_add, mv.ids.p, mv.cnt);
    if (rq) {
      d2d(afa.p + n_add, mv.fa.p, mv.cnt);
      d2d(afs.p + n_add, mv.fs.p, mv.cnt);
    }
    LB2_LAUNCH("fill_valid", fill_moved_kernel, cdiv(mv.cnt, 256), 256, 0, mv.part.p, mv.cnt, akeep.p + n_add);
  }
  // the split partition's stored rows come back only through their decisions
  std::vector<uint32_t> pm(K);
  for (int q = 0; q < K; ++q) pm[q] = (uint32_t)q;
  pm[part] = NONE;
  DevBuf<uint32_t> pm_dev(K);
  h2d(pm_dev.p, pm.data(), K);
  lb2_optimize_params mp = op;
  mp.new_centroids = newc_model.p;
  mp.new_k = new_k;
  mp.part_map = pm_dev.p;
  mp.add_part_ids = n_tot ? apart.p : nullptr;
  mp.add_payload = n_tot ? apay.p : nullptr;
  mp.add_rq_add = rq && n_tot ? afa.p : nullptr;
  mp.add_rq_scale = rq && n_tot ? afs.p : nullptr;
  mp.add_row_ids = n_tot ? aid.p : nullptr;
  mp.n_add = n_tot;
  mp.remove_row_ids = rm_all.empty() ? nullptr : rm_dev.p;
  mp.n_remove = rm_all.size();
  std::unique_ptr<lb2_index> ix = index_merge(old, mp, what, n_tot ? akeep.p : nullptr);
  if (sp->new_centroids_out) {
    VecOut o(sp->new_centroids_out, (size_t)new_k * d, model_dtype(dt));
    d2d(o.get(), newc.p, (size_t)new_k * d);
    o.commit();
  }
  if (sp->dest_out) {
    OutArg<uint32_t> o(sp->dest_out, n_a + n_b);
    d2d(o.get(), mv.dest_all.p, n_a + n_b);
    o.commit();
  }
  sync_stream();
  *out = ix.release();
  LB2_API_END
}

lb2_status lb2_index_join(const lb2_index* old, const lb2_join_params* jp, lb2_index** out) {
  LB2_API_BEGIN
  LB2_REQUIRE(old && jp && out, "null argument");
  const char* what = "lb2_index_join";
  check_kind(old, what);
  const int K = old->K, d = old->d;
  const uint32_t part = jp->part;
  LB2_REQUIRE(K > 1, "%s: the only partition cannot be joined", what);
  LB2_REQUIRE(part < (uint32_t)K, "%s: partition %u out of range (the index has %d)", what, part, K);
  const uint64_t n_a = jp->n;
  LB2_REQUIRE(n_a == 0 || (jp->vectors && jp->row_ids), "%s: null raw rows", what);
  const lb2_dtype dt = old->dtype;
  // join_partition (builder.rs:1401-1423): centroid `part` is deleted, the ids after it shift down by one
  const uint32_t new_k = K - 1;
  DevBuf<float> newc((size_t)new_k * d);
  if (part) d2d(newc.p, old->centroids.p, (size_t)part * d);
  if (part + 1 < (uint32_t)K)
    d2d(newc.p + (size_t)part * d, old->centroids.p + (size_t)(part + 1) * d, (size_t)(K - part - 1) * d);
  DevBuf<uint8_t> newc_model = model_centroids(newc.p, (size_t)new_k * d, dt);
  std::vector<uint32_t> pm(K);
  for (int q = 0; q < K; ++q) pm[q] = q < (int)part ? (uint32_t)q : (q == (int)part ? NONE : (uint32_t)q - 1);
  DevBuf<uint32_t> pm_dev(K);
  h2d(pm_dev.p, pm.data(), K);
  Moved mv;
  InArg<uint8_t> va(jp->vectors, (size_t)n_a * d * dtype_size(dt));
  InArg<uint64_t> ia(jp->row_ids, n_a);
  if (n_a) {
    std::unique_ptr<lb2_index> model = make_index(old->kind, new_k, d, old->metric, dt);
    copy_model(old, model.get(), newc_model.p);
    if (old->kind == IndexKind::RQ)  // IVF_RQ's moved rows take their nearest new centroid by the index's rule
      set_partition_index(model.get(), old->pi_mode, old->pi_seed, old->pi_batch);
    const std::vector<uint32_t> cands = reassign_candidates(old, part);
    decide_and_transform(old, what, part, nullptr, cands, va.get(), ia.get(), n_a, nullptr, nullptr, nullptr, 0,
                         nullptr, nullptr, 0, true, model.get(), mv);
  }
  lb2_optimize_params mp;
  memset(&mp, 0, sizeof(mp));
  mp.new_centroids = newc_model.p;
  mp.new_k = new_k;
  mp.part_map = pm_dev.p;
  mp.add_part_ids = mv.cnt ? mv.part.p : nullptr;
  mp.add_payload = mv.cnt ? mv.payload.p : nullptr;
  mp.add_rq_add = mv.cnt && old->kind == IndexKind::RQ ? mv.fa.p : nullptr;
  mp.add_rq_scale = mv.cnt && old->kind == IndexKind::RQ ? mv.fs.p : nullptr;
  mp.add_row_ids = mv.cnt ? mv.ids.p : nullptr;
  mp.n_add = mv.cnt;
  mp.remove_row_ids = jp->remove_row_ids;
  mp.n_remove = jp->n_remove;
  mp.remap_old_ids = jp->remap_old_ids;
  mp.remap_new_ids = jp->remap_new_ids;
  mp.n_remap = jp->n_remap;
  mp.seed = jp->seed;
  mp.insert_batch = jp->insert_batch;
  std::unique_ptr<lb2_index> ix = index_merge(old, mp, what);
  if (jp->dest_out && n_a) {
    OutArg<uint32_t> o(jp->dest_out, n_a);
    d2d(o.get(), mv.dest_all.p, n_a);
    o.commit();
  }
  sync_stream();
  *out = ix.release();
  LB2_API_END
}

}  // extern "C"
