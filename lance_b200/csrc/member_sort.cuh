// member_sort.cuh -- stable counting sort of rows by cluster id (member_sort.cu).  The Lloyd loop builds its member
// lists with it every iteration, and an index groups its rows by partition with it.  The single-cluster sort body
// is here because the fused small-problem Lloyd kernel (lloyd.cu) inlines it.
#pragma once
#include <stdint.h>

#include <cooperative_groups.h>

#include "common.cuh"
namespace lb2 {

// Stable counting sort of rows by cluster id, batched over B problems:
// members[b][offsets[b][k] .. offsets[b][k+1]) = rows of cluster k in ascending row order.
struct MemberSort {
  DevBuf<uint32_t> chunk_hist, counts, offsets, members;
  void run(const uint32_t* ids, const uint8_t* valid, uint64_t n, int K, int B,
           const uint8_t* active);
};

// lanes of `act` that hold the same key as this lane.  (__match_any_sync gives the same mask but
// the MATCH unit is slow -- ~100 cycles per warp-wide call and not pipelined across warps, measured
// with ncu on the single-CTA sort -- while a ballot per key bit is a handful of cycles.)
__device__ __forceinline__ unsigned same_key_mask(unsigned act, uint32_t key, int nbits) {
  unsigned grp = act;
  for (int bit = 0; bit < nbits; ++bit) {
    const bool one = (key >> bit) & 1u;
    const unsigned bal = __ballot_sync(act, one);
    grp &= one ? bal : ~bal;
  }
  return grp;
}

// Small problems (K <= 1024): the whole stable counting sort of one problem in ONE launch by a
// thread-block CLUSTER of 8 CTAs x 32 warps: every warp owns a contiguous chunk of rows, per-warp
// histograms and running counters live in shared memory, and the cross-CTA prefix is read through
// distributed shared memory between two cluster barriers (no global-memory round trips, no MATCH).
constexpr int SORT_CLUSTER = 8;
// the sort of ONE problem by the calling cluster (8 CTAs x 1024 threads; sm = 34 * K words of shared memory):
// also the member-list phase of the fused small-problem kernel below
template <int NT>
__device__ __forceinline__ void cluster_sort_body(const uint32_t* __restrict__ idb, const uint8_t* __restrict__ vb,
                                                  uint64_t n, int K, uint32_t* __restrict__ counts_b,
                                                  uint32_t* __restrict__ offsets_b, uint32_t* __restrict__ mem,
                                                  uint32_t* sm, uint32_t* wsum) {
  namespace cg = cooperative_groups;
  cg::cluster_group cluster = cg::this_cluster();
  const unsigned crank = cluster.block_rank();
  constexpr int NW = NT / 32;
  uint32_t* wh = sm;             // [NW][K] per-warp histogram, then running counters
  uint32_t* tot = sm + NW * K;   // [K]     this CTA's per-key total (read by the other CTAs)
  uint32_t* off = tot + K;       // [K]     first output slot of this CTA's rows, per key
  const int tid = threadIdx.x, w = tid >> 5, lane = tid & 31;
  for (int i = tid; i < NW * K; i += NT) wh[i] = 0;
  if (tid < 32) wsum[tid] = 0;
  __syncthreads();
  constexpr uint32_t NONE = 0xffffffffu;
  const uint64_t nwarps = (uint64_t)NW * SORT_CLUSTER;
  const uint64_t chunk = ((n + nwarps - 1) / nwarps + 31) / 32 * 32;  // rows per warp, multiple of 32
  const uint64_t r0 = min(n, ((uint64_t)crank * NW + w) * chunk), r1 = min(n, r0 + chunk);
  for (uint64_t base = r0; base < r1; base += 32 * 8) {  // 8 independent loads in flight per lane
    uint32_t key[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const uint64_t r = base + u * 32 + lane;
      key[u] = (r < r1 && (!vb || vb[r])) ? idb[r] : NONE;
    }
#pragma unroll
    for (int u = 0; u < 8; ++u)
      if (key[u] != NONE) atomicAdd(&wh[w * K + key[u]], 1u);
  }
  __syncthreads();
  if (tid < K) {  // exclusive scan over this CTA's warps
    uint32_t run = 0;
    for (int ww = 0; ww < NW; ++ww) {
      const uint32_t t = wh[ww * K + tid];
      wh[ww * K + tid] = run;
      run += t;
    }
    tot[tid] = run;
  }
  cluster.sync();
  uint32_t total = 0, before = 0;  // over all CTAs / over the preceding CTAs, for key `tid`
  if (tid < K) {
    for (unsigned c = 0; c < SORT_CLUSTER; ++c) {
      const uint32_t t = cluster.map_shared_rank(tot, c)[tid];
      total += t;
      if (c < crank) before += t;
    }
  }
  uint32_t incl = total;  // inclusive scan of the per-key totals over the block (K <= 1024)
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  if (lane == 31) wsum[w] = incl;
  __syncthreads();
  if (w == 0) {
    uint32_t v = wsum[lane], inc2 = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t t = __shfl_up_sync(0xffffffffu, inc2, o);
      if (lane >= o) inc2 += t;
    }
    wsum[lane] = inc2 - v;  // exclusive
  }
  __syncthreads();
  const uint32_t excl = wsum[w] + incl - total;
  if (tid < K) {
    off[tid] = excl + before;
    if (crank == 0) {
      counts_b[tid] = total;
      offsets_b[tid] = excl;
      if (tid == K - 1) offsets_b[K] = excl + total;
    }
  }
  __syncthreads();
  const int nbits = 32 - __clz(max(K - 1, 1));
  for (uint64_t base0 = r0; base0 < r1; base0 += 32 * 8) {
    uint32_t keys[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const uint64_t r = base0 + u * 32 + lane;
      keys[u] = (r < r1 && (!vb || vb[r])) ? idb[r] : NONE;
    }
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const uint64_t r = base0 + u * 32 + lane;
      const uint32_t key = keys[u];
      const bool ok = key != NONE;
      const unsigned act = __ballot_sync(0xffffffffu, ok);
      if (ok) {
        const unsigned grp = same_key_mask(act, key, nbits);
        const int rank = __popc(grp & ((1u << lane) - 1));
        const uint32_t start = wh[w * K + key];
        mem[off[key] + start + rank] = (uint32_t)r;
        __syncwarp(act);
        if (rank == 0) wh[w * K + key] = start + __popc(grp);
      }
      __syncwarp();
    }
  }
  cluster.sync();  // nobody leaves while a neighbour may still read its `tot`
}

}  // namespace lb2
