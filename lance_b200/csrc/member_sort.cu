// member_sort.cu -- MemberSort::run: the four-kernel stable counting sort, or one thread-block cluster for
// K <= 1024 and n <= 2^21 (cluster_sort_body, member_sort.cuh).
#include <algorithm>

#include "member_sort.cuh"

namespace lb2 {

// ------------------------------------------------------------------------------------------------
// stable counting sort of rows by cluster id
// ------------------------------------------------------------------------------------------------
__global__ void hist_kernel(const uint32_t* __restrict__ ids, const uint8_t* __restrict__ valid,
                            uint64_t n, int K, int chunk_rows, uint32_t* __restrict__ chunk_hist,
                            const uint8_t* __restrict__ active) {
  const int b = blockIdx.y;
  if (active && !active[b]) return;
  const uint64_t r0 = (uint64_t)blockIdx.x * chunk_rows;
  const uint64_t r1 = min(n, r0 + (uint64_t)chunk_rows);
  uint32_t* h = chunk_hist + ((size_t)b * gridDim.x + blockIdx.x) * K;
  for (uint64_t r = r0 + threadIdx.x; r < r1; r += blockDim.x)
    if (!valid || valid[(size_t)b * n + r]) atomicAdd(&h[ids[(size_t)b * n + r]], 1u);
}

// per (b, k): exclusive scan over chunks (in place), total -> counts
__global__ void scan_chunks_kernel(uint32_t* __restrict__ chunk_hist, int nchunks, int K, int B,
                                   uint32_t* __restrict__ counts) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= B * K) return;
  const int b = g / K, k = g % K;
  uint32_t run = 0;
  for (int c = 0; c < nchunks; ++c) {
    uint32_t* p = chunk_hist + ((size_t)b * nchunks + c) * K + k;
    const uint32_t t = *p;
    *p = run;
    run += t;
  }
  counts[g] = run;
}

// per b: offsets[b][0..K] = exclusive scan of counts[b][:]
__global__ void offsets_kernel(const uint32_t* __restrict__ counts, int K,
                               uint32_t* __restrict__ offsets) {
  __shared__ uint32_t part[1024];
  const int b = blockIdx.x, t = threadIdx.x;
  const int seg = (K + 1023) / 1024;
  const int s = t * seg, e = min(K, s + seg);
  uint32_t sum = 0;
  for (int k = s; k < e; ++k) sum += counts[(size_t)b * K + k];
  part[t] = sum;
  __syncthreads();
  if (t == 0) {
    uint32_t run = 0;
    for (int i = 0; i < 1024; ++i) {
      uint32_t v = part[i];
      part[i] = run;
      run += v;
    }
    offsets[(size_t)b * (K + 1) + K] = run;
  }
  __syncthreads();
  uint32_t run = part[t];
  for (int k = s; k < e; ++k) {
    offsets[(size_t)b * (K + 1) + k] = run;
    run += counts[(size_t)b * K + k];
  }
}

// one warp per (chunk, b): rows in ascending order, rank inside a batch of 32 by match_any
__global__ void scatter_kernel(const uint32_t* __restrict__ ids, const uint8_t* __restrict__ valid,
                               uint64_t n, int K, int chunk_rows, uint32_t* __restrict__ chunk_hist,
                               const uint32_t* __restrict__ offsets, uint32_t* __restrict__ members,
                               const uint8_t* __restrict__ active) {
  const int b = blockIdx.y;
  if (active && !active[b]) return;
  const int lane = threadIdx.x;
  const int nbits = 32 - __clz(max(K - 1, 1));
  const uint64_t r0 = (uint64_t)blockIdx.x * chunk_rows;
  const uint64_t r1 = min(n, r0 + (uint64_t)chunk_rows);
  uint32_t* h = chunk_hist + ((size_t)b * gridDim.x + blockIdx.x) * K;
  const uint32_t* off = offsets + (size_t)b * (K + 1);
  for (uint64_t base = r0; base < r1; base += 32) {
    const uint64_t r = base + lane;
    const bool ok = r < r1 && (!valid || valid[(size_t)b * n + r]);
    const unsigned act = __ballot_sync(0xffffffffu, ok);
    if (ok) {
      const uint32_t key = ids[(size_t)b * n + r];
      const unsigned grp = same_key_mask(act, key, nbits);
      const int rank = __popc(grp & ((1u << lane) - 1));
      const uint32_t start = h[key];
      members[(size_t)b * n + off[key] + start + rank] = (uint32_t)r;
      __syncwarp(act);
      if (rank == 0) h[key] = start + __popc(grp);
    }
    __syncwarp();
  }
}

__global__ void __cluster_dims__(SORT_CLUSTER, 1, 1) __launch_bounds__(1024)
cluster_sort_kernel(const uint32_t* __restrict__ ids, const uint8_t* __restrict__ valid, uint64_t n,
                    int K, uint32_t* __restrict__ counts, uint32_t* __restrict__ offsets,
                    uint32_t* __restrict__ members, const uint8_t* __restrict__ active) {
  const int b = blockIdx.y;
  if (active && !active[b]) return;  // uniform over the cluster
  extern __shared__ uint32_t sm[];
  __shared__ uint32_t wsum[32];
  cluster_sort_body<1024>(ids + (size_t)b * n, valid ? valid + (size_t)b * n : nullptr, n, K, counts + (size_t)b * K,
                          offsets + (size_t)b * (K + 1), members + (size_t)b * n, sm, wsum);
}

// ------------------------------------------------------------------------------------------------
// member lists (also used to group rows by partition when an index is loaded)
// ------------------------------------------------------------------------------------------------
void MemberSort::run(const uint32_t* ids, const uint8_t* valid, uint64_t n, int K, int B,
                     const uint8_t* active) {
  if (K <= 1024 && n <= (1ull << 21) && n >= 1) {
    if (counts.n < (size_t)B * K) counts.alloc((size_t)B * K);
    if (offsets.n < (size_t)B * (K + 1)) offsets.alloc((size_t)B * (K + 1));
    if (members.n < (size_t)B * n) members.alloc((size_t)B * n);
    const size_t smem = sizeof(uint32_t) * (34 * (size_t)K);
    set_smem(cluster_sort_kernel, smem);
    LB2_LAUNCH("member_sort_cluster", cluster_sort_kernel, dim3(SORT_CLUSTER, B), 1024, smem, ids,
               valid, n, K, counts.p, offsets.p, members.p, active);
    return;
  }
  // chunk size: keep the per-chunk histogram table below ~256 MB
  // one warp scatters one chunk sequentially (32 rows per step): keep chunks short so that the
  // grid is wide, but bound the per-chunk histogram table (B * nchunks * K counters) to ~64 MB
  int chunk_rows = 256;
  while ((uint64_t)chunk_rows * 1024 < n) chunk_rows *= 2;  // at most ~1024 chunks (scan is per chunk)
  while ((double)B * (double)cdiv(n, chunk_rows) * K * 4.0 > 64e6) chunk_rows *= 2;
  const int nchunks = std::max(1u, cdiv(n, chunk_rows));
  if (chunk_hist.n < (size_t)B * nchunks * K) chunk_hist.alloc((size_t)B * nchunks * K);
  if (counts.n < (size_t)B * K) counts.alloc((size_t)B * K);
  if (offsets.n < (size_t)B * (K + 1)) offsets.alloc((size_t)B * (K + 1));
  if (members.n < (size_t)B * n) members.alloc((size_t)B * std::max<uint64_t>(n, 1));
  LB2_CUDA(cudaMemsetAsync(chunk_hist.p, 0, sizeof(uint32_t) * (size_t)B * nchunks * K, ctx().stream));
  dim3 grid(nchunks, B);
  LB2_LAUNCH("member_sort", hist_kernel, grid, 256, 0, ids, valid, n, K, chunk_rows, chunk_hist.p, active);
  LB2_LAUNCH("member_sort", scan_chunks_kernel, cdiv((uint64_t)B * K, 128), 128, 0, chunk_hist.p,
             nchunks, K, B, counts.p);
  LB2_LAUNCH("member_sort", offsets_kernel, B, 1024, 0, counts.p, K, offsets.p);
  LB2_LAUNCH("member_sort", scatter_kernel, grid, 32, 0, ids, valid, n, K, chunk_rows, chunk_hist.p,
             offsets.p, members.p, active);
}

}  // namespace lb2
