// probe.cu -- how many partitions each query of a search with minimum / maximum nprobes probes.
//
// Replaces  early_pruning / adjust_probes          rust/lance/src/io/exec/knn.rs:1108-1130
//           ANNIvfSubIndexExec::initial_search     knn.rs:837-882
//           ANNIvfSubIndexExec::late_search        knn.rs:714-835 (the cutoff and the no-rows shortcut)
//
// The ranking sorts every centroid distance of a query, so its cost does not depend on how many probes are used:
// up to RANK_TILE partitions in one block's shared memory (bitonic sort on packed (total-order key, id) words),
// more in sorted tiles of RANK_TILE merged pairwise in global memory (each element finds its place in the partner
// run by binary search).  A packed word orders as select_probes_kernel does: by (f32::total_cmp, partition id).
#include "common.cuh"
#include "exact.cuh"
#include "probe.cuh"

namespace lb2 {

constexpr int RANK_THREADS = 1024;

__device__ __forceinline__ uint64_t rank_word(float d, uint32_t id) {
  return ((uint64_t)((uint32_t)total_order_key(d) ^ 0x80000000u) << 32) | id;
}
__device__ __forceinline__ float rank_dist(uint64_t w) {  // inverse of total_order_key: the distance's own bits
  const int32_t key = (int32_t)((uint32_t)(w >> 32) ^ 0x80000000u);
  return __int_as_float(key ^ (int32_t)((uint32_t)(key >> 31) >> 1));
}

// grid (tiles, nq): tile x of query y sorted in shared memory; runs == null (one tile): its first L -> ids / pd
__global__ void __launch_bounds__(RANK_THREADS)
rank_tile_kernel(const float* __restrict__ dists, int K, int L, uint64_t* __restrict__ runs, uint32_t* __restrict__ ids,
                 float* __restrict__ pd) {
  extern __shared__ uint64_t rk[];  // [RANK_TILE]
  const size_t q = blockIdx.y;
  const int t0 = blockIdx.x * RANK_TILE, n = min(RANK_TILE, K - t0), tid = threadIdx.x;
  int N = 1;
  while (N < n) N <<= 1;
  for (int i = tid; i < N; i += RANK_THREADS) rk[i] = i < n ? rank_word(dists[q * K + t0 + i], t0 + i) : ~0ull;
  __syncthreads();
  for (int k2 = 2; k2 <= N; k2 <<= 1) {
    for (int j = k2 >> 1; j > 0; j >>= 1) {
      for (int i = tid; i < N; i += RANK_THREADS) {
        const int o = i ^ j;
        if (o > i) {
          const uint64_t a = rk[i], b = rk[o];
          if ((a > b) == ((i & k2) == 0)) { rk[i] = b; rk[o] = a; }
        }
      }
      __syncthreads();
    }
  }
  if (runs) {
    for (int i = tid; i < n; i += RANK_THREADS) runs[q * K + t0 + i] = rk[i];
  } else {
    for (int i = tid; i < L; i += RANK_THREADS) {
      ids[q * L + i] = (uint32_t)rk[i];
      pd[q * L + i] = rank_dist(rk[i]);
    }
  }
}

// one pass merging sorted runs of R into runs of 2R; the last pass (ids != null) writes the first L
__global__ void __launch_bounds__(256)
rank_merge_kernel(const uint64_t* __restrict__ src, uint64_t* __restrict__ dst, uint64_t nq, int K, int R, int L,
                  uint32_t* __restrict__ ids, float* __restrict__ pd) {
  const uint64_t g = (uint64_t)blockIdx.x * 256 + threadIdx.x;
  if (g >= nq * K) return;
  const uint64_t q = g / K;
  const int j = (int)(g % K), r = j / R, start = r * R, pstart = (r ^ 1) * R;
  const uint64_t v = src[g];
  int pos = j;
  if (pstart < K) {  // rank of v in the partner run: the words are distinct, so "less than" places it exactly
    const uint64_t* p = src + q * K + pstart;
    int lo = 0, hi = min(R, K - pstart);
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (p[mid] < v) lo = mid + 1; else hi = mid;
    }
    pos = (r & ~1) * R + (j - start) + lo;
  }
  if (ids) {
    if (pos < L) {
      ids[q * L + pos] = (uint32_t)v;
      pd[q * L + pos] = rank_dist(v);
    }
  } else {
    dst[q * K + pos] = v;
  }
}

void rank_probes(const float* dists, uint64_t nq, int K, int L, uint32_t* ids, float* pd) {
  if (nq == 0 || K == 0) return;
  const size_t smem = sizeof(uint64_t) * RANK_TILE;
  set_smem(rank_tile_kernel, smem);
  const unsigned tiles = cdiv((uint64_t)K, RANK_TILE);
  if (tiles == 1) {
    LB2_LAUNCH("rank_probes", rank_tile_kernel, dim3(1, (unsigned)nq), RANK_THREADS, smem, dists, K, L,
               (uint64_t*)nullptr, ids, pd);
    return;
  }
  DevBuf<uint64_t> a(nq * K), b(nq * K);
  LB2_LAUNCH("rank_probes", rank_tile_kernel, dim3(tiles, (unsigned)nq), RANK_THREADS, smem, dists, K, L, a.p, ids, pd);
  for (int R = RANK_TILE; R < K; R *= 2) {
    const bool last = 2 * (uint64_t)R >= (uint64_t)K;
    LB2_LAUNCH("rank_probes_merge", rank_merge_kernel, cdiv(nq * K, 256), 256, 0, (const uint64_t*)a.p, b.p, nq, K, R,
               L, last ? ids : nullptr, last ? pd : nullptr);
    std::swap(a.p, b.p);
  }
}

// one warp per partition: the allow bitmap's popcount over the partition's storage range; with a table of bitmaps
// (allows) grid row y counts bitmap y into c[y * K ..]
__global__ void __launch_bounds__(256)
partition_counts_kernel(const uint64_t* __restrict__ off, int K, const uint64_t* __restrict__ allow,
                        const uint64_t* const* __restrict__ allows, uint32_t kc, uint32_t* __restrict__ c) {
  const int p = (int)((blockIdx.x * 256 + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (p >= K) return;
  if (allows) {
    allow = allows[blockIdx.y];
    c += (size_t)blockIdx.y * K;
  }
  const uint64_t a = off[p], b = off[p + 1];
  uint64_t cnt = 0;
  if (!allow) {
    cnt = b - a;
  } else if (a < b) {
    for (uint64_t w = (a >> 6) + lane; w <= ((b - 1) >> 6); w += 32) {
      const uint64_t w0 = w << 6, lo = max(a, w0) - w0, hi = min(b, w0 + 64) - w0;
      const uint64_t m = (hi == 64 ? ~0ull : (1ull << hi) - 1) & ~((1ull << lo) - 1);
      cnt += __popcll(allow[w] & m);
    }
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  }
  if (lane == 0) c[p] = (uint32_t)min(cnt, (uint64_t)kc);
}

void partition_counts(const uint64_t* part_offsets, int K, const uint64_t* allow, uint32_t kc, uint32_t* c) {
  if (K == 0) return;
  LB2_LAUNCH("partition_counts", partition_counts_kernel, cdiv((uint64_t)K * 32, 256), 256, 0, part_offsets, K, allow,
             (const uint64_t* const*)nullptr, kc, c);
}

void partition_counts_table(const uint64_t* part_offsets, int K, const uint64_t* const* allows, int nf, uint32_t* c) {
  if (K == 0 || nf == 0) return;
  LB2_LAUNCH("partition_counts", partition_counts_kernel, dim3(cdiv((uint64_t)K * 32, 256), (unsigned)nf), 256, 0,
             part_offsets, K, (const uint64_t*)nullptr, allows, 0xffffffffu, c);
}

// early_pruning (knn.rs:1117-1130): Rust's slice::partition_point(|d| d <= d0 * f), i.e. binary_search_by as
// Rust 1.90's core implements it (a fixed number of halving steps, then one last probe).  For finite distances
// this is the count of distances <= d0 * f; with NaN among them it is what that search returns.
__device__ __forceinline__ uint32_t early_pruning(const float* d, uint32_t L, uint32_t k) {
  if (L == 0) return 0;
  const float f = k <= 1 ? 0.6f : (k <= 10 ? 7.0f : 81.0f);
  const float thr = __fmul_rn(d[0], f);
  uint32_t size = L, base = 0;
  while (size > 1) {
    const uint32_t half = size / 2, mid = base + half;
    if (d[mid] <= thr) base = mid;
    size -= half;
  }
  return base + (d[base] <= thr ? 1u : 0u);
}

struct CutoffArgs {
  uint32_t min_np, late_width, k;
  int has_max_len, iterable;
  uint64_t max_len;
};

// one thread per query
__global__ void __launch_bounds__(128)
probe_cutoff_kernel(const CutoffArgs a0, uint64_t nq, int L, const uint32_t* __restrict__ pids,
                    const float* __restrict__ pd, const uint32_t* __restrict__ cpart, uint32_t* __restrict__ cslot,
                    int slot_stride, uint32_t* __restrict__ nsearch, uint32_t* __restrict__ shortcut,
                    uint32_t* __restrict__ nmax, uint32_t* __restrict__ nprobes_out,
                    const QueryProbe* __restrict__ qpr) {
  const uint64_t q = (uint64_t)blockIdx.x * 128 + threadIdx.x;
  if (q >= nq) return;
  CutoffArgs a = a0;
  uint32_t Lu = (uint32_t)L, kc = 0xffffffffu;
  if (qpr) {  // a batch: the query's own rule, and its own filter's counts capped by its own k'
    const QueryProbe& r = qpr[q];
    a.min_np = r.min_np;
    a.k = r.k;
    a.has_max_len = r.has_max_len;
    a.iterable = r.mask_ids != nullptr;
    a.max_len = r.max_len;
    Lu = r.L;
    kc = r.kc;
    if (!cslot || !r.ranged) cpart = r.cpart;
  }
  auto c = [&](uint32_t t) -> uint64_t {
    return cpart ? min(kc, cpart[pids[q * L + t]]) : cslot[q * slot_stride + t];
  };
  const uint32_t k = a.k;
  // adjust_probes (knn.rs:1108-1115) then initial_search's min(partitions.len())
  const uint32_t min_np = min(max(a.min_np, early_pruning(pd + q * L, Lu, k)), Lu);
  uint64_t sum0 = 0;
  for (uint32_t t = 0; t < min_np; ++t) sum0 += c(t);
  const uint64_t found0 = min(sum0, (uint64_t)k);  // initial_ids holds at most k ids (knn.rs:680-691)
  uint32_t n = min_np, sc = 0;
  if (Lu > min_np && found0 < k) {
    if (a.has_max_len && a.iterable && found0 < a.max_len && a.max_len <= k) {
      sc = 1;  // knn.rs:746-783: the allow list's missing ids at +inf instead of a late search
    } else {
      // late partition t is searched while found0 plus the rows of the late partitions that finished before it
      // started (all but the late_width - 1 just before it) stays below the target
      const uint64_t target = a.has_max_len ? min(a.max_len, (uint64_t)k) : k;
      uint64_t acc = found0;
      for (uint32_t t = 0; min_np + t < Lu; ++t) {
        if (t >= a.late_width) acc += c(min_np + t - a.late_width);
        if (acc >= target) break;
        ++n;
      }
    }
  }
  nsearch[q] = n;
  shortcut[q] = sc;
  atomicMax(nmax, n);
  if (nprobes_out) nprobes_out[q] = n;
  if (cslot)  // the lists past the cutoff were scanned ahead of it: emptied
    for (uint32_t t = n; t < Lu; ++t) cslot[q * slot_stride + t] = 0;
}

void probe_cutoff(const ProbeRule& r, uint64_t nq, int L, const uint32_t* pids, const float* pd, const uint32_t* cpart,
                  uint32_t* cslot, int slot_stride, uint32_t* nsearch, uint32_t* shortcut, uint32_t* nmax,
                  uint32_t* nprobes_out, const QueryProbe* qpr) {
  if (nq == 0) return;
  const CutoffArgs a{r.min_np, r.late_width, r.k, r.has_max_len, r.mask_ids != nullptr, r.max_len};
  LB2_LAUNCH("probe_cutoff", probe_cutoff_kernel, cdiv(nq, 128), 128, 0, a, nq, L, pids, pd, cpart, cslot, slot_stride,
             nsearch, shortcut, nmax, nprobes_out, qpr);
}

__global__ void gather_probes_kernel(uint64_t nq, int L, const uint32_t* __restrict__ pids, const float* __restrict__ pd,
                                     const uint32_t* __restrict__ nsearch, int nl, uint32_t sentinel,
                                     uint32_t* __restrict__ out_ids, float* __restrict__ out_pd,
                                     const QueryProbe* __restrict__ qpr) {
  const uint64_t g = (uint64_t)blockIdx.x * 256 + threadIdx.x;
  if (g >= nq * nl) return;
  const uint64_t q = g / nl;
  const uint32_t t = (uint32_t)(g % nl), n = nsearch ? nsearch[q] : (qpr ? qpr[q].L : (uint32_t)L);
  const bool live = t < n && t < (uint32_t)L;
  out_ids[g] = live ? pids[q * L + t] : sentinel;
  out_pd[g] = live ? pd[q * L + t] : 0.0f;
}

void gather_probes(uint64_t nq, int L, const uint32_t* pids, const float* pd, const uint32_t* nsearch, int nl,
                   uint32_t sentinel, uint32_t* out_ids, float* out_pd, const QueryProbe* qpr) {
  if (nq == 0 || nl == 0) return;
  LB2_LAUNCH("gather_probes", gather_probes_kernel, cdiv(nq * nl, 256), 256, 0, nq, L, pids, pd, nsearch, nl, sentinel,
             out_ids, out_pd, qpr);
}

// one block per query.  The query's lists hold found0 < max_len <= k <= 1024 rows when it takes the shortcut.
__global__ void __launch_bounds__(128)
shortcut_kernel(const uint32_t* __restrict__ shortcut, const uint64_t* __restrict__ mask_ids, uint64_t nmask, int nl,
                int kc, float* __restrict__ cand_d, uint64_t* __restrict__ cand_id, uint32_t* __restrict__ cand_cnt,
                const QueryProbe* __restrict__ qpr) {
  __shared__ uint64_t found[1024];
  __shared__ uint32_t s_nf, s_out, s_wsum[4];
  const uint64_t q = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const size_t list = q * nl + (nl - 1);
  if (!shortcut[q]) {
    if (tid == 0) cand_cnt[list] = 0;
    return;
  }
  const int stride = kc;  // a batch: the query's own ids and k'; the lists' stride stays kc
  if (qpr) {
    mask_ids = qpr[q].mask_ids;
    nmask = qpr[q].num_mask_ids;
    kc = (int)qpr[q].kc;
  }
  if (tid == 0) { s_nf = 0; s_out = 0; }
  __syncthreads();
  for (int t = 0; t < nl - 1; ++t) {
    const uint32_t cnt = cand_cnt[q * nl + t];
    for (uint32_t e = tid; e < cnt; e += 128) {
      const uint32_t at = atomicAdd(&s_nf, 1u);
      if (at < 1024) found[at] = cand_id[(q * nl + t) * stride + e];
    }
  }
  __syncthreads();
  const uint32_t nf = min(s_nf, 1024u);
  for (uint64_t i0 = 0; i0 < nmask; i0 += 128) {
    const uint32_t out0 = s_out;
    if (out0 >= (uint32_t)kc) break;
    const uint64_t i = i0 + tid;
    bool keep = false;
    uint64_t id = 0;
    if (i < nmask) {
      id = mask_ids[i];
      keep = i == 0 || mask_ids[i - 1] != id;  // a repeated id counts once, as in the reference's HashSet
      for (uint32_t f = 0; f < nf && keep; ++f) keep = found[f] != id;
    }
    const unsigned bal = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) s_wsum[warp] = __popc(bal);
    __syncthreads();
    uint32_t pos = out0 + __popc(bal & ((1u << lane) - 1));
    for (int w = 0; w < warp; ++w) pos += s_wsum[w];
    if (keep && pos < (uint32_t)kc) {
      cand_id[list * stride + pos] = id;
      cand_d[list * stride + pos] = __int_as_float(0x7f800000);
    }
    __syncthreads();
    if (tid == 0) s_out = min((uint32_t)kc, out0 + s_wsum[0] + s_wsum[1] + s_wsum[2] + s_wsum[3]);
    __syncthreads();
  }
  if (tid == 0) cand_cnt[list] = s_out;
}

void shortcut_lists(uint64_t nq, const uint32_t* shortcut, const uint64_t* mask_ids, uint64_t num_mask_ids, int nl,
                    int kc, float* cand_d, uint64_t* cand_id, uint32_t* cand_cnt, const QueryProbe* qpr) {
  if (nq == 0) return;
  LB2_LAUNCH("probe_shortcut", shortcut_kernel, (unsigned)nq, 128, 0, shortcut, mask_ids, num_mask_ids, nl, kc, cand_d,
             cand_id, cand_cnt, qpr);
}

}  // namespace lb2
