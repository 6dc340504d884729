// lloyd.cu -- Lloyd iterations on the device, batched over B independent problems
// (B = 1 for the IVF coarse quantiser, B = M for the PQ sub-space codebooks).
//
// Replaces  KMeans::train_kmeans            lance-index/src/vector/kmeans.rs:610-719
//           KMeansAlgoFloat::to_kmeans      kmeans.rs:371-446   (centroid update)
//           compute_membership_and_loss     kmeans.rs:250-281   (radius / f64 loss per cluster)
//           compute_cluster_sizes           kmeans.rs:210-232
//           split_clusters                  kmeans.rs:174-207
//
// Design: the reference sums each cluster's rows SEQUENTIALLY IN ROW ORDER in f32 and its losses in
// f64, so the result depends on the order.  Instead of atomics (fast but order-free) we build, per
// iteration, a stable counting sort of the rows by cluster (member lists in ascending row order)
// and add each cluster's members in that order: one warp per (cluster, 8-dimension chunk) gathers the
// member rows 128 at a time and lanes 0..7 run the sequential f32 chains (update_body_warp), one warp
// per cluster the f64 loss chain (stats_body).  Where no addition can round -- see "order-independent
// sums" below -- the chain is replaced by a parallel reduction that returns the same bits.  Given the
// same initial centroids the trained model is therefore BIT-IDENTICAL to the reference loop (every
// variant is checked by tests/test_lloyd_variants.py), at the cost of a sort of n 4-byte keys per
// iteration.  The scalar bookkeeping of an iteration runs in epilogue_kernel, and iterations 2..
// replay one captured CUDA graph.
#include <cooperative_groups.h>

#include <algorithm>
#include <cmath>
#include <limits>
#include <map>
#include <unordered_map>

#include "assign.cuh"
#include "comm.cuh"
#include "common.cuh"
#include "exact.cuh"
#include "kmeans.cuh"
#include "member_sort.cuh"
#include "tc_assign.cuh"
#include "tc_pq.cuh"

namespace lb2 {

// ------------------------------------------------------------------------------------------------
// ordered centroid update (kmeans.rs:388-418): one thread per (b, cluster, t)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void update_body(size_t g, const float* __restrict__ x, int ldx, int ds, int K, int B, uint64_t n,
                              const uint32_t* __restrict__ members,
                              const uint32_t* __restrict__ offsets, float* __restrict__ centroids,
                              const uint8_t* __restrict__ active, int scale) {
  if (g >= (size_t)B * K * ds) return;
  const int b = g / ((size_t)K * ds);
  if (active && !active[b]) return;
  const int k = (g / ds) % K, t = g % ds;
  const uint32_t* off = offsets + (size_t)b * (K + 1);
  const uint32_t s = off[k], e = off[k + 1];
  const uint32_t* mem = members + (size_t)b * n;
  const float* col = x + (size_t)b * ds + t;
  float acc = 0.0f;
  uint32_t j = s;
  for (; j + 16 <= e; j += 16) {
    float v[16];
#pragma unroll
    for (int q = 0; q < 16; ++q) v[q] = col[(size_t)mem[j + q] * ldx];
#pragma unroll
    for (int q = 0; q < 16; ++q) acc = f_add(acc, v[q]);
  }
  for (; j < e; ++j) acc = f_add(acc, col[(size_t)mem[j] * ldx]);
  const uint32_t cnt = e - s;
  if (scale && cnt > 0) acc = __fmul_rn(acc, __fdiv_rn(1.0f, (float)cnt));  // kmeans.rs:414-416
  centroids[g] = acc;
}

// ---- order-independent sums -------------------------------------------------------------------
// The reference adds a cluster's members one after the other (f32 centroid sums, f64 loss), and a
// floating-point sum depends on that order -- unless no addition rounds.  If every term is an integer
// multiple of 2^g and sum|term| < 2^(g+p) (p = 24 for f32, 53 for f64), every partial sum of ANY
// association is such a multiple below 2^(g+p), hence exactly representable: all orders give the same
// bits.  g = min over the non-zero terms of (unbiased exponent - 23 + trailing zeros of the 24-bit
// significand).  The kernels below test this per cluster (with one bit of margin, the bound itself
// being computed in floating point) and then reduce in parallel; otherwise they run the sequential
// chain.  The f64 loss uses the general test (distances nearly always pass); the f32 centroid sums use
// the special case g = 0 (integer-valued columns: SIFT, u8, quantised data), which costs three adds per
// term to check.  A per-problem hint stops retrying once a problem's data has failed.
__device__ __forceinline__ int pow2_granule(float v, bool& bad) {
  const uint32_t bits = __float_as_uint(v) & 0x7fffffffu;
  if (bits == 0) return 0x7fffffff;  // zero is a multiple of everything
  uint32_t ex = bits >> 23;
  if (ex == 255) { bad = true; return 0x7fffffff; }
  uint32_t mant = bits & 0x7fffffu;
  if (ex) mant |= 0x800000u; else ex = 1;
  return (int)ex - 150 + (__ffs((int)mant) - 1);
}
__device__ __forceinline__ double pow2_f64(int e) {  // 2^e, -1022 <= e <= 1023
  return __longlong_as_double((long long)(e + 1023) << 52);
}

// The centroid update for ds % 8 == 0, one WARP per (b, cluster, 8-dim chunk).
//   fast path (see above): lanes stride the members, private f32 sums, one warp reduction;
//   sequential path: the 32 lanes fetch 128 member rows at a time (index load + 32-byte gather, all
//   independent -> one memory round trip per 128 members instead of one per 16), park them in shared
//   memory, then lanes 0..7 add their dimension in member order -- update_body's sums exactly.
constexpr int UPD_TILE = 128;
__device__ __forceinline__ void update_body_warp(size_t w, float* tile, const float* __restrict__ x, int ldx, int ds,
                                                 int K, int B, uint64_t n, const uint32_t* __restrict__ members,
                                                 const uint32_t* __restrict__ offsets,
                                                 float* __restrict__ centroids,
                                                 const uint8_t* __restrict__ active, int scale,
                                                 uint8_t* __restrict__ exact_hint) {
  const int lane = threadIdx.x & 31;
  const int nch = ds >> 3;
  if (w >= (size_t)B * K * nch) return;
  const int b = (int)(w / ((size_t)K * nch));
  if (active && !active[b]) return;
  const int k = (int)((w / nch) % K), c = (int)(w % nch);
  const uint32_t* off = offsets + (size_t)b * (K + 1);
  const uint32_t s = off[k], e = off[k + 1];
  const uint32_t* mem = members + (size_t)b * n;
  const float* col = x + (size_t)b * ds + c * 8;
  float* out = centroids + ((size_t)b * K + k) * ds + c * 8;
  const float inv = (scale && e > s) ? __fdiv_rn(1.0f, (float)(e - s)) : 1.0f;  // kmeans.rs:414-416
  const bool do_scale = scale && e > s;

  if (e - s >= 64 && exact_hint[b]) {  // ---- fast path: only worth it for long chains
    // Centroid sums: the cheap special case g = 0 -- every term an INTEGER (SIFT / u8 / quantised
    // columns) and sum|term| < 2^23.  (v + 1.5*2^23) - 1.5*2^23 == v  <=>  v is an integer, for |v| < 2^22.
    float sum[8], asum[8];
#pragma unroll
    for (int t = 0; t < 8; ++t) { sum[t] = 0.0f; asum[t] = 0.0f; }
    float dev = 0.0f;  // max |v - round(v)|: 0 iff all terms are integers
    for (uint32_t j0 = s; j0 < e; j0 += 128) {
      float4 va[4], vb[4];
      bool have[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const uint32_t j = j0 + u * 32 + lane;
        have[u] = j < e;
        if (have[u]) {
          const float4* src = reinterpret_cast<const float4*>(col + (size_t)mem[j] * ldx);
          va[u] = src[0];
          vb[u] = src[1];
        }
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        if (have[u]) {
          const float v[8] = {va[u].x, va[u].y, va[u].z, va[u].w, vb[u].x, vb[u].y, vb[u].z, vb[u].w};
#pragma unroll
          for (int t = 0; t < 8; ++t) {
            sum[t] = __fadd_rn(sum[t], v[t]);
            asum[t] = __fadd_rn(asum[t], fabsf(v[t]));
            const float rt = __fadd_rn(__fadd_rn(v[t], 12582912.0f), -12582912.0f);
            dev = fmaxf(dev, fabsf(__fadd_rn(rt, -v[t])));
          }
        }
      }
    }
    // sum over the lanes of each lane's largest |.| sum bounds every dimension's sum|term| from above
    float amax = 0.0f;
#pragma unroll
    for (int t = 0; t < 8; ++t) amax = fmaxf(amax, asum[t]);
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) {
#pragma unroll
      for (int t = 0; t < 8; ++t) sum[t] = __fadd_rn(sum[t], __shfl_xor_sync(0xffffffffu, sum[t], o));
      amax = __fadd_rn(amax, __shfl_xor_sync(0xffffffffu, amax, o));
      dev = fmaxf(dev, __shfl_xor_sync(0xffffffffu, dev, o));
    }
    const bool exact = dev == 0.0f && amax < 8388608.0f;  // NaN / Inf terms fail the comparison
    if (exact) {
      if (lane < 8) {
        float r = 0.0f;
#pragma unroll
        for (int t = 0; t < 8; ++t)
          if (lane == t) r = sum[t];
        out[lane] = do_scale ? __fmul_rn(r, inv) : r;
      }
      return;
    }
    if (lane == 0) exact_hint[b] = 0;  // this problem's data is not of the exact kind: stop trying
  }

  float acc = 0.0f;
  constexpr int UU = UPD_TILE / 32;
  float4 pa[UU], pb[UU];  // the next tile's rows, fetched while the current tile is being summed
  auto fetch = [&](uint32_t base) {
    uint32_t r[UU];
#pragma unroll
    for (int u = 0; u < UU; ++u) {
      const uint32_t j = base + u * 32 + lane;
      r[u] = j < e ? mem[j] : 0xffffffffu;
    }
#pragma unroll
    for (int u = 0; u < UU; ++u) {
      if (r[u] != 0xffffffffu) {
        const float4* src = reinterpret_cast<const float4*>(col + (size_t)r[u] * ldx);
        pa[u] = src[0];
        pb[u] = src[1];
      }
    }
  };
  if (s < e) fetch(s);
  for (uint32_t base = s; base < e; base += UPD_TILE) {
    const uint32_t cnt = min((uint32_t)UPD_TILE, e - base);
#pragma unroll
    for (int u = 0; u < UU; ++u) {
      float4* dst = reinterpret_cast<float4*>(tile + (u * 32 + lane) * 8);
      dst[0] = pa[u];
      dst[1] = pb[u];
    }
    __syncwarp();
    if (base + UPD_TILE < e) fetch(base + UPD_TILE);
    if (lane < 8) {
      uint32_t q = 0;
      for (; q + 16 <= cnt; q += 16) {  // 16 loads ahead of a 4-cycle add chain
        float v[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) v[i] = tile[(q + i) * 8 + lane];
#pragma unroll
        for (int i = 0; i < 16; ++i) acc = f_add(acc, v[i]);
      }
      for (; q < cnt; ++q) acc = f_add(acc, tile[q * 8 + lane]);
    }
    __syncwarp();
  }
  if (lane < 8) out[lane] = do_scale ? __fmul_rn(acc, inv) : acc;
}

// per (b, cluster): f64 loss in row order, radius (max), last member row (kmeans.rs:266-280)
__device__ __forceinline__ void stats_body(int w, const float* __restrict__ dists, uint64_t n, int K, int B,
                             const uint32_t* __restrict__ members,
                             const uint32_t* __restrict__ offsets, double* __restrict__ losses,
                             float* __restrict__ radius, uint32_t* __restrict__ last_row,
                             const uint8_t* __restrict__ active, uint8_t* __restrict__ loss_hint) {
  const int lane = threadIdx.x & 31;
  if (w >= B * K) return;
  const int b = w / K, k = w % K;
  if (active && !active[b]) return;
  const uint32_t* off = offsets + (size_t)b * (K + 1);
  const uint32_t s = off[k], e = off[k + 1];
  const uint32_t* mem = members + (size_t)b * n;
  const float* dv = dists + (size_t)b * n;
  double loss = 0.0;
  float rad = 0.0f;
  if (e - s >= 64 && loss_hint[b]) {  // ---- order-independent f64 sum (see "order-independent sums")
    double sd = 0.0, ad = 0.0;
    float rm = 0.0f;
    int g = 0x7fffffff;
    bool bad = false;
    for (uint32_t j0 = s; j0 < e; j0 += 256) {
      float v[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const uint32_t j = j0 + u * 32 + lane;
        v[u] = j < e ? dv[mem[j]] : 0.0f;
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        sd += (double)v[u];
        ad += (double)fabsf(v[u]);
        rm = fmaxf(rm, v[u]);
        g = min(g, pow2_granule(v[u], bad));
      }
    }
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) {
      sd += __shfl_xor_sync(0xffffffffu, sd, o);
      ad += __shfl_xor_sync(0xffffffffu, ad, o);
      rm = fmaxf(rm, __shfl_xor_sync(0xffffffffu, rm, o));
      g = min(g, __shfl_xor_sync(0xffffffffu, g, o));
    }
    bad = __any_sync(0xffffffffu, bad);
    if (!bad && (g == 0x7fffffff || ad < pow2_f64(g + 52))) {  // exact iff sum|.| < 2^(g+53); 1 bit margin
      if (lane == 0) {
        losses[w] = sd;
        radius[w] = rm;
        last_row[w] = mem[e - 1];
      }
      return;
    }
    if (lane == 0) loss_hint[b] = 0;
  }
  // 256 members per round, the NEXT round's (index, distance) gathers in flight while this round's
  // values are folded in member order: the only serial work left is the f64 add chain itself
  constexpr int SU = 8;
  float cur[SU], nxt[SU];
#pragma unroll
  for (int u = 0; u < SU; ++u) {
    const uint32_t j = s + u * 32 + lane;
    cur[u] = j < e ? dv[mem[j]] : 0.0f;
  }
  for (uint32_t base = s; base < e; base += SU * 32) {
#pragma unroll
    for (int u = 0; u < SU; ++u) {
      const uint32_t j = base + (SU + u) * 32 + lane;
      nxt[u] = j < e ? dv[mem[j]] : 0.0f;
    }
#pragma unroll
    for (int u = 0; u < SU; ++u) {
      const uint32_t b0 = base + u * 32;
      if (b0 < e) {  // uniform
        const int cnt = min(32u, e - b0);
        if (cnt == 32) {
#pragma unroll
          for (int q = 0; q < 32; ++q) {
            const float v = __shfl_sync(0xffffffffu, cur[u], q);
            loss += (double)v;
            rad = fmaxf(rad, v);  // f32::max ignores NaN like fmaxf; dists of members are never NaN
          }
        } else {
          for (int q = 0; q < cnt; ++q) {
            const float v = __shfl_sync(0xffffffffu, cur[u], q);
            loss += (double)v;
            rad = fmaxf(rad, v);
          }
        }
      }
    }
#pragma unroll
    for (int u = 0; u < SU; ++u) cur[u] = nxt[u];
  }
  if (lane == 0) {
    losses[w] = loss;
    radius[w] = rad;
    last_row[w] = e > s ? mem[e - 1] : 0xffffffffu;
  }
}

// one launch for both: the first `update_blocks` blocks (128 threads each) run the ordered centroid
// update, the remaining blocks the per-cluster f64 loss / radius / last-member statistics
__global__ void __launch_bounds__(128)
update_stats_kernel(unsigned update_blocks, const float* __restrict__ x, int ldx, int ds, int K, int B,
                    uint64_t n, const uint32_t* __restrict__ members, const uint32_t* __restrict__ offsets,
                    float* __restrict__ centroids, const float* __restrict__ dists,
                    double* __restrict__ losses, float* __restrict__ radius,
                    uint32_t* __restrict__ last_row, const uint8_t* __restrict__ active, int scale,
                    int warp_update, uint8_t* __restrict__ hints /* [2][B]: exact-sum hints */) {
  __shared__ __align__(16) float tiles[4][UPD_TILE * 8];
  if (blockIdx.x < update_blocks) {
    if (warp_update)
      update_body_warp((size_t)blockIdx.x * 4 + (threadIdx.x >> 5), tiles[threadIdx.x >> 5], x, ldx, ds, K, B, n,
                       members, offsets, centroids, active, scale, hints);
    else
      update_body((size_t)blockIdx.x * 128 + threadIdx.x, x, ldx, ds, K, B, n, members, offsets, centroids, active, scale);
  } else {
    stats_body((int)(((size_t)(blockIdx.x - update_blocks) * 128 + threadIdx.x) >> 5), dists, n, K, B,
               members, offsets, losses, radius, last_row, active, hints + B);
  }
}

// ---- multi-GPU (SURVEY 8e): ONE exchange per Lloyd iteration ------------------------------------------
// Every rank packs its partial results of the iteration into one blob
//     [ sums f32 BK*ds | counts u32 BK | radius f32 BK | last member row u32 BK (global, +1; 0 = none) | loss f64 BK ]
// (update_stats_kernel writes the sums straight into it), the blobs are all-gathered in ONE collective, and
// every rank reduces the gathered blobs in RANK ORDER -- so all ranks hold bit-identical models whatever
// algorithm the transport uses, and the whole iteration (collective included) replays from a CUDA graph.
struct ExchangeLayout {
  size_t off_counts, off_radius, off_last, off_loss, bytes;
};
static ExchangeLayout exchange_layout(size_t BK, int ds) {
  ExchangeLayout L;
  L.off_counts = (BK * ds * sizeof(float) + 15) / 16 * 16;
  L.off_radius = L.off_counts + BK * 4;
  L.off_last = L.off_radius + BK * 4;
  L.off_loss = (L.off_last + BK * 4 + 7) / 8 * 8;
  L.bytes = (L.off_loss + BK * 8 + 15) / 16 * 16;
  return L;
}
__global__ void pack_partials_kernel(uint8_t* __restrict__ blob, ExchangeLayout L, size_t BK,
                                     const uint32_t* __restrict__ counts, const float* __restrict__ radius,
                                     const uint32_t* __restrict__ last_row, const double* __restrict__ losses,
                                     uint32_t row_offset) {
  const size_t g = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= BK) return;
  reinterpret_cast<uint32_t*>(blob + L.off_counts)[g] = counts[g];
  reinterpret_cast<float*>(blob + L.off_radius)[g] = radius[g];
  reinterpret_cast<uint32_t*>(blob + L.off_last)[g] = last_row[g] == 0xffffffffu ? 0u : last_row[g] + row_offset + 1u;
  reinterpret_cast<double*>(blob + L.off_loss)[g] = losses[g];
}
__global__ void reduce_partials_kernel(const uint8_t* __restrict__ gathered, int nranks, ExchangeLayout L, size_t BK,
                                       int ds, int K, float* __restrict__ centroids, uint32_t* __restrict__ counts,
                                       float* __restrict__ radius, uint32_t* __restrict__ last_row,
                                       double* __restrict__ losses, const uint8_t* __restrict__ active) {
  const size_t g = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= BK * ds) return;
  const size_t ck = g / ds;
  if (active && !active[ck / K]) return;
  float sum = 0.0f;
  uint32_t cnt = 0;
  for (int r = 0; r < nranks; ++r) {
    const uint8_t* blob = gathered + (size_t)r * L.bytes;
    sum = __fadd_rn(sum, reinterpret_cast<const float*>(blob)[g]);
    cnt += reinterpret_cast<const uint32_t*>(blob + L.off_counts)[ck];
  }
  centroids[g] = cnt > 0 ? __fmul_rn(sum, __fdiv_rn(1.0f, (float)cnt)) : sum;  // kmeans.rs:414-416
  if (g % ds == 0) {
    float rad = 0.0f;
    uint32_t last = 0;
    double loss = 0.0;
    for (int r = 0; r < nranks; ++r) {
      const uint8_t* blob = gathered + (size_t)r * L.bytes;
      rad = fmaxf(rad, reinterpret_cast<const float*>(blob + L.off_radius)[ck]);
      last = max(last, reinterpret_cast<const uint32_t*>(blob + L.off_last)[ck]);
      loss += reinterpret_cast<const double*>(blob + L.off_loss)[ck];
    }
    counts[ck] = cnt;
    radius[ck] = rad;
    last_row[ck] = last == 0u ? 0xffffffffu : last - 1u;
    losses[ck] = loss;
  }
}

// initialisation: the k picked rows are GLOBAL row numbers (rank-major order); every rank copies the rows it
// owns into a zeroed buffer and a sharded run sums the buffers (each row has exactly one owner, x + 0 is exact)
// -- the picks, and with them the model, do not depend on how the sample is sharded.  One rank owns every row.
__global__ void gather_init_owned_kernel(const float* __restrict__ x, int ldx, int ds, int K, int B,
                                         const uint32_t* __restrict__ rows, uint32_t row_offset, uint32_t n_local,
                                         float* __restrict__ out) {
  const size_t g = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= (size_t)B * K * ds) return;
  const int b = g / ((size_t)K * ds), k = (g / ds) % K, t = g % ds;
  const uint32_t gr = rows[(size_t)b * K + k];
  const bool mine = gr >= row_offset && gr - row_offset < n_local;
  out[g] = mine ? x[(size_t)(gr - row_offset) * ldx + (size_t)b * ds + t] : 0.0f;
}

// ------------------------------------------------------------------------------------------------
// per-iteration scalar epilogue ON THE DEVICE: exactly the reference's bookkeeping
//   compute_cluster_sizes (kmeans.rs:210-232), compute_balance_loss (:234-237), loss sum (:693),
//   split_clusters (:174-207, our rng), tolerance test (:704), next iteration's bias (:341-345).
// One block per problem; thread 0 runs the order-dependent scalar parts.
// ------------------------------------------------------------------------------------------------
struct LloydState {  // one per problem, device resident
  double loss;        // previous iteration's loss (f64::MAX at start)
  double last_loss;   // this iteration's loss
  float adjusted;     // adjusted_balance_factor (f32::MAX at start)
  float bf_cur;       // balance factor used by the membership step that just ran
  uint64_t rng;       // splitmix64 state
  uint32_t iters;     // epilogues run while active
};

__device__ __forceinline__ uint64_t sm64_next(uint64_t& s) {
  uint64_t z = (s += 0x9E3779B97F4A7C15ull);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// (a device function so that the fused small-problem kernel can run it too: problem b, by the NT threads of
// the calling block)
template <int NT>
__device__ __forceinline__ void epilogue_body(int b, int K, int ds, uint64_t n, float bf_param, double tolerance,
                const uint32_t* __restrict__ counts, const double* __restrict__ losses,
                const float* __restrict__ radius, const uint32_t* __restrict__ last_row,
                uint64_t* __restrict__ cluster_sizes, float* __restrict__ bias, int bias_ld,
                float* __restrict__ centroids, LloydState* __restrict__ states,
                uint8_t* __restrict__ active, TcPqPrepArgs pq_prep) {
  const int tid = threadIdx.x;
  __shared__ int s_i, s_j;
  LloydState& st = states[b];
  uint64_t* cs = cluster_sizes + (size_t)b * K;
  const uint32_t* cnt = counts + (size_t)b * K;
  const double* ls = losses + (size_t)b * K;
  float* cb = centroids + (size_t)b * K * ds;
  // (1) order-independent parts in parallel: cluster sizes, sum of squares, and the
  //     "first cluster to reach the final maximum" = max count, then smallest last member row
  __shared__ unsigned long long s_red_a[NT];  // packed (count << 32 | ~last_row) -> max
  __shared__ unsigned long long s_red_sq[NT];
  __shared__ int s_red_id[NT];
  __shared__ double s_chunk[1024];
  __shared__ int s_any_empty;
  {
    unsigned long long best = 0, sq = 0;
    int best_id = 0;
    bool have = false;
    int empty = 0;
    for (int k = tid; k < K; k += blockDim.x) {
      const uint32_t c = cnt[k];
      cs[k] = c;
      sq += (unsigned long long)c * c;
      empty |= (c == 0);
      const uint32_t lr = c > 0 ? last_row[(size_t)b * K + k] : 0xffffffffu;
      const unsigned long long key = ((unsigned long long)c << 32) | (uint32_t)(~lr);
      // ties on (count, last_row) cannot happen for c > 0 (a row belongs to one cluster); for
      // c == 0 everywhere the reference keeps id 0 -> prefer the lowest k on equal keys
      if (!have || key > best) { best = key; best_id = k; have = true; }
    }
    s_red_a[tid] = have ? best : 0ull;
    s_red_id[tid] = have ? best_id : 0x7fffffff;
    s_red_sq[tid] = sq;
    const int any = __syncthreads_or(empty);
    if (tid == 0) s_any_empty = any;
    for (int off = NT / 2; off >= 1; off >>= 1) {
      if (tid < off) {
        const unsigned long long o = s_red_a[tid + off];
        const int oi = s_red_id[tid + off];
        if (o > s_red_a[tid] || (o == s_red_a[tid] && oi < s_red_id[tid])) {
          s_red_a[tid] = o;
          s_red_id[tid] = oi;
        }
        s_red_sq[tid] += s_red_sq[tid + off];
      }
      __syncthreads();
    }
  }
  // (2) the f64 loss sum is order dependent (kmeans.rs:693): staged through shared memory in
  //     chunks, added sequentially by thread 0
  double sum = 0.0;
  for (int k0 = 0; k0 < K; k0 += 1024) {
    for (int k = tid; k < 1024 && k0 + k < K; k += blockDim.x) s_chunk[k] = ls[k0 + k];
    __syncthreads();
    if (tid == 0) {
      const int m = min(1024, K - k0);
      for (int k = 0; k < m; ++k) sum += s_chunk[k];
    }
    __syncthreads();
  }
  if (tid == 0) {
    const int max_id = s_red_id[0] == 0x7fffffff ? 0 : s_red_id[0];
    const uint64_t size_sq = s_red_sq[0];
    st.adjusted = __fdiv_rn(__fsub_rn(radius[(size_t)b * K + max_id],
                                      __fdiv_rn((float)ls[max_id], (float)cs[max_id])),
                            (float)n);
    const float balance_loss =
        __fmul_rn(st.bf_cur, __fsub_rn((float)size_sq, __fdiv_rn((float)(n * n), (float)K)));
    st.last_loss = sum + (double)balance_loss;
    st.iters += 1;
  }
  __syncthreads();
  // split_clusters: sequential over empty clusters, vector part by the whole block
  int next = 0;
  for (; s_any_empty;) {
    if (tid == 0) {
      int i = next;
      while (i < K && cs[i] != 0) ++i;
      s_i = i < K ? i : -1;
      if (i < K) {
        uint64_t j = 0;
        for (uint64_t tries = 0;; ++tries) {
          const float p = __fdiv_rn(__fsub_rn((float)cs[j], 1.0f), (float)(n - (uint64_t)K));
          const float u = (float)(sm64_next(st.rng) >> 40) * (1.0f / 16777216.0f);
          if (u < p) break;
          j = (j + 1) % (uint64_t)K;
          if (tries >= 64ull * K) {
            j = 0;
            for (int c = 1; c < K; ++c)
              if (cs[c] > cs[j]) j = c;
            break;
          }
        }
        cs[i] = cs[j] / 2;
        cs[j] -= cs[i];
        s_j = (int)j;
      }
    }
    __syncthreads();
    const int i = s_i, j = s_j;
    if (i < 0) break;
    const float eps = 1.0f / 1024.0f;
    for (int t = tid; t < ds; t += blockDim.x) {
      const float cj = cb[(size_t)j * ds + t];
      if ((t & 1) == 0) {
        cb[(size_t)i * ds + t] = __fmul_rn(cj, 1.0f + eps);
        cb[(size_t)j * ds + t] = __fmul_rn(cj, 1.0f - eps);
      } else {
        cb[(size_t)i * ds + t] = __fmul_rn(cj, 1.0f - eps);
        cb[(size_t)j * ds + t] = __fmul_rn(cj, 1.0f + eps);
      }
    }
    next = i + 1;
    __syncthreads();
  }
  // convergence (kmeans.rs:704) and the next iteration's balance factor / bias
  __shared__ float s_bf;
  if (tid == 0) {
    if (fabs(st.loss - st.last_loss) < tolerance * st.last_loss) {
      active[b] = 0;
    } else {
      st.loss = st.last_loss;
    }
    st.bf_cur = fminf(st.adjusted, bf_param);  // f32::min: the non-NaN operand
    s_bf = st.bf_cur;
  }
  __syncthreads();
  if (bias)
    for (int k = tid; k < K; k += blockDim.x)
      bias[(size_t)b * bias_ld + k] = __fmul_rn(s_bf, (float)cs[k]);
  if (NT == 256 && pq_prep.bm) {  // PQ tensor path (K == 256 codewords x 8 dims, 256 threads): operands of the NEXT iteration
    __shared__ float s_n2[256];
    __syncthreads();  // the split above may have rewritten codewords
    tc_pq_prep_block(cb, b, pq_prep, s_n2);
  }
}

__global__ void __launch_bounds__(256)
epilogue_kernel(int K, int ds, uint64_t n, float bf_param, double tolerance,
                const uint32_t* __restrict__ counts, const double* __restrict__ losses,
                const float* __restrict__ radius, const uint32_t* __restrict__ last_row,
                uint64_t* __restrict__ cluster_sizes, float* __restrict__ bias, int bias_ld,
                float* __restrict__ centroids, LloydState* __restrict__ states,
                uint8_t* __restrict__ active, TcPqPrepArgs pq_prep, volatile uint32_t* host_words) {
  const int b = blockIdx.x;
  if (pq_prep.bm && threadIdx.x == 0) pq_prep.fb_count[b] = 0;  // next iteration's undecided-row list (active or not)
  if (!active[b]) return;
  epilogue_body<256>(b, K, ds, n, bf_param, tolerance, counts, losses, radius, last_row, cluster_sizes, bias, bias_ld,
                     centroids, states, active, pq_prep);
  // progress word of problem b in PINNED HOST memory (one posted 4-byte write over PCIe, no copy-engine operation
  // in the stream): iteration << 1 | still active.  Posted only while the problem is active, so the last word is
  // the one of the iteration that converged it (PollWords).
  if (threadIdx.x == 0)  // thread 0 wrote iters and active[b] above
    host_words[b] = (states[b].iters << 1) | (active[b] ? 1u : 0u);
}


// ------------------------------------------------------------------------------------------------
// Small problems (hierarchical k-means splits a cluster with k' <= 16, kmeans.rs:885-895: thousands of
// Lloyd runs over a few hundred .. a few thousand rows): the WHOLE run in one launch.  A thread-block
// cluster of 8 CTAs x 512 threads iterates  assign (exact, 16 lanes per row = the reference's lane
// accumulators) -> stable member sort (cluster_sort_body) -> ordered centroid sums + f64 loss (the same
// update_body_warp / stats_body as the general path) -> scalar epilogue (epilogue_body, CTA 0)  with cluster
// barriers between the phases; nothing returns to the host until the run has converged.  Same device functions,
// same order of every floating-point operation as the multi-kernel path -> bit-identical models; ~10 us per
// iteration instead of ~10 launches.
// ------------------------------------------------------------------------------------------------
constexpr int SMALL_UPD_WARPS = 8;  // warps per CTA that run update / stats tasks (one 4 KB tile each)
constexpr int SMALL_NT = 512;       // 512 threads: 128 registers each (the update / stats bodies need them)
template <int METRIC>
__global__ void __cluster_dims__(SORT_CLUSTER, 1, 1) __launch_bounds__(SMALL_NT)
lloyd_small_kernel(const float* __restrict__ x, uint32_t n, int d, int K, float* __restrict__ centroids,
                   float bf_param, double tolerance, int max_iters, uint32_t* __restrict__ ids,
                   float* __restrict__ dists, uint8_t* __restrict__ valid, uint32_t* __restrict__ counts,
                   uint32_t* __restrict__ offsets, uint32_t* __restrict__ members, double* __restrict__ losses,
                   float* __restrict__ radius, uint32_t* __restrict__ last_row,
                   uint64_t* __restrict__ cluster_sizes, float* __restrict__ bias, LloydState* __restrict__ state,
                   uint8_t* __restrict__ active, uint8_t* __restrict__ hints, int warp_update) {
  namespace cg = cooperative_groups;
  cg::cluster_group cluster = cg::this_cluster();
  const unsigned crank = cluster.block_rank();
  extern __shared__ __align__(16) uint8_t small_smem[];
  float* cs = reinterpret_cast<float*>(small_smem);                    // [K][d] centroids of this iteration
  float* sb = cs + (size_t)K * d;                                       // [16] bias
  float* tiles = sb + 16;                                               // [SMALL_UPD_WARPS][UPD_TILE * 8]
  uint32_t* sort_sm = reinterpret_cast<uint32_t*>(tiles + SMALL_UPD_WARPS * UPD_TILE * 8);  // [(NT/32 + 2) * K]
  __shared__ uint32_t wsum[32];
  const int tid = threadIdx.x, warp = tid >> 5, l = tid & 15;
  const unsigned hmask = 0xffffu << (16 * ((tid >> 4) & 1));
  const int n16 = d & ~15;
  const int nch = d >> 3;
  const uint32_t hw_global = crank * (SMALL_NT / 16) + (tid >> 4), hw_total = SORT_CLUSTER * (SMALL_NT / 16);  // half-warps
  for (int it = 1; it <= max_iters; ++it) {
    // ---- centroids + bias of this iteration into shared memory
    for (int i = tid; i < K * d; i += SMALL_NT) cs[i] = centroids[i];
    if (tid < 16) sb[tid] = tid < K ? bias[tid] : 0.0f;
    __syncthreads();
    // ---- membership (kmeans.rs:317-369): lane l of a half-warp owns lane accumulator l (l2.rs:82-88)
    for (uint32_t r = hw_global; r < n; r += hw_total) {
      const float* xv = x + (size_t)r * d;
      float acc[16];
#pragma unroll
      for (int j = 0; j < 16; ++j) acc[j] = 0.0f;
      for (int e0 = l; e0 < n16; e0 += 16 * 8) {  // eight row elements in flight per lane (the loads are what costs)
        float xr[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) xr[u] = e0 + 16 * u < n16 ? xv[e0 + 16 * u] : 0.0f;
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          const int e = e0 + 16 * u;
          if (e < n16) {
#pragma unroll
            for (int j = 0; j < 16; ++j)
              if (j < K) acc[j] = f_add(acc[j], term<METRIC>(xr[u], cs[j * d + e]));
          }
        }
      }
      float best_key = __int_as_float(0x7f800000), best_val = best_key;
      uint32_t best_idx = 0xffffffffu;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        if (j < K) {  // uniform
          float sq = 0.0f;  // sequential tail (l2.rs:69-79), every lane redundantly
          for (int e = n16; e < d; ++e) sq = f_add(sq, term<METRIC>(xv[e], cs[j * d + e]));
          float t = 0.0f;
#pragma unroll
          for (int q = 0; q < 16; ++q) t = f_add(t, __shfl_sync(hmask, acc[j], q, 16));
          const float v = finish<METRIC>(f_add(sq, t));
          const float key = f_add(v, sb[j]);
          if (key < best_key) { best_key = key; best_val = v; best_idx = j; }
        }
      }
      if (l == 0) {
        const bool ok = best_idx != 0xffffffffu;
        ids[r] = ok ? best_idx : 0u;
        dists[r] = ok ? best_val : __int_as_float(0x7fc00000);
        valid[r] = ok ? 1 : 0;
      }
    }
    __threadfence();
    cluster.sync();
    // ---- member lists (stable counting sort of the rows by cluster)
    cluster_sort_body<SMALL_NT>(ids, valid, n, K, counts, offsets, members, sort_sm, wsum);
    __threadfence();
    cluster.sync();
    // ---- ordered centroid sums (kmeans.rs:388-418) and per-cluster f64 loss / radius (kmeans.rs:266-280)
    if (warp_update) {
      if (warp < SMALL_UPD_WARPS) {
        const int ntask = K * nch + K;
        for (int t = crank * SMALL_UPD_WARPS + warp; t < ntask; t += SORT_CLUSTER * SMALL_UPD_WARPS) {
          if (t < K * nch)
            update_body_warp((size_t)t, tiles + warp * UPD_TILE * 8, x, d, d, K, 1, n, members, offsets, centroids,
                             nullptr, 1, hints);
          else
            stats_body(t - K * nch, dists, n, K, 1, members, offsets, losses, radius, last_row, nullptr, hints + 1);
          __syncwarp();
        }
      }
    } else {
      for (size_t g = (size_t)crank * SMALL_NT + tid; g < (size_t)K * d; g += (size_t)SORT_CLUSTER * SMALL_NT)
        update_body(g, x, d, d, K, 1, n, members, offsets, centroids, nullptr, 1);
      for (int t = crank * (SMALL_NT / 32) + warp; t < K; t += SORT_CLUSTER * (SMALL_NT / 32))
        stats_body(t, dists, n, K, 1, members, offsets, losses, radius, last_row, nullptr, hints + 1);
    }
    __threadfence();
    cluster.sync();
    // ---- the iteration's scalar bookkeeping (cluster sizes, balance loss, split_clusters, tolerance test, bias)
    if (crank == 0)
      epilogue_body<SMALL_NT>(0, K, d, n, bf_param, tolerance, counts, losses, radius, last_row, cluster_sizes, bias,
                          16, centroids, state, active, TcPqPrepArgs());
    __threadfence();
    cluster.sync();
    if (!*reinterpret_cast<volatile uint8_t*>(active)) break;  // converged (kmeans.rs:704)
  }
}

static bool lloyd_small_ok(uint64_t n, int B, int ds, int K, bool dist) {
  static const bool off = getenv("LB2_NO_SMALL_KMEANS") && *getenv("LB2_NO_SMALL_KMEANS");
  // one cluster = 8 SMs of plain FP32 against ~10 launches: measured (tools/small_kmeans_timing.py) to pay off only
  // for the tiniest runs (n * k * d <= 2^20, e.g. 512 rows x 2 centroids x 128: 43 vs 66 us per iteration)
  return !off && !dist && B == 1 && K >= 1 && K <= 16 && n >= 1 && n <= 16384 && (uint64_t)K * ds <= 24576 &&
         n * (uint64_t)K * ds <= (1ull << 20) && !ctx().profiling;
}

// ------------------------------------------------------------------------------------------------
// the Lloyd loop: no host round trip per iteration; the host only reads the progress words
// ------------------------------------------------------------------------------------------------
// Convergence is learnt WITHOUT draining the stream and without any operation in it: epilogue_kernel posts one
// word per problem into pinned, device-mapped host memory -- iteration << 1 | active -- for as long as the problem
// is active, so the last word it ever posts names the iteration that converged it.  After enqueuing iteration it,
// the host asks whether every problem converged by want = it - 1; the device meanwhile has iteration it queued, and
// at most one no-op iteration is enqueued past convergence (every kernel returns at once for an inactive problem).
// The answer depends only on the iteration of convergence, not on when the host reads the word, so every rank of a
// sharded run (bit-identical states) enqueues the same iterations and none waits in an exchange its peer skipped.
// (A blocking copy + synchronise every 4 iterations left the GPU idle for a copy and a graph launch each time; an
// asynchronous copy + event per iteration cost as much in the stream: measured, tools/iter_timing.py.)
// One block per (thread, device), kept for the thread's lifetime and grown to the largest B it has served.
class PollWords {
 public:
  // the calling thread's words for the current device, reset to 1 (iteration 0, active) for problems 0 .. B-1;
  // the stream must be idle (no epilogue of an earlier run still to post)
  static PollWords& reset(int B) {
    static thread_local std::map<int, PollWords> per_device;
    PollWords& w = per_device[ctx().device];
    if (w.cap_ < B) {
      if (w.host_) LB2_CUDA(cudaFreeHost(const_cast<uint32_t*>(w.host_)));
      w.host_ = nullptr;
      w.cap_ = 0;
      void *p = nullptr, *dp = nullptr;
      LB2_CUDA(cudaHostAlloc(&p, sizeof(uint32_t) * B, cudaHostAllocMapped | cudaHostAllocPortable));
      w.host_ = static_cast<volatile uint32_t*>(p);
      w.cap_ = B;
      LB2_CUDA(cudaHostGetDevicePointer(&dp, p, 0));
      w.dev_ = static_cast<uint32_t*>(dp);
    }
    for (int b = 0; b < B; ++b) w.host_[b] = 1u;
    return w;
  }
  uint32_t* device() const { return dev_; }
  // has every problem 0 .. B-1 converged at an iteration <= want?  Waits, for each problem, until its word is of
  // iteration want or later, or shows it converged.
  bool done(int B, uint32_t want) const {
    uint64_t spins = 0;
    for (int b = 0; b < B; ++b) {
      uint32_t w;
      while (!settled(w = host_[b], want)) {
        if ((++spins & 0xFFFFF) == 0) {  // every ~1M reads: has the stream died or drained without reporting?
          const cudaError_t q = cudaStreamQuery(ctx().stream);
          if (q != cudaErrorNotReady) {
            if (q != cudaSuccess) LB2_CUDA(q);
            if (!settled(host_[b], want)) fail(LB2_CUDA_ERROR, "k-means progress word %d never arrived", b);
          }
        }
      }
      if ((w & 1u) || (w >> 1) > want) return false;
    }
    return true;
  }

 private:
  static bool settled(uint32_t w, uint32_t want) { return !(w & 1u) || (w >> 1) >= want; }
  volatile uint32_t* host_ = nullptr;
  uint32_t* dev_ = nullptr;
  int cap_ = 0;
};

void lloyd_train(const float* x, uint64_t n_in, int ldx, int B, int ds, int K, const LloydParams& p,
                 const float* init_dev, float* centroids, std::vector<double>* loss_out,
                 std::vector<uint32_t>* iters_out) {
  LB2_REQUIRE(current_comm() || n_in >= (uint64_t)K, "KMeans: can not train %d centroids with %llu vectors", K,
              (unsigned long long)n_in);
  // kmeans.rs:623-627: only the first 512*k rows are used
  Comm* cm = current_comm();
  const bool dist = cm && cm->nranks > 1;
  uint64_t n = n_in >= (uint64_t)K * 512 ? (uint64_t)K * 512 : n_in;
  uint64_t n_global = n, row_offset = 0;
  if (dist) {
    // every rank holds a row shard of the sample; rows are ordered rank-major
    n = std::min<uint64_t>(n_in, ((uint64_t)K * 512 + cm->nranks - 1) / cm->nranks);
    std::vector<uint32_t> all(cm->nranks, 0);
    all[cm->rank] = (uint32_t)n;
    sum_over_ranks(all);
    n_global = 0;
    for (int r = 0; r < cm->nranks; ++r) {
      if (r < cm->rank) row_offset += all[r];
      n_global += all[r];
    }
    LB2_REQUIRE(n_global >= (uint64_t)K, "KMeans: can not train %d centroids with %llu vectors", K,
                (unsigned long long)n_global);
  }
  LB2_REQUIRE(n_global < 0xfffffffeull, "training sample too large");
  const size_t BK = (size_t)B * K;
  const bool small = B > 1;

  // ---- init (kmeans.rs:149-170; our rng): k distinct rows by a partial Fisher-Yates ------------
  std::vector<LloydState> h_states(B);
  for (int b = 0; b < B; ++b) {
    h_states[b].loss = std::numeric_limits<double>::max();
    h_states[b].last_loss = 0.0;
    h_states[b].adjusted = std::numeric_limits<float>::max();
    h_states[b].bf_cur = std::fmin(std::numeric_limits<float>::max(), p.balance_factor);
    h_states[b].iters = 0;
  }
  if (init_dev) {
    if (init_dev != centroids) d2d(centroids, init_dev, BK * ds);
    for (int b = 0; b < B; ++b) h_states[b].rng = p.seed + b;
  } else {
    // partial Fisher-Yates over the virtual array idx[i] = i, kept sparse (only touched slots are
    // stored): identical picks to the dense version, O(K) instead of O(n) host work per problem.
    // Sharded: the picks range over the GLOBAL rows (rank-major), see gather_init_owned_kernel.
    std::vector<uint32_t> rows(BK);
    std::unordered_map<uint64_t, uint32_t> moved;
    for (int b = 0; b < B; ++b) {
      SplitMix64 rng(p.seed + b);
      moved.clear();
      auto at = [&](uint64_t i) {
        auto it = moved.find(i);
        return it == moved.end() ? (uint32_t)i : it->second;
      };
      for (int i = 0; i < K; ++i) {
        const uint64_t j = i + rng.next() % (n_global - i);
        const uint32_t vi = at(i), vj = at(j);
        moved[i] = vj;
        moved[j] = vi;
        rows[(size_t)b * K + i] = vj;
      }
      h_states[b].rng = rng.s;  // split_clusters continues the same stream
    }
    DevBuf<uint32_t> rows_d(BK);
    h2d(rows_d.p, rows.data(), BK);
    LB2_LAUNCH("kmeans_init", gather_init_owned_kernel, cdiv(BK * ds, 256), 256, 0, x, ldx, ds, K, B, rows_d.p,
               (uint32_t)row_offset, (uint32_t)n, centroids);
    if (dist) comm_allreduce_f32(centroids, BK * ds, RedOp::Sum);
    sync_stream();  // rows (host vector) must outlive the copy
  }

  DevBuf<uint32_t> ids((size_t)B * n), last_row(BK);
  DevBuf<float> dists((size_t)B * n), radius(BK), bias;
  DevBuf<uint8_t> valid((size_t)B * n), active_d(B);
  DevBuf<double> losses(BK);
  DevBuf<uint64_t> cluster_sizes(BK);
  DevBuf<LloydState> states(B);
  cluster_sizes.zero();
  h2d(states.p, h_states.data(), B);
  LB2_CUDA(cudaMemsetAsync(active_d.p, 1, B, ctx().stream));
  // the trained model is in `centroids`; the loss and iteration count of every problem come back here
  auto read_back = [&]() {
    d2h(h_states.data(), states.p, B);
    sync_stream();
    if (loss_out) {
      loss_out->resize(B);
      for (int b = 0; b < B; ++b) (*loss_out)[b] = h_states[b].last_loss;
    }
    if (iters_out) {
      iters_out->resize(B);
      for (int b = 0; b < B; ++b) (*iters_out)[b] = h_states[b].iters;
    }
  };
  if (!small) {
    bias.alloc(K);
    bias.zero();  // iteration 1: cluster sizes are all zero -> bias 0
  }
  // multi-GPU: this rank's packed partial results and the gathered blobs of all ranks (see "ONE exchange")
  const ExchangeLayout xl = exchange_layout(BK, ds);
  DevBuf<uint8_t> blob, gathered;
  if (dist) {
    blob.alloc(xl.bytes);
    gathered.alloc(xl.bytes * (size_t)cm->nranks);
  }
  float* sums_p = dist ? reinterpret_cast<float*>(blob.p) : nullptr;
  DevBuf<uint8_t> hints((size_t)2 * B);  // order-independent-sum hints (update, loss) per problem
  LB2_CUDA(cudaMemsetAsync(hints.p, 1, (size_t)2 * B, ctx().stream));
  MemberSort ms;
  if (lloyd_small_ok(n, B, ds, K, dist) && (p.metric == METRIC_L2 || p.metric == METRIC_DOT) && ldx == ds) {
    // the whole run in ONE launch (lloyd_small_kernel)
    ms.counts.alloc(K);
    ms.offsets.alloc(K + 1);
    ms.members.alloc(n);
    DevBuf<float> bias16(16);
    bias16.zero();
    const int warp_update = (ds % 8 == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0) ? 1 : 0;
    const size_t smem = sizeof(float) * ((size_t)K * ds + 16 + SMALL_UPD_WARPS * UPD_TILE * 8) +
                        sizeof(uint32_t) * (SMALL_NT / 32 + 2) * (size_t)K;
#define LB2_SMALL(MET)                                                                                              \
    do {                                                                                                            \
      set_smem(lloyd_small_kernel<MET>, smem);                                                                      \
      LB2_LAUNCH("kmeans_small_fused", lloyd_small_kernel<MET>, SORT_CLUSTER, SMALL_NT, smem, x, (uint32_t)n, ds, K, \
                 centroids, p.balance_factor, p.tolerance, p.max_iters, ids.p, dists.p, valid.p, ms.counts.p,       \
                 ms.offsets.p, ms.members.p, losses.p, radius.p, last_row.p, cluster_sizes.p, bias16.p, states.p,   \
                 active_d.p, hints.p, warp_update);                                                                 \
    } while (0)
    if (p.metric == METRIC_DOT) LB2_SMALL(METRIC_DOT); else LB2_SMALL(METRIC_L2);
#undef LB2_SMALL
    read_back();
    return;
  }
  TcWorkspace tcws;
  TcPqWorkspace pqws;
  PqAssignWorkspace pqaws;  // the wide PQ routes' scratch, allocated by the eager first iteration
  DevBuf<float> rn2;
  const bool pq_tc = small && ldx == B * ds && tc_pq_supported(n, ldx, B, ds, K, p.metric, x);
  TcPqPrepArgs pq_prep;      // bm == nullptr unless the PQ tensor path is in use
  bool pq_prepared = false;  // true once an epilogue has written the next iteration's operands
  if (pq_tc) {  // per-sub-space norms of the (fixed) training rows, once
    rn2.alloc(n * B);
    tc_pq_residual_norms(x, nullptr, nullptr, n, B, nullptr, rn2.p);
    pq_prep = tc_pq_prep_args(B, ldx, &pqws);
  }
  sync_stream();
  const PollWords& words = PollWords::reset(B);  // (after the synchronise: no earlier epilogue still posts)
  // one Lloyd iteration = ~18 short kernels: membership, member sort, stats, update, scalar epilogue
  auto iteration = [&]() {
    if (!small) {
      assign_f32_ex(x, n, ds, centroids, K, p.metric, bias.p, ids.p, dists.p, valid.p, active_d.p, tcws);
    } else if (pq_tc) {
      // the first call prepares the operands itself; afterwards the epilogue of iteration i has
      // already written them for iteration i + 1
      tc_pq_assign(x, rn2.p, n, ldx, B, centroids, nullptr, nullptr, ids.p, dists.p, valid.p,
                   active_d.p, &pqws, /*prepared=*/pq_prepared);
      pq_prepared = true;
    } else {
      pq_assign_f32(x, n, ldx, B, ds, centroids, K, p.metric, nullptr, nullptr, nullptr, nullptr, ids.p, dists.p,
                    valid.p, active_d.p, &pqaws);
    }
    ms.run(ids.p, valid.p, n, K, B, active_d.p);
    // ds % 8 == 0 (and 16-byte aligned rows): warp-cooperative update, one warp per (b, cluster, 8 dims)
    const int warp_update = (ds % 8 == 0 && ldx % 4 == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0) ? 1 : 0;
    const unsigned ub = warp_update ? cdiv(BK * (uint64_t)(ds / 8), 4) : cdiv(BK * ds, 128);
    const unsigned sb = cdiv((uint64_t)BK * 32, 128);
    LB2_LAUNCH("kmeans_update_stats", update_stats_kernel, ub + sb, 128, 0, ub, x, ldx, ds, K, B, n,
               ms.members.p, ms.offsets.p, dist ? sums_p : centroids, dists.p, losses.p, radius.p,
               last_row.p, active_d.p, dist ? 0 : 1, warp_update, hints.p);
    if (dist) {  // SURVEY 8e: one exchange step per iteration over NVLink
      LB2_LAUNCH("kmeans_pack_partials", pack_partials_kernel, cdiv(BK, 256), 256, 0, blob.p, xl, BK, ms.counts.p,
                 radius.p, last_row.p, losses.p, (uint32_t)row_offset);
      comm_allgather_bytes(blob.p, gathered.p, xl.bytes);
      LB2_LAUNCH("kmeans_reduce_partials", reduce_partials_kernel, cdiv(BK * ds, 256), 256, 0, gathered.p, cm->nranks,
                 xl, BK, ds, K, centroids, ms.counts.p, radius.p, last_row.p, losses.p, active_d.p);
    }
    LB2_LAUNCH("kmeans_epilogue", epilogue_kernel, B, 256, 0, K, ds, n_global, p.balance_factor,
               p.tolerance, ms.counts.p, losses.p, radius.p, last_row.p, cluster_sizes.p,
               small ? nullptr : bias.p, K, centroids, states.p, active_d.p, pq_prep, words.device());
  };
  // The first iteration runs eagerly (allocates every workspace, sets kernel attributes); the
  // iteration is then captured ONCE into a CUDA graph and replayed, so that the loop is not bound
  // by ~18 host launches per iteration.  (Event profiling and LB2_TC_STATS need eager launches.)
  // (NCCL collectives are capturable; the sharded iteration is replayed from the graph like the local one)
  // (eager launches for the small splits of hierarchical training were tried and lose: 577 vs 481 ms for a
  // K = 8192 tree -- the loop is bound by host launch throughput, which is what the graph relieves)
  const bool use_graph = p.max_iters > 1 && !ctx().profiling && !(getenv("LB2_TC_STATS") && *getenv("LB2_TC_STATS")) &&
                         !(getenv("LB2_NO_GRAPH") && *getenv("LB2_NO_GRAPH"));
  struct Graph {  // the captured iteration, released on every way out of lloyd_train
    cudaGraph_t graph = nullptr;
    cudaGraphExec_t exec = nullptr;
    ~Graph() {
      if (exec) cudaGraphExecDestroy(exec);
      if (graph) cudaGraphDestroy(graph);
    }
  } g;
  uint64_t graph_nodes = 0;
  iteration();
  bool done = p.max_iters == 1;
  if (!done && use_graph) {
    const uint64_t l0 = ctx().launches;
    LB2_CUDA(cudaStreamBeginCapture(ctx().stream, cudaStreamCaptureModeThreadLocal));
    try {
      iteration();
    } catch (...) {
      cudaStreamEndCapture(ctx().stream, &g.graph);
      throw;
    }
    LB2_CUDA(cudaStreamEndCapture(ctx().stream, &g.graph));
    graph_nodes = ctx().launches - l0;
    ctx().launches = l0;
    LB2_CUDA(cudaGraphInstantiate(&g.exec, g.graph, 0));
  }
  for (int it = 2; it <= p.max_iters && !done; ++it) {
    if (g.exec) {
      LB2_CUDA(cudaGraphLaunch(g.exec, ctx().stream));
      ctx().launches += graph_nodes;
    } else {
      iteration();
    }
    done = words.done(B, (uint32_t)it - 1);  // (see PollWords)
  }
  read_back();
}

}  // namespace lb2
