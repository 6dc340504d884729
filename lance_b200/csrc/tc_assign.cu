// tc_assign.cu -- tensor-core FILTER for nearest-centroid assignment (sm_90a: wgmma + TMA + mbarrier).
//
// Replaces the O(n*K*d) part of  compute_membership_and_dist  (lance-index/src/vector/kmeans.rs:317-369)
// and  compute_partitions_with_dists (kmeans.rs:1275-1294)  WITHOUT changing a single output bit:
//
//   1. tc_filter_kernel: score(x, c) = x.c - (|c|^2 + bias_c)/2 for a 64-row x 256-centroid tile as a
//      TF32 GEMM (wgmma.mma_async tf32, f32 operands straight from TMA-swizzled shared memory, f32
//      accumulators in registers; two consumer warpgroups alternate).  The epilogue keeps the top-3 scores
//      of every row and classifies the row with a conservative error bound tau:
//        flag 0: top1 - top2 > tau   -> top1 IS the reference's argmin (no other centroid can win)
//        flag 1: top1 - top3 > tau   -> the winner is top1 or top2: decide with exact arithmetic
//        flag 2: otherwise (or NaN)  -> the row goes through the exact kernel (assign.cu)
//   2. rerank_kernel: for flag<=1 rows the reference-order f32 distance (exact.cuh) of the one or
//      two candidates, the reference's strict-< / lowest-index rule, and the exact distance output.
//   3. flag-2 rows are compacted and fed to assign_tile_kernel through a row-index list.
//
// Error bound (DESIGN.md section 5): TF32 keeps 11 significant bits, so each operand carries a
// relative error <= 2^-10 (truncation); |x.c - tf32(x).tf32(c)| <= 2^-9 * sum|x_i||c_i|
// <= 2^-10 (|x|^2 + |c|^2).  Two scores are compared, index packing perturbs by 2^-15 |score|, the
// f32 accumulation by far less: tau = 3 * 2^-10 * (|x|^2 + max_c |c|^2) covers 2x the bound with
// 20% to spare; below the normal f32 range the norm term has a floor (cert_tau, tc_common.cuh).  Whatever
// tau is, results stay exact as long as the bound holds; a larger tau only sends more rows to the exact paths.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "assign.cuh"
#include "common.cuh"
#include "exact.cuh"
#include "tc_assign.cuh"
#include "tc_common.cuh"

namespace lb2 {

namespace tc {

struct SmemLayout {
  // offsets from the 1024-aligned base
  uint32_t b_off, a_off, cnh_off, bar_off, total;
};
__host__ __device__ inline SmemLayout smem_layout(int nkc, int stages) {
  SmemLayout L;
  L.b_off = 0;
  L.a_off = nkc * B_CHUNK_BYTES;
  L.cnh_off = L.a_off + stages * A_STAGE_BYTES;
  L.bar_off = L.cnh_off + TN * 4;
  L.total = L.bar_off + (2 * MAX_STAGES + 1) * 8;
  return L;
}

// the classification of a row from its top-3 scores (flag 0: unique, 1: two candidates, 2: undecided)
__device__ __forceinline__ uint32_t verdict(float m1, float m2, float m3, float tau) {
  if (m1 - m2 > tau) return 0;
  if (m1 - m3 > tau) return 1;
  return 2;
}

// ------------------------------------------------------------------------------------------------
// the filter kernel (persistent, one CTA per SM)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(NUM_THREADS, 1)
tc_filter_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_c,
                 uint64_t n, int nkc, int stages, const float* __restrict__ cnh_g,
                 const float* __restrict__ row_norm2, const float* __restrict__ cn2_g,
                 uint32_t* __restrict__ res, const uint8_t* __restrict__ active, float tau_scale) {
  if (active && !active[0]) return;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_align1024(smem_raw);
  const SmemLayout L = smem_layout(nkc, stages);
  float* cnh = reinterpret_cast<float*>(smem + L.cnh_off);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L.bar_off);
  const uint32_t sb = smem_u32(smem);
  auto full_bar = [&](int s) { return smem_u32(&bars[s]); };
  auto empty_bar = [&](int s) { return smem_u32(&bars[MAX_STAGES + s]); };
  const uint32_t b_full = smem_u32(&bars[2 * MAX_STAGES]);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint64_t num_tiles = (n + TM - 1) / TM;

  __shared__ float s_cmax2;
  for (int i = threadIdx.x; i < TN; i += NUM_THREADS) cnh[i] = cnh_g[i];
  if (warp == 3) {  // max_c |c|^2 (a spare producer warp)
    float m = 0.0f;
    for (int i = lane; i < TN; i += 32) m = fmaxf(m, cn2_g[i]);
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, off));
    if (lane == 0) s_cmax2 = m;
  }
  if (threadIdx.x == 32) {
    for (int s = 0; s < stages; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 4);  // one arrival per consumer warp
    }
    mbar_init(b_full, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp < 4) {
    // ===== TMA producer =====
    setmaxnreg_dec<PRODUCER_REGS>();
    if (threadIdx.x == 0) {
      mbar_expect_tx(b_full, (uint32_t)nkc * B_CHUNK_BYTES);
      for (int kc = 0; kc < nkc; ++kc)
        tma_load_2d(sb + L.b_off + kc * B_CHUNK_BYTES, &map_c, b_full, kc * KC, 0);
      int s = 0;
      uint32_t ph = 0;
      for_units_producer(num_tiles, 1, [&](uint64_t tile, int) {
        for (int kc = 0; kc < nkc; ++kc) {
          mbar_wait_relaxed(empty_bar(s), ph ^ 1);
          mbar_expect_tx(full_bar(s), A_STAGE_BYTES);
          tma_load_2d(sb + L.a_off + s * A_STAGE_BYTES, &map_x, full_bar(s), kc * KC, (int)(tile * TM));
          if (++s == stages) { s = 0; ph ^= 1; }
        }
      });
    }
  } else {
    // ===== consumers: wgmma into registers, top-3 per row =====
    setmaxnreg_inc<CONSUMER_REGS>();
    const int w = (threadIdx.x >> 7) - 1;
    const float cmax2 = s_cmax2;
    float acc[128];
    mbar_wait(b_full, 0);
    for_units_consumer(num_tiles, 1, nkc, w, [&](uint64_t tile, int, uint64_t k, auto pass_turn) {
      mma_unit<0>(acc, nkc,
          [&](int kc, uint32_t& a_addr, uint32_t& b_addr) {
            const uint64_t kk = k + (uint64_t)kc;
            const int s = (int)(kk % (uint64_t)stages);
            mbar_wait(full_bar(s), (uint32_t)((kk / (uint64_t)stages) & 1));
            a_addr = sb + L.a_off + s * A_STAGE_BYTES;
            b_addr = sb + L.b_off + kc * B_CHUNK_BYTES;
            return s;
          },
          [&](int s) {
            __syncwarp();
            if (lane == 0) mbar_arrive(empty_bar(s));
          });
      pass_turn();
      float m[3];
      top3_frag(acc, cnh, m);
      if ((lane & 3) < 2) {  // lanes 0 / 1 of the quad write rows r0 / r0 + 8
        const uint64_t row = tile * TM + frag_row(lane & 1);
        if (row < n) {
          const uint32_t flag = verdict(m[0], m[1], m[2], cert_tau(tau_scale, row_norm2[row] + cmax2));
          res[row] = (__float_as_uint(m[0]) & 0xFFu) | ((__float_as_uint(m[1]) & 0xFFu) << 12) | (flag << 30);
        }
      }
    });
  }
}

// ------------------------------------------------------------------------------------------------
// general shapes: any d % 32 == 0 and any K.  The centroid matrix no longer fits in shared memory,
// so A (64 rows x 32 floats) AND B (256 centroids x 32 floats) chunks are streamed together through
// the TMA ring (40 KB per stage), centroid tiles of 256 are visited one after the other with the
// running top-3 (now with full indices) kept in registers by the warpgroup that owns the row tile.
// ------------------------------------------------------------------------------------------------
constexpr int GEN_STAGES = 5;
constexpr int GEN_STAGE_BYTES = A_STAGE_BYTES + B_CHUNK_BYTES;  // 40 KB

struct GenLayout {
  uint32_t stage_off, bar_off, total;
};
__host__ __device__ inline GenLayout gen_layout() {
  GenLayout L;
  L.stage_off = 0;
  L.bar_off = GEN_STAGES * GEN_STAGE_BYTES;
  L.total = L.bar_off + 2 * GEN_STAGES * 8;
  return L;
}

// insert (v, i) into the descending triple (g, gi)
__device__ __forceinline__ void top3_insert_idx(float v, uint32_t i, float* g, uint32_t* gi) {
  if (v > g[0]) {
    g[2] = g[1]; gi[2] = gi[1];
    g[1] = g[0]; gi[1] = gi[0];
    g[0] = v; gi[0] = i;
  } else if (v > g[1]) {
    g[2] = g[1]; gi[2] = gi[1];
    g[1] = v; gi[1] = i;
  } else if (v > g[2]) {
    g[2] = v; gi[2] = i;
  }
}

// OPK: operand kind (0 = f32 rows as TF32, 32 per 128-byte chunk; 1 = f16, 2 = bf16: 64 per chunk).
// MODE 0: top-3 per row + verdict (res / res_hi; top1_val[row] = best score of the rows left undecided).
// MODE 1: candidate pass over a list of undecided rows: every column with score >= thr[row] is appended to the
//         row's candidate slots (cand_cnt / cand), see cand_exact_kernel.
template <int OPK, int MODE>
__global__ void __launch_bounds__(NUM_THREADS, 1)
tc_filter_general_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_c,
                         uint64_t n, int nkc, int ntiles, const float* __restrict__ cnh_g,
                         const float* __restrict__ row_norm2, const float* __restrict__ cmax2_ptr,
                         uint32_t* __restrict__ res, uint32_t* __restrict__ res_hi,
                         const uint8_t* __restrict__ active, float tau_scale,
                         const uint32_t* __restrict__ n_dev, uint32_t n_cap, float* __restrict__ top1_val,
                         const float* __restrict__ thr_g, uint32_t* __restrict__ cand_cnt,
                         uint32_t* __restrict__ cand) {
  constexpr int KCE = OPK == 0 ? KC : 2 * KC;  // elements per 128-byte chunk
  if (active && !active[0]) return;
  if (n_dev) n = min(*n_dev, n_cap);  // refinement pass: the row count lives on the device
  if (n == 0) return;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_align1024(smem_raw);
  const GenLayout L = gen_layout();
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L.bar_off);
  const uint32_t sb = smem_u32(smem);
  auto full_bar = [&](int s) { return smem_u32(&bars[s]); };
  auto empty_bar = [&](int s) { return smem_u32(&bars[GEN_STAGES + s]); };
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint64_t num_tiles = (n + TM - 1) / TM;

  if (threadIdx.x == 32) {
    for (int s = 0; s < GEN_STAGES; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 4);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp < 4) {
    setmaxnreg_dec<PRODUCER_REGS>();
    if (threadIdx.x == 0) {  // ===== TMA producer: A and B chunk of every (row tile, centroid tile, k chunk)
      int s = 0;
      uint32_t ph = 0;
      for_units_producer(num_tiles, ntiles, [&](uint64_t tile, int nt) {
        for (int kc = 0; kc < nkc; ++kc) {
          mbar_wait_relaxed(empty_bar(s), ph ^ 1);
          mbar_expect_tx(full_bar(s), GEN_STAGE_BYTES);
          const uint32_t st = sb + L.stage_off + s * GEN_STAGE_BYTES;
          tma_load_2d(st, &map_x, full_bar(s), kc * KCE, (int)(tile * TM));
          tma_load_2d(st + A_STAGE_BYTES, &map_c, full_bar(s), kc * KCE, nt * TN);
          if (++s == GEN_STAGES) { s = 0; ph ^= 1; }
        }
      });
    }
  } else {
    setmaxnreg_inc<CONSUMER_REGS>();
    const int w = (threadIdx.x >> 7) - 1;
    const float cmax2 = *cmax2_ptr;
    const float ninf = __int_as_float(0xff800000);
    float acc[128];
    float g[3];      // running top-3 of the lane's fragment row over the centroid tiles seen
    uint32_t gi[3];
    for_units_consumer(num_tiles, ntiles, nkc, w, [&](uint64_t tile, int nt, uint64_t k, auto pass_turn) {
      mma_unit<OPK>(acc, nkc,
          [&](int kc, uint32_t& a_addr, uint32_t& b_addr) {
            const uint64_t kk = k + (uint64_t)kc;
            const int s = (int)(kk % GEN_STAGES);
            mbar_wait(full_bar(s), (uint32_t)((kk / GEN_STAGES) & 1));
            a_addr = sb + L.stage_off + s * GEN_STAGE_BYTES;
            b_addr = a_addr + A_STAGE_BYTES;
            return s;
          },
          [&](int s) {
            __syncwarp();
            if (lane == 0) mbar_arrive(empty_bar(s));
          });
      pass_turn();
      const float* cn = cnh_g + (size_t)nt * TN;
      const uint64_t row0 = tile * TM + frag_row(0), row1 = tile * TM + frag_row(1);
      if (MODE == 1) {
        const float thr[2] = {row0 < n ? thr_g[row0] : __int_as_float(0x7f800000),
                              row1 < n ? thr_g[row1] : __int_as_float(0x7f800000)};
        const uint64_t rc0 = row0 < n ? row0 : 0, rc1 = row1 < n ? row1 : 0;
        uint32_t* const cnt[2] = {cand_cnt + rc0, cand_cnt + rc1};
        uint32_t* const cs[2] = {cand + rc0 * CAND_SLOTS, cand + rc1 * CAND_SLOTS};
        cand_frag(acc, cn, thr, (uint32_t)nt * TN, cnt, cs);
        return;
      }
      float m[3];
      top3_frag(acc, cn, m);
      if (nt == 0) {
#pragma unroll
        for (int j = 0; j < 3; ++j) { g[j] = ninf; gi[j] = 0; }
      }
      const uint32_t base = (uint32_t)nt * TN;
#pragma unroll
      for (int j = 0; j < 3; ++j) top3_insert_idx(m[j], base + (__float_as_uint(m[j]) & 0xFFu), g, gi);
      if (nt == ntiles - 1 && (lane & 3) < 2) {  // row tile complete: lanes 0 / 1 of the quad write rows r0 / r0 + 8
        const uint64_t row = (lane & 1) ? row1 : row0;
        if (row < n) {
          const uint32_t flag = verdict(g[0], g[1], g[2], cert_tau(tau_scale, row_norm2[row] + cmax2));
          res[row] = gi[0] | (flag << 30);
          res_hi[row] = gi[1];
          if (top1_val && flag == 2) top1_val[row] = g[0];
        }
      }
    });
  }
}

// padded copy [Kp][d] (Kp multiple of 256), cnh, |c|^2 for any K: one warp per centroid
__global__ void prep_centroids_general_kernel(const float* __restrict__ c, int K, int Kp, int d,
                                              const float* __restrict__ bias, float* __restrict__ cpad,
                                              float* __restrict__ cnh, float* __restrict__ cn2,
                                              uint32_t* __restrict__ fb_count) {
  const int k = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (blockIdx.x == 0 && threadIdx.x == 0) { fb_count[0] = 0; fb_count[1] = 0; fb_count[2] = 0; fb_count[3] = 0; }
  if (k >= Kp) return;
  float n2 = 0.0f;
  for (int e = lane; e < d; e += 32) {
    const float v = k < K ? c[(size_t)k * d + e] : 0.0f;
    cpad[(size_t)k * d + e] = v;
    n2 += v * v;
  }
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) n2 += __shfl_xor_sync(0xffffffffu, n2, off);
  if (lane == 0) {
    cnh[k] = k < K ? -0.5f * (n2 + (bias ? bias[k] : 0.0f)) : -3.0e38f;
    cn2[k] = (k < K && n2 == n2) ? n2 : 0.0f;
  }
}
__global__ void max_reduce_kernel(const float* __restrict__ v, int n, float* __restrict__ out) {
  __shared__ float s[32];
  float m = 0.0f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) m = fmaxf(m, v[i]);
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, off));
  if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    float r = 0.0f;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) r = fmaxf(r, s[i]);
    *out = r;
  }
}

// ------------------------------------------------------------------------------------------------
// preparation kernels
// ------------------------------------------------------------------------------------------------
// padded copy of the centroids [TN][d] (zero rows past K), cnh[k] = -(|c_k|^2 + bias_k)/2 (-3e38 pads),
// cmax2 = max_k |c_k|^2 (plain f32; any rounding is inside the error budget)
__global__ void prep_centroids_kernel(const float* __restrict__ c, int K, int d,
                                      const float* __restrict__ bias, float* __restrict__ cpad,
                                      float* __restrict__ cnh, float* __restrict__ cn2,
                                      float* __restrict__ cT, int Kp, uint32_t* __restrict__ fb_count) {
  // grid = TN/8 blocks of 256 threads: one warp per (padded) centroid row.  Also writes the
  // transposed NaN-padded copy cT[e][Kp] used by the exact fallback kernel and resets the
  // fallback-row counter, so one launch prepares everything the iteration needs.
  const int k = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (blockIdx.x == 0 && threadIdx.x == 0) { fb_count[0] = 0; fb_count[1] = 0; fb_count[2] = 0; fb_count[3] = 0; }
  float n2 = 0.0f;
  for (int e = lane; e < d; e += 32) {
    const float v = k < K ? c[(size_t)k * d + e] : 0.0f;
    cpad[(size_t)k * d + e] = v;
    if (k < Kp) cT[(size_t)e * Kp + k] = k < K ? v : __int_as_float(0x7fc00000);
    n2 += v * v;
  }
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) n2 += __shfl_xor_sync(0xffffffffu, n2, off);
  if (lane == 0) {
    // pads: a huge negative FINITE score (an inf would turn into NaN when the index is packed in)
    cnh[k] = k < K ? -0.5f * (n2 + (bias ? bias[k] : 0.0f)) : -3.0e38f;
    cn2[k] = (k < K && n2 == n2) ? n2 : 0.0f;
  }
}

// |x|^2 per row, 16 lanes per row (plain f32, inside the error budget; NaN/Inf propagate -> flag 2)
__global__ void row_norm_kernel(const float* __restrict__ x, uint64_t n, int d, float* __restrict__ out) {
  const uint64_t hw = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 4;
  const int l = threadIdx.x & 15;
  if (hw >= n) return;  // whole half-warp exits together
  const float* v = x + hw * d;
  float s = 0.0f;
  for (int e = l * 4; e < d; e += 64) {
    const float4 f = *reinterpret_cast<const float4*>(v + e);
    s += f.x * f.x + f.y * f.y + f.z * f.z + f.w * f.w;
  }
  const unsigned mask = 0xffffu << (16 * ((threadIdx.x >> 4) & 1));
#pragma unroll
  for (int off = 8; off >= 1; off >>= 1) s += __shfl_xor_sync(mask, s, off, 16);
  if (l == 0) out[hw] = s;
}

// ------------------------------------------------------------------------------------------------
// exact re-rank of the one or two surviving candidates (16 lanes per row; lane l owns the
// reference's lane-accumulator l, l2.rs:82-88), flag-2 rows are appended to the fallback list
// ------------------------------------------------------------------------------------------------
// With `src_list` the kernel serves the refinement pass: entry i of res / res_hi belongs to row
// src_list[i], i < min(*src_count, src_cap); list entries beyond src_cap (no room in the refinement
// buffers) are forwarded to the overflow list (ovf_rows) untouched.
__global__ void __launch_bounds__(256)
rerank_kernel(const float* __restrict__ x, uint64_t n, int d, const float* __restrict__ cent,
              const float* __restrict__ bias, const uint32_t* __restrict__ res,
              const uint32_t* __restrict__ res_hi, int need_dist,
              uint32_t* __restrict__ part, float* __restrict__ dist, uint8_t* __restrict__ valid,
              uint32_t* __restrict__ fb_rows, uint32_t* __restrict__ fb_count,
              const uint8_t* __restrict__ active, const uint32_t* __restrict__ src_list,
              const uint32_t* __restrict__ src_count, uint32_t src_cap, const float* __restrict__ val_in,
              float* __restrict__ val_out, uint32_t* __restrict__ ovf_rows, uint32_t* __restrict__ ovf_count) {
  if (active && !active[0]) return;
  const int l = threadIdx.x & 15;
  const unsigned mask = 0xffffu << (16 * ((threadIdx.x >> 4) & 1));
  uint64_t total = n;
  if (src_list) {
    total = *src_count;
    need_dist = 1;  // the first pass left these rows without any output
  }
  for (uint64_t idx = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 4; idx < total;
       idx += ((uint64_t)gridDim.x * blockDim.x) >> 4) {
    uint64_t row = idx;
    if (src_list) {
      row = src_list[idx];
      if (idx >= src_cap) {  // overflow of the refinement buffers: straight to the full-K exact scan
        if (l == 0) ovf_rows[atomicAdd(ovf_count, 1u)] = (uint32_t)row;
        continue;
      }
    }
    const uint32_t r = res[idx];
    const uint32_t flag = r >> 30;
    const uint32_t i1 = res_hi ? (r & 0x3FFFFFFFu) : (r & 0xFFFu);
    const uint32_t i2 = res_hi ? res_hi[idx] : ((r >> 12) & 0xFFFu);
    if (flag == 2) {
      if (l == 0) {
        fb_rows[atomicAdd(fb_count, 1u)] = (uint32_t)row;
        if (val_out) val_out[row] = val_in[idx];  // best score of the pass that just ran, for the candidate pass
      }
      continue;
    }
    if (flag == 0 && !need_dist) {
      if (l == 0) {
        part[row] = i1;
        if (valid) valid[row] = 1;
      }
      continue;
    }
    const float* xv = x + row * d;
    const int ncand = flag == 0 ? 1 : 2;
    float best_key = __int_as_float(0x7f800000), best_val = best_key;
    uint32_t best_idx = 0xffffffffu;
    for (int c = 0; c < ncand; ++c) {
      const uint32_t ci = c == 0 ? i1 : i2;
      const float* cv = cent + (size_t)ci * d;
      float acc = 0.0f;
      for (int e = l; e < d; e += 16) acc = f_add(acc, sq_diff(xv[e], cv[e]));
      float t = 0.0f;
#pragma unroll
      for (int qq = 0; qq < 16; ++qq) t = f_add(t, __shfl_sync(mask, acc, qq, 16));
      const float v = f_add(0.0f, t);
      const float key = bias ? f_add(v, bias[ci]) : v;
      if (key < best_key || (key == best_key && ci < best_idx)) {
        best_key = key; best_val = v; best_idx = ci;
      }
    }
    if (l == 0) {
      const bool ok = best_idx != 0xffffffffu;
      part[row] = ok ? best_idx : 0u;
      if (dist) dist[row] = ok ? best_val : __int_as_float(0x7fc00000);
      if (valid) valid[row] = ok ? 1 : 0;
    }
  }
}

// ---- refinement of the rows the TF32 filter left undecided ------------------------------------------
// A second tensor-core pass over those rows only, with the operands split into TF32-exact pieces
//     x = xh + xl (+ <= 2^-22 |x|),   c = ch + cl (+ <= 2^-22 |c|),     x.c ~ xh.ch + xh.cl + xl.ch,
// i.e. the SAME filter kernel run on A' = [xh | xh | xl] (gathered, 3d wide) and B' = [ch | cl | ch]: every
// product is exact in TF32, what is dropped is <= 1.51 * 2^-22 (|x|^2 + |c|^2), the f32 accumulation over
// 3d/8 MMA steps <= 3d * 2^-26 (|x|^2 + |c|^2) (two ulps per step on the running magnitude), packing the
// column index into the low mantissa byte 2^-16 (|x|^2 + 2|c|^2).  tau' = (2^-13 + 3d * 2^-25)(|x|^2 +
// max|c|^2) covers twice their sum; it is ~1/20 .. 1/45 of the first pass's tau, so all but a sliver of the
// undecided rows become unique / two-candidate rows and only true near-ties reach the full-K exact scan.
__device__ __forceinline__ float rn_tf32(float v) {  // round to nearest-even TF32 (10 explicit mantissa bits)
  uint32_t b = __float_as_uint(v);
  if ((b & 0x7f800000u) == 0x7f800000u) return v;  // Inf / NaN
  b += 0xFFFu + ((b >> 13) & 1u);
  return __uint_as_float(b & 0xFFFFE000u);
}
__global__ void gather_split_kernel(const float* __restrict__ x, int d, const float* __restrict__ row_norm2,
                                    const uint32_t* __restrict__ list, const uint32_t* __restrict__ count,
                                    uint32_t cap, float* __restrict__ a3, float* __restrict__ rn2c,
                                    const uint8_t* __restrict__ active, const float* __restrict__ top1_val,
                                    float tau_scale, const float* __restrict__ cmax2, float* __restrict__ thr,
                                    uint32_t* __restrict__ cand_cnt) {
  if (active && !active[0]) return;
  const uint32_t cnt = min(*count, cap);
  const int d4 = d >> 2;
  for (uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; g < (uint64_t)cnt * d4;
       g += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t i = (uint32_t)(g / d4);
    const int e = (int)(g % d4) * 4;
    const uint32_t row = list[i];
    const float4 v = *reinterpret_cast<const float4*>(x + (size_t)row * d + e);
    float4 h, lo;
    h.x = rn_tf32(v.x); h.y = rn_tf32(v.y); h.z = rn_tf32(v.z); h.w = rn_tf32(v.w);
    lo.x = rn_tf32(v.x - h.x); lo.y = rn_tf32(v.y - h.y); lo.z = rn_tf32(v.z - h.z); lo.w = rn_tf32(v.w - h.w);
    float* o = a3 + (size_t)i * 3 * d + e;
    *reinterpret_cast<float4*>(o) = h;
    *reinterpret_cast<float4*>(o + d) = h;
    *reinterpret_cast<float4*>(o + 2 * d) = lo;
    if (e == 0) {
      const float rn = row_norm2[row];
      rn2c[i] = rn;
      if (thr) {  // candidate pass: everything within tau of the best score the previous pass saw
        thr[i] = top1_val[row] - cert_tau(tau_scale, rn + *cmax2);
        cand_cnt[i] = 0;
      }
    }
  }
}
// the same for 16-bit rows (products of f16 / bf16 operands are exact: no split)
__global__ void gather16_kernel(const uint16_t* __restrict__ x, int d, const float* __restrict__ row_norm2,
                                const uint32_t* __restrict__ list, const uint32_t* __restrict__ count,
                                uint32_t cap, uint16_t* __restrict__ a16, float* __restrict__ rn2c,
                                const uint8_t* __restrict__ active, const float* __restrict__ top1_val,
                                float tau_scale, const float* __restrict__ cmax2, float* __restrict__ thr,
                                uint32_t* __restrict__ cand_cnt) {
  if (active && !active[0]) return;
  const uint32_t cnt = min(*count, cap);
  const int d8 = d >> 3;
  for (uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; g < (uint64_t)cnt * d8;
       g += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t i = (uint32_t)(g / d8);
    const int e = (int)(g % d8) * 8;
    const uint32_t row = list[i];
    *reinterpret_cast<uint4*>(a16 + (size_t)i * d + e) = *reinterpret_cast<const uint4*>(x + (size_t)row * d + e);
    if (e == 0) {
      const float rn = row_norm2[row];
      rn2c[i] = rn;
      thr[i] = top1_val[row] - cert_tau(tau_scale, rn + *cmax2);
      cand_cnt[i] = 0;
    }
  }
}
// padded centroids [Kp][d] as f16 / bf16; *inexact is raised when a value does not survive the conversion (the
// 16-bit operand path needs the model to be exactly representable -- models trained on such columns are)
__global__ void prep16_kernel(const float* __restrict__ cpad, size_t total, int bf16, uint16_t* __restrict__ out,
                              uint32_t* __restrict__ inexact) {
  const size_t g = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= total) return;
  const float v = cpad[g];
  float back;
  uint16_t bits;
  if (bf16) {
    const __nv_bfloat16 h = __float2bfloat16_rn(v);
    bits = __bfloat16_as_ushort(h);
    back = __bfloat162float(h);
  } else {
    const __half h = __float2half_rn(v);
    bits = __half_as_ushort(h);
    back = __half2float(h);
  }
  out[g] = bits;
  if (!(back == v) && v == v) atomicOr(inexact, 1u);  // (NaN centroids stay NaN)
}

// exact decision among the candidates of one undecided row (16 lanes per row, reference arithmetic and the
// strict-< / lowest-index rule, like rerank_kernel).  Rows without a candidate (NaN / Inf rows) or with more than
// CAND_SLOTS (duplicated centroids) go to the full-K exact scan.
__global__ void __launch_bounds__(256)
cand_exact_kernel(const float* __restrict__ x, int d, const float* __restrict__ cent, const float* __restrict__ bias,
                  const uint32_t* __restrict__ list, const uint32_t* __restrict__ count, uint32_t cap,
                  const uint32_t* __restrict__ cand_cnt, const uint32_t* __restrict__ cand,
                  uint32_t* __restrict__ part, float* __restrict__ dist, uint8_t* __restrict__ valid,
                  uint32_t* __restrict__ fb_rows, uint32_t* __restrict__ fb_count,
                  const uint8_t* __restrict__ active) {
  if (active && !active[0]) return;
  const int l = threadIdx.x & 15;
  const unsigned mask = 0xffffu << (16 * ((threadIdx.x >> 4) & 1));
  const uint32_t total = min(*count, cap);
  for (uint64_t idx = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 4; idx < total;
       idx += ((uint64_t)gridDim.x * blockDim.x) >> 4) {
    const uint32_t row = list[idx];
    const uint32_t nc = cand_cnt[idx];
    if (nc == 0 || nc > (uint32_t)CAND_SLOTS) {
      if (l == 0) fb_rows[atomicAdd(fb_count, 1u)] = row;
      continue;
    }
    const float* xv = x + (size_t)row * d;
    float best_key = __int_as_float(0x7f800000), best_val = best_key;
    uint32_t best_idx = 0xffffffffu;
    for (uint32_t c = 0; c < nc; ++c) {
      const uint32_t ci = cand[idx * CAND_SLOTS + c];
      const float* cv = cent + (size_t)ci * d;
      float acc = 0.0f;
      for (int e = l; e < d; e += 16) acc = f_add(acc, sq_diff(xv[e], cv[e]));
      float t = 0.0f;
#pragma unroll
      for (int qq = 0; qq < 16; ++qq) t = f_add(t, __shfl_sync(mask, acc, qq, 16));
      const float v = f_add(0.0f, t);
      const float key = bias ? f_add(v, bias[ci]) : v;
      if (key < best_key || (key == best_key && ci < best_idx)) {
        best_key = key; best_val = v; best_idx = ci;
      }
    }
    if (best_idx == 0xffffffffu) {  // every candidate distance was NaN / +inf: let the exact scan decide
      if (l == 0) fb_rows[atomicAdd(fb_count, 1u)] = row;
      continue;
    }
    if (l == 0) {
      part[row] = best_idx;
      if (dist) dist[row] = best_val;
      if (valid) valid[row] = 1;
    }
  }
}
// B' = [ch | cl | ch] from the padded centroid copy [Kp][d] (pad rows are zero)
__global__ void split_centroids_kernel(const float* __restrict__ cpad, size_t total, int d, float* __restrict__ b3) {
  const size_t g = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= total) return;
  const size_t k = g / d;
  const int e = (int)(g % d);
  const float v = cpad[g], h = rn_tf32(v), lo = rn_tf32(v - h);
  float* o = b3 + k * 3 * d + e;
  o[0] = h;
  o[d] = lo;
  o[2 * d] = h;
}

// list entries beyond the gather capacity -> the full-K exact list
__global__ void forward_overflow_kernel(const uint32_t* __restrict__ list, const uint32_t* __restrict__ count, uint32_t cap,
                                        uint32_t* __restrict__ out, uint32_t* __restrict__ out_count,
                                        const uint8_t* __restrict__ active) {
  if (active && !active[0]) return;
  const uint32_t total = *count;
  for (uint64_t i = (uint64_t)cap + (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (uint64_t)gridDim.x * blockDim.x)
    out[atomicAdd(out_count, 1u)] = list[i];
}

}  // namespace tc

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
// Shared by every host thread: the first calls of the tensor-core filter may come from several threads at once, so
// the pointer is a function-local static initialised once (C++ makes that thread-safe).  A failed lookup throws out
// of the initialiser, which leaves the static uninitialised and lets the next call try again.
static PFN_cuTensorMapEncodeTiled_v12000 get_encode_fn() {
  static const PFN_cuTensorMapEncodeTiled_v12000 fn = [] {
    cudaDriverEntryPointQueryResult qres;
    void* p = nullptr;
    LB2_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres));
    if (!p || qres != cudaDriverEntryPointSuccess) fail(LB2_CUDA_ERROR, "cuTensorMapEncodeTiled not available");
    return reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(p);
  }();
  return fn;
}

CUtensorMap make_map_2d(const float* base, uint64_t rows, uint64_t cols, uint32_t box_rows) {
  CUtensorMap m;
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {cols * sizeof(float)};
  cuuint32_t box[2] = {(cuuint32_t)tc::KC, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = get_encode_fn()(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), dims, strides,
                               box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                               CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) fail(LB2_CUDA_ERROR, "cuTensorMapEncodeTiled failed (%d)", (int)r);
  return m;
}

CUtensorMap make_map_2d_16(const void* base, bool bf16, uint64_t rows, uint64_t cols, uint32_t box_rows) {
  CUtensorMap m;
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {cols * 2};
  cuuint32_t box[2] = {(cuuint32_t)(2 * tc::KC), box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = get_encode_fn()(&m, bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2,
                               const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                               CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) fail(LB2_CUDA_ERROR, "cuTensorMapEncodeTiled (16-bit) failed (%d)", (int)r);
  return m;
}

static bool tc_resident_shape(int d, int K) { return d <= 128 && K <= tc::TN; }
constexpr float TAU_TF32 = 0.0029296875f;  // 3 * 2^-10, see the header comment

// 16-bit operand pass: tau covers the index packing (2^-15 |score| per compared score) and the f32 accumulation
// inside the tensor core (d/16 steps of 16 exact products each; every addend may lose one unit of the running
// magnitude) -- twice their sum, as for the TF32 pass
static float tau16_scale(int d) { return 1.220703125e-4f + (float)d * 1.1920929e-7f; }  // 2^-13 + d * 2^-23
static float tau3x_scale(int d3) { return 1.220703125e-4f + (float)d3 * 2.98023224e-8f; }  // 2^-13 + 3d * 2^-25

template <int OPK, int MODE>
static void launch_general(unsigned grid, size_t smem, const CUtensorMap& ma, const CUtensorMap& mb, uint64_t n, int nkc,
                           int ntiles, const float* cnh, const float* rn2, const float* cmax2, uint32_t* res,
                           uint32_t* res_hi, const uint8_t* active, float tau, const uint32_t* n_dev, uint32_t n_cap,
                           float* top1_val, const float* thr, uint32_t* cand_cnt, uint32_t* cand, const char* name) {
  using namespace tc;
  set_smem(tc_filter_general_kernel<OPK, MODE>, smem);
  LB2_LAUNCH(name, (tc_filter_general_kernel<OPK, MODE>), grid, NUM_THREADS, smem, ma, mb, n, nkc, ntiles, cnh, rn2, cmax2,
             res, res_hi, active, tau, n_dev, n_cap, top1_val, thr, cand_cnt, cand);
}
static void launch_general_dyn(int opk, int mode, unsigned grid, size_t smem, const CUtensorMap& ma, const CUtensorMap& mb,
                               uint64_t n, int nkc, int ntiles, const float* cnh, const float* rn2, const float* cmax2,
                               uint32_t* res, uint32_t* res_hi, const uint8_t* active, float tau, const uint32_t* n_dev,
                               uint32_t n_cap, float* top1_val, const float* thr, uint32_t* cand_cnt, uint32_t* cand,
                               const char* name) {
#define LB2_GEN(O, M)                                                                                                \
  launch_general<O, M>(grid, smem, ma, mb, n, nkc, ntiles, cnh, rn2, cmax2, res, res_hi, active, tau, n_dev, n_cap, \
                       top1_val, thr, cand_cnt, cand, name)
  if (mode == 0) {
    if (opk == 0) LB2_GEN(0, 0); else if (opk == 1) LB2_GEN(1, 0); else LB2_GEN(2, 0);
  } else {
    if (opk == 0) LB2_GEN(0, 1); else if (opk == 1) LB2_GEN(1, 1); else LB2_GEN(2, 1);
  }
#undef LB2_GEN
}

// Rows the first pass left undecided (ws.fb_rows / fb_count[0]).
//   f32 rows (first pass TF32):  3xTF32 top-3 pass over the list -> exact re-rank of what it settles; the rest
//       (fb_rows2 / fb_count[1]) -> 3xTF32 CANDIDATE pass: all columns within tau' of the best score -> exact
//       decision among those candidates (cand_exact_kernel).
//   16-bit rows (first pass already exact up to the accumulation): the candidate pass directly on the list.
//   What is still open (no candidate: NaN / Inf rows; > CAND_SLOTS candidates: duplicated centroids; rows that did
//   not fit the gather buffers) runs through the full-K exact kernel (fb_rows3 / fb_count[2]).
// `cpad` = zero-padded centroids [Kp][d], cnh / cmax2 as prepared for the first pass; x16 / cpad16 for OPK != 0.
// Returns whether the refinement passes ran (otherwise every undecided row took the full-K exact scan).
static bool tc_refine_and_fallback(const float* x, uint64_t n, int d, const float* cent, int K, int Kp,
                                   const float* bias, const float* cpad, const float* cnh, const float* cmax2,
                                   uint32_t* part, float* dist, uint8_t* valid, const uint8_t* active,
                                   TcWorkspace& ws, bool cT_ready, int opk, const void* x16) {
  using namespace tc;
  const char* e_force = getenv("LB2_FORCE_REFINE");
  const bool force = e_force && *e_force;
  const int d3 = 3 * d;
  const size_t row_bytes = opk ? (size_t)d * 2 : (size_t)d3 * 4;
  // room for 1/8 of the rows, at most ~1.5 GB of gathered rows (callers chunk large inputs, assign_f32_ex);
  // list entries beyond the capacity go straight to the exact kernel
  const uint32_t cap = (uint32_t)std::min<uint64_t>(std::min<uint64_t>(n, std::max<uint64_t>(4096, n / 8)),
                                                    std::max<uint64_t>(TM, ((size_t)3 << 29) / row_bytes));
  const GenLayout L = gen_layout();
  const size_t smem = L.total + 1024;
  // worth its launches only when the first pass was a large one (the undecided list of a 65 536-row training
  // call is a few hundred rows: the exact kernel finishes them sooner)
  const bool refine = smem <= ctx().smem_optin && (force || (uint64_t)n * (uint64_t)K >= (1ull << 26) || (uint64_t)n * (uint64_t)K * (uint64_t)d >= (1ull << 32));
  if (!refine) {
    assign_rows_f32(x, n, d, cent, K, METRIC_L2, bias, ws.fb_rows.p, ws.fb_count.p, part, dist, valid, active, ws,
                    cT_ready);
    return false;
  }
  const size_t a_floats = ((size_t)cap * row_bytes + 3) / 4;
  if (ws.a3.n < a_floats) ws.a3.alloc(a_floats);
  if (ws.rn2c.n < (size_t)2 * cap) ws.rn2c.alloc((size_t)2 * cap);  // |x|^2 and the candidate threshold
  if (ws.res2.n < (size_t)3 * cap) ws.res2.alloc((size_t)3 * cap);  // verdicts (2) + best score of the pass
  if (ws.fb_rows2.n < 2 * n) ws.fb_rows2.alloc(2 * n);              // lists 2 and 3
  if (ws.cand.n < (size_t)cap * (CAND_SLOTS + 1)) ws.cand.alloc((size_t)cap * (CAND_SLOTS + 1));
  if (ws.top1_val.n < n) ws.top1_val.alloc(n);
  float* thr = ws.rn2c.p + cap;
  uint32_t* cand_cnt = ws.cand.p;
  uint32_t* cand = ws.cand.p + cap;
  uint32_t* list1 = ws.fb_rows.p;
  uint32_t* list2 = ws.fb_rows2.p;
  uint32_t* list3 = ws.fb_rows2.p + n;
  uint32_t* cnt = ws.fb_count.p;  // [0] list 1, [1] list 2, [2] list 3
  const unsigned sms = (unsigned)ctx().num_sms;
  const unsigned grid = (unsigned)std::min<uint64_t>(cdiv(cap, TM), (uint64_t)sms);
  const unsigned ggrid = (unsigned)std::min<uint64_t>(cdiv((uint64_t)cap * (d / 4), 256), 8 * sms);
  const unsigned rgrid = (unsigned)std::min<uint64_t>(cdiv((uint64_t)cap * 16, 256), 8 * sms);
  if (opk) {
    const float tau = tau16_scale(d);
    uint16_t* a16 = reinterpret_cast<uint16_t*>(ws.a3.p);
    LB2_LAUNCH("tc_refine_gather", gather16_kernel, ggrid, 256, 0, static_cast<const uint16_t*>(x16), d, ws.row_norm2.p,
               list1, cnt, cap, a16, ws.rn2c.p, active, ws.top1_val.p, tau, cmax2, thr, cand_cnt);
    const CUtensorMap map_a = make_map_2d_16(a16, opk == 2, cap, d, TM);
    const CUtensorMap map_b = make_map_2d_16(ws.cpad16.p, opk == 2, Kp, d, TN);
    launch_general_dyn(opk, 1, grid, smem, map_a, map_b, (uint64_t)cap, d / (2 * KC), Kp / TN, cnh, ws.rn2c.p, cmax2,
                       nullptr, nullptr, active, tau, cnt, cap, nullptr, thr, cand_cnt, cand, "tc_candidates");
    // rows beyond the gather capacity: rerank_kernel's list mode only forwards them (res is not read for them)
    LB2_LAUNCH("tc_candidates_exact", cand_exact_kernel, rgrid, 256, 0, x, d, cent, bias, list1, cnt, cap, cand_cnt, cand,
               part, dist, valid, list3, cnt + 2, active);
    LB2_LAUNCH("tc_candidates_exact", forward_overflow_kernel, 8 * sms, 256, 0, list1, cnt, cap, list3, cnt + 2, active);
  } else {
    if (ws.b3.n < (size_t)Kp * d3) ws.b3.alloc((size_t)Kp * d3);
    const float tau2 = tau3x_scale(d3);
    LB2_LAUNCH("tc_refine_gather", gather_split_kernel, ggrid, 256, 0, x, d, ws.row_norm2.p, list1, cnt, cap, ws.a3.p,
               ws.rn2c.p, active, (const float*)nullptr, 0.0f, (const float*)nullptr, (float*)nullptr,
               (uint32_t*)nullptr);
    LB2_LAUNCH("tc_refine_gather", split_centroids_kernel, cdiv((uint64_t)Kp * d, 256), 256, 0, cpad, (size_t)Kp * d, d,
               ws.b3.p);
    const CUtensorMap map_a = make_map_2d(ws.a3.p, cap, d3, TM);
    const CUtensorMap map_b = make_map_2d(ws.b3.p, Kp, d3, TN);
    float* val2 = reinterpret_cast<float*>(ws.res2.p + 2 * (size_t)cap);
    launch_general_dyn(0, 0, grid, smem, map_a, map_b, (uint64_t)cap, d3 / KC, Kp / TN, cnh, ws.rn2c.p, cmax2, ws.res2.p,
                       ws.res2.p + cap, active, tau2, cnt, cap, val2, nullptr, nullptr, nullptr, "tc_refine_filter");
    LB2_LAUNCH("tc_refine_rerank", rerank_kernel, (unsigned)std::min<uint64_t>(cdiv((uint64_t)n * 16, 256), 8 * sms), 256, 0,
               x, n, d, cent, bias, ws.res2.p, (const uint32_t*)(ws.res2.p + cap), 1, part, dist, valid, list2, cnt + 1,
               active, (const uint32_t*)list1, (const uint32_t*)cnt, cap, (const float*)val2, ws.top1_val.p, list3,
               cnt + 2);
    // candidate pass over what the 3xTF32 top-3 left open (list 2 <= cap entries)
    LB2_LAUNCH("tc_refine_gather", gather_split_kernel, ggrid, 256, 0, x, d, ws.row_norm2.p, list2, cnt + 1, cap, ws.a3.p,
               ws.rn2c.p, active, (const float*)ws.top1_val.p, tau2, cmax2, thr, cand_cnt);
    launch_general_dyn(0, 1, grid, smem, map_a, map_b, (uint64_t)cap, d3 / KC, Kp / TN, cnh, ws.rn2c.p, cmax2, nullptr,
                       nullptr, active, tau2, cnt + 1, cap, nullptr, thr, cand_cnt, cand, "tc_candidates");
    LB2_LAUNCH("tc_candidates_exact", cand_exact_kernel, rgrid, 256, 0, x, d, cent, bias, list2, cnt + 1, cap, cand_cnt,
               cand, part, dist, valid, list3, cnt + 2, active);
  }
  assign_rows_f32(x, n, d, cent, K, METRIC_L2, bias, list3, cnt + 2, part, dist, valid, active, ws, cT_ready);
  return true;
}

bool tc_assign_supported(uint64_t n, int d, int K, int metric, const float* x) {
  if (getenv("LB2_DISABLE_TC") && *getenv("LB2_DISABLE_TC")) return false;
  return metric == METRIC_L2 && d % tc::KC == 0 && d >= 32 && d <= 4096 && K >= 2 && K < (1 << 28) &&
         n >= 1 && n < (1ull << 31) && (reinterpret_cast<uintptr_t>(x) & 15) == 0;
}

// ---- native 16-bit rows ----------------------------------------------------------------------------------------
// The chunk loops of api.cu pass, next to the f32 view x of a chunk, the same rows in their own f16 / bf16 type
// (x16).  If the model is exactly representable in that type (models trained on such columns are, round_model) the
// filter passes of the general shape read the 16-bit rows directly: f16 / bf16 wgmma at twice the TF32 rate, exact
// products, a tau ~10x smaller.  The exact kernels keep reading x (conversion is exact).
// Returns the operand kind of x16 (1: f16, 2: bf16), or 0 when the filter reads x.
static int native_opk(const void* x16, int x16_dtype, int d) {
  const char* off = getenv("LB2_NO_NATIVE16");
  if (!x16 || (off && *off) || d % (2 * tc::KC) != 0 || (reinterpret_cast<uintptr_t>(x16) & 15)) return 0;
  return x16_dtype == LB2_F16 ? 1 : x16_dtype == LB2_BF16 ? 2 : 0;
}

// Two shapes: resident (d <= 128, K <= TN: tc_filter_kernel keeps the whole centroid tile in shared memory) and
// general (tc_filter_general_kernel streams centroid tiles of TN with the rows, running top-3 over the tiles).
void tc_assign_f32(const float* x, uint64_t n, int d, const float* cent, int K, const float* bias,
                   uint32_t* part, float* dist, uint8_t* valid, const uint8_t* active,
                   TcWorkspace& ws, const void* x16, int x16_dtype) {
  using namespace tc;
  const bool resident = tc_resident_shape(d, K);
  const int ntiles = (K + TN - 1) / TN, Kp = ntiles * TN;
  int stages = MAX_STAGES;  // resident: as many TMA stages as fit next to the centroid tile
  size_t smem = gen_layout().total + 1024;
  if (resident) {
    SmemLayout L = smem_layout(d / KC, stages);
    while (stages > 2 && L.total + 1024 > ctx().smem_optin) L = smem_layout(d / KC, --stages);
    smem = L.total + 1024;
  }
  if (smem > ctx().smem_optin) fail(LB2_UNSUPPORTED, "tc_assign: shared memory");
  if (ws.cpad.n < (size_t)Kp * d) ws.cpad.alloc((size_t)Kp * d);
  if (ws.cnh.n < (size_t)2 * Kp + 1) ws.cnh.alloc((size_t)2 * Kp + 1);
  if (ws.row_norm2.n < n || ws.norm_src != x || ws.norm_n != n) {
    if (ws.row_norm2.n < n) ws.row_norm2.alloc(n);
    LB2_LAUNCH("tc_row_norms", row_norm_kernel, cdiv(n * 16, 256), 256, 0, x, n, d, ws.row_norm2.p);
    ws.norm_src = x;
    ws.norm_n = n;
  }
  const uint64_t res_n = resident ? n : 2 * n;  // general: the second candidate's full index in res[n ..]
  if (ws.res.n < res_n) ws.res.alloc(res_n);
  if (ws.fb_rows.n < n) ws.fb_rows.alloc(n);
  if (ws.fb_count.n < 4) ws.fb_count.alloc(4);
  float* cnh = ws.cnh.p;
  float* cn2 = ws.cnh.p + Kp;
  float* cmax2 = ws.cnh.p + 2 * (size_t)Kp;
  if (resident) {  // the same launch writes the transposed copy the exact kernels read (cT_ready below)
    const int Kp64 = (K + 63) / 64 * 64;
    if (ws.cT.n < (size_t)d * Kp64) ws.cT.alloc((size_t)d * Kp64);
    LB2_LAUNCH("tc_prep_centroids", prep_centroids_kernel, TN / 8, 256, 0, cent, K, d, bias, ws.cpad.p, cnh, cn2,
               ws.cT.p, Kp64, ws.fb_count.p);
  } else {
    LB2_LAUNCH("tc_prep_centroids", prep_centroids_general_kernel, cdiv(Kp, 8), 256, 0, cent, K, Kp, d, bias,
               ws.cpad.p, cnh, cn2, ws.fb_count.p);
  }
  LB2_LAUNCH("tc_prep_centroids", max_reduce_kernel, 1, resident ? 256 : 1024, 0, cn2, Kp, cmax2);
  int opk = resident || active ? 0 : native_opk(x16, x16_dtype, d);  // (training loops never pass native rows)
  if (opk) {
    if (ws.cpad16.n < (size_t)Kp * d) ws.cpad16.alloc((size_t)Kp * d);
    LB2_LAUNCH("tc_prep_centroids", prep16_kernel, cdiv((size_t)Kp * d, 256), 256, 0, ws.cpad.p, (size_t)Kp * d,
               opk == 2 ? 1 : 0, ws.cpad16.p, ws.fb_count.p + 3);
    uint32_t inexact = 0;
    d2h(&inexact, ws.fb_count.p + 3, 1);
    sync_stream();
    if (inexact) opk = 0;
  }
  const uint64_t tiles = (n + TM - 1) / TM;
  const unsigned grid = (unsigned)std::min<uint64_t>(tiles, (uint64_t)ctx().num_sms);
  const char* filter = resident ? "tc_filter" : opk ? "tc_filter_general16" : "tc_filter_general";
  if (opk) {
    if (ws.top1_val.n < n) ws.top1_val.alloc(n);
    const CUtensorMap map_x = make_map_2d_16(x16, opk == 2, n, d, TM);
    const CUtensorMap map_c = make_map_2d_16(ws.cpad16.p, opk == 2, Kp, d, TN);
    launch_general_dyn(opk, 0, grid, smem, map_x, map_c, n, d / (2 * KC), ntiles, cnh, ws.row_norm2.p, cmax2, ws.res.p,
                       ws.res.p + n, active, tau16_scale(d), nullptr, 0u, ws.top1_val.p, nullptr, nullptr, nullptr,
                       filter);
  } else {
    const CUtensorMap map_x = make_map_2d(x, n, d, TM);
    const CUtensorMap map_c = make_map_2d(ws.cpad.p, Kp, d, TN);
    if (resident) {
      set_smem(tc_filter_kernel, smem);
      LB2_LAUNCH(filter, tc_filter_kernel, grid, NUM_THREADS, smem, map_x, map_c, n, d / KC, stages, cnh,
                 ws.row_norm2.p, cn2, ws.res.p, active, TAU_TF32);
    } else {
      launch_general_dyn(0, 0, grid, smem, map_x, map_c, n, d / KC, ntiles, cnh, ws.row_norm2.p, cmax2, ws.res.p,
                         ws.res.p + n, active, TAU_TF32, nullptr, 0u, nullptr, nullptr, nullptr, nullptr, filter);
    }
  }
  LB2_LAUNCH("tc_rerank", rerank_kernel, cdiv(n * 16, 256), 256, 0, x, n, d, cent, bias, ws.res.p,
             (const uint32_t*)(resident ? nullptr : ws.res.p + n), dist != nullptr ? 1 : 0, part, dist, valid,
             ws.fb_rows.p, ws.fb_count.p, active, (const uint32_t*)nullptr, (const uint32_t*)nullptr, 0u,
             (const float*)nullptr, (float*)nullptr, (uint32_t*)nullptr, (uint32_t*)nullptr);
  // undecided rows: the exact kernels over the compacted row list (grids sized for the worst case; CTAs beyond the
  // device-side count exit immediately -> no host synchronisation)
  const bool refined = tc_refine_and_fallback(x, n, d, cent, K, Kp, bias, ws.cpad.p, cnh, cmax2, part, dist, valid,
                                              active, ws, /*cT_ready=*/resident, opk, x16);
  if (getenv("LB2_TC_STATS") && *getenv("LB2_TC_STATS")) {  // diagnostics: how selective was each pass?
    std::vector<uint32_t> h(n);
    uint32_t c[3];
    d2h(h.data(), ws.res.p, n);  // (the first pass's verdicts: the later passes keep their own)
    d2h(c, ws.fb_count.p, 3);
    sync_stream();
    uint64_t f[4] = {0, 0, 0, 0};
    for (uint64_t i = 0; i < n; ++i) f[h[i] >> 30]++;
    fprintf(stderr, "[lb2 %s] n=%llu K=%d d=%d: unique %.2f%%, two-candidate %.2f%%, undecided %.2f%%\n", filter,
            (unsigned long long)n, K, d, 100.0 * f[0] / n, 100.0 * f[1] / n, 100.0 * f[2] / n);
    if (refined)
      fprintf(stderr, "[lb2 %s] undecided after pass 1: %u, after the top-3 refinement: %u, full-K exact scan: %u\n",
              filter, c[0], c[1], c[2]);
  }
}

}  // namespace lb2
