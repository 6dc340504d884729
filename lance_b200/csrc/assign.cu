// assign.cu -- EXACT (reference-order f32) nearest-centroid kernels.
//
// Replaces the inner loops of
//   KMeansAlgoFloat::compute_membership_and_dist   lance-index/src/vector/kmeans.rs:317-369
//   compute_partitions_with_dists                   kmeans.rs:1275-1294
//   compute_partition (PQ code assignment)          kmeans.rs:1350-1369, pq.rs:148-178
//   l2_distance_batch / dot_distance_batch          lance-linalg/src/distance/l2.rs:194, dot.rs:164
// Four kernels, all producing bit-identical distances to the reference's 16-lane scalar loops:
//   (a) assign_tile_kernel   d % 16 == 0, d <= 256: 64 rows x 64 centroids per tile, 4x4 per thread,
//       lane-outer / chunk-inner so only two accumulators per pair are live;
//   (b) small_d_kernel       d < 16 (PQ sub-vectors, tail-only path of l2.rs:69-79), batched over
//       the M sub-spaces, optional fused residual (residual.rs:86-95), u8 codes or u32 ids out;
//   (c) generic_kernel       any d: half-warp per centroid, lane l owns lane-accumulator l;
//   (d) pq_wide_kernel       PQ sub-vectors of 16 <= ds <= 256: (a)'s tile and order plus the sequential
//       tail, with (b)'s batching over the sub-spaces, fused residual and outputs.
// pq_assign_f32 gives every PQ sub-vector width a route: (b) below 16, (d) up to 256, and wider sub-spaces
// one at a time through assign_f32_ex on a contiguous copy.
#include "assign.cuh"
#include "common.cuh"
#include "exact.cuh"
#include "tc_assign.cuh"

namespace lb2 {

// ------------------------------------------------------------------------------------------------
// transposed, padded copy of the centroids: cT[e][Kp], pad columns = NaN (never win an argmin).
// blockIdx.y selects one of a batch of such matrices (the M codebooks of a product quantizer)
// ------------------------------------------------------------------------------------------------
__global__ void transpose_pad_kernel(const float* __restrict__ c, int K, int d, int Kp,
                                     float* __restrict__ cT) {
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= d * Kp) return;
  c += (size_t)blockIdx.y * K * d;
  cT += (size_t)blockIdx.y * d * Kp;
  int e = idx / Kp, k = idx % Kp;
  cT[idx] = k < K ? c[(size_t)k * d + e] : __int_as_float(0x7fc00000);
}

// ------------------------------------------------------------------------------------------------
// (a) tile kernel
// ------------------------------------------------------------------------------------------------
// RT = rows per thread (4: 64-row tiles for bulk work; 1: 16-row tiles so that a short row list
// -- the tensor-core filter's ambiguous rows -- still spreads over all SMs)
// SPLIT (short row lists only): blockIdx.y selects ONE 64-centroid chunk, the partial (key, value, index)
// of every row goes to split_out[(list position * gridDim.y + chunk) * 3 ..] and split_merge_kernel picks
// the reference's winner -- the same work spread over gridDim.y times as many CTAs
template <int METRIC, bool WRITE_ALL, int RT, bool SPLIT = false>
__global__ void __launch_bounds__(256)
assign_tile_kernel(const float* __restrict__ x, uint64_t n, int d, const float* __restrict__ cT,
                   int K, int Kp, const float* __restrict__ bias, uint32_t* __restrict__ part,
                   float* __restrict__ dist, uint8_t* __restrict__ valid,
                   float* __restrict__ all_out, const uint8_t* __restrict__ active,
                   const uint32_t* __restrict__ row_list, const uint32_t* __restrict__ row_count,
                   uint32_t cnt_lo, uint32_t cnt_hi, float* __restrict__ split_out = nullptr) {
  if (active && !active[0]) return;
  // optional indirection: process only rows row_list[0 .. *row_count) (the tensor-core filter's
  // ambiguous rows); outputs are written at the ORIGINAL row positions.  [cnt_lo, cnt_hi) selects
  // the list lengths this instantiation serves (short lists: 16-row tiles, long lists: 64-row tiles)
  if (row_list) {
    n = *row_count;
    if (n < cnt_lo || n >= cnt_hi) return;
  }
  extern __shared__ float smem[];
  const int ld = d + 1;
  constexpr int ROWS = 16 * RT;
  float* xs = smem;              // [ROWS][d+1]
  float* cs = smem + ROWS * ld;  // [d][64]
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  // grid-stride over row tiles: bulk launches give every CTA exactly one tile; row-list launches use a
  // small persistent grid (the list length is only known on the device)
  for (uint64_t row0 = (uint64_t)blockIdx.x * ROWS; row0 < n; row0 += (uint64_t)gridDim.x * ROWS) {
  __syncthreads();  // the previous tile's readers are done with xs
  for (int idx = tid; idx < ROWS * d / 4; idx += 256) {  // float4 granules
    int r = (idx * 4) / d, e = (idx * 4) % d;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (row0 + r < n) {
      const uint64_t src = row_list ? row_list[row0 + r] : row0 + r;
      v = *reinterpret_cast<const float4*>(x + src * d + e);
    }
    float* dst = xs + r * ld + e;
    dst[0] = v.x; dst[1] = v.y; dst[2] = v.z; dst[3] = v.w;
  }
  float best_key[RT], best_val[RT];
  uint32_t best_idx[RT];
#pragma unroll
  for (int i = 0; i < RT; ++i) {
    best_key[i] = __int_as_float(0x7f800000);
    best_val[i] = __int_as_float(0x7f800000);
    best_idx[i] = 0xffffffffu;
  }
  const int nchunk = d >> 4;
  const float* xrow = xs + (ty * RT) * ld;
  const int ct_begin = SPLIT ? (int)blockIdx.y * 64 : 0, ct_end = SPLIT ? ct_begin + 64 : Kp;
  for (int ct = ct_begin; ct < ct_end; ct += 64) {
    __syncthreads();
    for (int idx = tid; idx < d * 16; idx += 256) {
      int e = idx >> 4, q = idx & 15;
      *reinterpret_cast<float4*>(cs + e * 64 + q * 4) =
          *reinterpret_cast<const float4*>(cT + (size_t)e * Kp + ct + q * 4);
    }
    __syncthreads();
    float total[RT][4];
#pragma unroll
    for (int i = 0; i < RT; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) total[i][j] = 0.0f;
    for (int l = 0; l < 16; ++l) {
      float acc[RT][4];
#pragma unroll
      for (int i = 0; i < RT; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.0f;
#pragma unroll 2
      for (int c = 0; c < nchunk; ++c) {
        const int e = c * 16 + l;
        const float4 cv = *reinterpret_cast<const float4*>(cs + e * 64 + tx * 4);
        float xv[RT];
#pragma unroll
        for (int i = 0; i < RT; ++i) xv[i] = xrow[i * ld + e];
#pragma unroll
        for (int i = 0; i < RT; ++i) {
          acc[i][0] = f_add(acc[i][0], term<METRIC>(xv[i], cv.x));
          acc[i][1] = f_add(acc[i][1], term<METRIC>(xv[i], cv.y));
          acc[i][2] = f_add(acc[i][2], term<METRIC>(xv[i], cv.z));
          acc[i][3] = f_add(acc[i][3], term<METRIC>(xv[i], cv.w));
        }
      }
#pragma unroll
      for (int i = 0; i < RT; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) total[i][j] = f_add(total[i][j], acc[i][j]);
    }
#pragma unroll
    for (int i = 0; i < RT; ++i) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const uint32_t cidx = ct + tx * 4 + j;
        const float v = finish<METRIC>(total[i][j]);
        if (WRITE_ALL) {
          const uint64_t r = row0 + ty * RT + i;
          if (r < n && cidx < (uint32_t)K) all_out[r * K + cidx] = v;
        } else {
          const float key = bias ? f_add(v, bias[cidx < (uint32_t)K ? cidx : 0]) : v;
          if (key < best_key[i]) {
            best_key[i] = key;
            best_val[i] = v;
            best_idx[i] = cidx;
          }
        }
      }
    }
  }
  if (WRITE_ALL) continue;
#pragma unroll
  for (int i = 0; i < RT; ++i) {
#pragma unroll
    for (int off = 8; off >= 1; off >>= 1) {
      float ok = __shfl_xor_sync(0xffffffffu, best_key[i], off);
      float ov = __shfl_xor_sync(0xffffffffu, best_val[i], off);
      uint32_t oi = __shfl_xor_sync(0xffffffffu, best_idx[i], off);
      if (better(ok, oi, best_key[i], best_idx[i])) {
        best_key[i] = ok; best_val[i] = ov; best_idx[i] = oi;
      }
    }
    const uint64_t rr = row0 + ty * RT + i;
    if (SPLIT) {
      if (tx == 0 && rr < n) {
        float* o = split_out + (rr * gridDim.y + blockIdx.y) * 3;
        o[0] = best_key[i];
        o[1] = best_val[i];
        o[2] = __uint_as_float(best_idx[i]);
      }
      continue;
    }
    if (tx == 0 && rr < n) {
      const uint64_t r = row_list ? row_list[rr] : rr;
      const bool ok = best_idx[i] != 0xffffffffu;
      part[r] = ok ? best_idx[i] : 0u;
      if (dist) dist[r] = ok ? best_val[i] : __int_as_float(0x7fc00000);
      if (valid) valid[r] = ok ? 1 : 0;
    }
  }
  }  // row tiles
}

// winner over the chunk partials of a SPLIT launch: strict-< on the key, lowest index on ties (chunks are
// visited in ascending centroid order, exactly like the un-split loop)
__global__ void split_merge_kernel(const float* __restrict__ split_out, int nchunks,
                                   const uint32_t* __restrict__ row_list, const uint32_t* __restrict__ row_count,
                                   uint32_t cnt_hi, uint32_t* __restrict__ part, float* __restrict__ dist,
                                   uint8_t* __restrict__ valid, const uint8_t* __restrict__ active) {
  if (active && !active[0]) return;
  const uint32_t n = *row_count;
  if (n >= cnt_hi) return;
  const uint32_t rr = blockIdx.x * blockDim.x + threadIdx.x;
  if (rr >= n) return;
  float bk = __int_as_float(0x7f800000), bv = bk;
  uint32_t bi = 0xffffffffu;
  for (int c = 0; c < nchunks; ++c) {
    const float* o = split_out + ((size_t)rr * nchunks + c) * 3;
    const uint32_t idx = __float_as_uint(o[2]);
    if (idx != 0xffffffffu && o[0] < bk) { bk = o[0]; bv = o[1]; bi = idx; }
  }
  const uint32_t r = row_list[rr];
  const bool ok = bi != 0xffffffffu;
  part[r] = ok ? bi : 0u;
  if (dist) dist[r] = ok ? bv : __int_as_float(0x7fc00000);
  if (valid) valid[r] = ok ? 1 : 0;
}

// ------------------------------------------------------------------------------------------------
// (b) small-d kernel (d < 16: only the sequential "remainder" loop of l2.rs:69-79 runs)
//   grid = (row tiles of 64, M).  x element (row, t) = x[row*ldx + m*DS + t] (- centroid[part[row]]).
// ------------------------------------------------------------------------------------------------
template <int DS, int METRIC, bool CODES>
__global__ void __launch_bounds__(256)
small_d_kernel(const float* __restrict__ x, uint64_t n, int ldx, const float* __restrict__ codebook,
               int Kc, const float* __restrict__ ivf_centroids, const uint32_t* __restrict__ part_ids,
               const uint8_t* __restrict__ row_valid, uint8_t* __restrict__ codes, int M,
               uint32_t* __restrict__ ids, float* __restrict__ dists, uint8_t* __restrict__ valid,
               const uint8_t* __restrict__ active) {
  const int m = blockIdx.y;
  if (active && !active[m]) return;
  __shared__ __align__(16) float cs[DS][64];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const uint64_t row0 = (uint64_t)blockIdx.x * 64;
  const float* cb = codebook + (size_t)m * Kc * DS;

  float xr[4][DS];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const uint64_t r = row0 + ty * 4 + i;
    if (r < n) {
      const float* src = x + r * (uint64_t)ldx + m * DS;
      if (ivf_centroids) {
        const float* c = ivf_centroids + (uint64_t)part_ids[r] * ldx + m * DS;
#pragma unroll
        for (int t = 0; t < DS; ++t) xr[i][t] = __fsub_rn(src[t], c[t]);  // residual.rs:93
      } else {
#pragma unroll
        for (int t = 0; t < DS; ++t) xr[i][t] = src[t];
      }
    } else {
#pragma unroll
      for (int t = 0; t < DS; ++t) xr[i][t] = 0.0f;
    }
  }
  float best_val[4];
  uint32_t best_idx[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    best_val[i] = __int_as_float(0x7f800000);
    best_idx[i] = 0xffffffffu;
  }
  for (int ct = 0; ct < Kc; ct += 64) {
    __syncthreads();
    for (int idx = tid; idx < 64 * DS; idx += 256) {
      int k = idx / DS, t = idx % DS;
      cs[t][k] = (ct + k < Kc) ? cb[(size_t)(ct + k) * DS + t] : __int_as_float(0x7fc00000);
    }
    __syncthreads();
    float tot[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) tot[i][j] = 0.0f;
#pragma unroll
    for (int t = 0; t < DS; ++t) {
      const float4 cv = *reinterpret_cast<const float4*>(&cs[t][tx * 4]);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        tot[i][0] = f_add(tot[i][0], term<METRIC>(xr[i][t], cv.x));
        tot[i][1] = f_add(tot[i][1], term<METRIC>(xr[i][t], cv.y));
        tot[i][2] = f_add(tot[i][2], term<METRIC>(xr[i][t], cv.z));
        tot[i][3] = f_add(tot[i][3], term<METRIC>(xr[i][t], cv.w));
      }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float v = finish<METRIC>(f_add(tot[i][j], 0.0f));
        const uint32_t cidx = ct + tx * 4 + j;
        if (v < best_val[i]) {
          best_val[i] = v;
          best_idx[i] = cidx;
        }
      }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
#pragma unroll
    for (int off = 8; off >= 1; off >>= 1) {
      float ov = __shfl_xor_sync(0xffffffffu, best_val[i], off);
      uint32_t oi = __shfl_xor_sync(0xffffffffu, best_idx[i], off);
      if (better(ov, oi, best_val[i], best_idx[i])) {
        best_val[i] = ov; best_idx[i] = oi;
      }
    }
    const uint64_t r = row0 + ty * 4 + i;
    if (tx == 0 && r < n) {
      const bool ok = best_idx[i] != 0xffffffffu;
      if (CODES) {
        // pq.rs:165 `unwrap_or(0)`; rows KeepFinite would drop get all-zero codes
        const bool rv = row_valid ? row_valid[r] != 0 : true;
        codes[r * (uint64_t)M + m] = (ok && rv) ? (uint8_t)best_idx[i] : (uint8_t)0;
      } else {
        ids[(uint64_t)m * n + r] = ok ? best_idx[i] : 0u;
        if (dists) dists[(uint64_t)m * n + r] = ok ? best_val[i] : __int_as_float(0x7fc00000);
        if (valid) valid[(uint64_t)m * n + r] = ok ? 1 : 0;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// (c) generic kernel: 8 rows per CTA in smem, 16 half-warps stride over the centroids, lane l of a
// half-warp owns lane-accumulator l (elements 16c+l) -> coalesced 64-byte centroid reads.
// ------------------------------------------------------------------------------------------------
// SPLIT (short row lists only): blockIdx.y selects one range of kchunk centroids, the partial (key, value,
// index) of every row goes to split_out and split_merge_kernel picks the winner -- a few hundred rows against
// thousands of wide centroids are latency bound otherwise (one CTA walks the whole centroid matrix)
template <int METRIC, bool WRITE_ALL, int R, bool SPLIT = false>
__global__ void __launch_bounds__(256)
generic_kernel(const float* __restrict__ x, uint64_t n, int d, const float* __restrict__ cent, int K,
               const float* __restrict__ bias, uint32_t* __restrict__ part, float* __restrict__ dist,
               uint8_t* __restrict__ valid, float* __restrict__ all_out,
               const uint8_t* __restrict__ active, const uint32_t* __restrict__ row_list,
               const uint32_t* __restrict__ row_count, uint32_t cnt_lo = 0, uint32_t cnt_hi = 0xffffffffu,
               int kchunk = 0, float* __restrict__ split_out = nullptr) {
  if (active && !active[0]) return;
  if (row_list) {  // same indirection as the tile kernel
    n = *row_count;
    if (n < cnt_lo || n >= cnt_hi) return;
  }
  extern __shared__ float smem[];
  float* xs = smem;  // [R][d]
  __shared__ float red_key[16][R];
  __shared__ float red_val[16][R];
  __shared__ uint32_t red_idx[16][R];
  const int tid = threadIdx.x, hw = tid >> 4, l = tid & 15;
  for (uint64_t row0 = (uint64_t)blockIdx.x * R; row0 < n; row0 += (uint64_t)gridDim.x * R) {  // see tile kernel
  __syncthreads();
  for (int idx = tid; idx < R * d; idx += 256) {
    int r = idx / d, e = idx % d;
    const uint64_t src = row0 + r < n ? (row_list ? (uint64_t)row_list[row0 + r] : row0 + r) : 0;
    xs[idx] = (row0 + r < n) ? x[src * d + e] : 0.0f;
  }
  __syncthreads();
  const int n16 = d & ~15;
  float bkey = __int_as_float(0x7f800000), bval = __int_as_float(0x7f800000);
  uint32_t bidx = 0xffffffffu;  // lane l tracks row (l & (R - 1)); R is 8 or 16
  const unsigned hmask = 0xffffu << (16 * ((tid >> 4) & 1));
  const int k_begin = SPLIT ? (int)blockIdx.y * kchunk : 0, k_end = SPLIT ? min(K, k_begin + kchunk) : K;
  for (int c = k_begin + hw; c < k_end; c += 16) {
    const float* cp = cent + (size_t)c * d;
    float acc[R];
#pragma unroll
    for (int r = 0; r < R; ++r) acc[r] = 0.0f;
    for (int e = l; e < n16; e += 16) {
      const float cv = cp[e];
#pragma unroll
      for (int r = 0; r < R; ++r) acc[r] = f_add(acc[r], term<METRIC>(xs[r * d + e], cv));
    }
    float mine = 0.0f;
#pragma unroll
    for (int r = 0; r < R; ++r) {
      float s = 0.0f;  // sequential tail (l2.rs:69-79), every lane computes it redundantly
      for (int e = n16; e < d; ++e) s = f_add(s, term<METRIC>(xs[r * d + e], cp[e]));
      float t = 0.0f;
#pragma unroll
      for (int q = 0; q < 16; ++q)
        t = f_add(t, __shfl_sync(hmask, acc[r], q, 16));
      const float v = finish<METRIC>(f_add(s, t));
      if (WRITE_ALL) {
        if (l == r && row0 + r < n) all_out[(row0 + r) * K + c] = v;
      } else if ((l & (R - 1)) == r) {
        mine = v;
      }
    }
    if (!WRITE_ALL) {
      const float key = bias ? f_add(mine, bias[c]) : mine;
      if (key < bkey) { bkey = key; bval = mine; bidx = c; }
    }
  }
  if (WRITE_ALL) continue;
  if (l < R) { red_key[hw][l] = bkey; red_val[hw][l] = bval; red_idx[hw][l] = bidx; }
  __syncthreads();
  if (tid < R) {
    float k0 = red_key[0][tid], v0 = red_val[0][tid];
    uint32_t i0 = red_idx[0][tid];
    for (int h = 1; h < 16; ++h)
      if (better(red_key[h][tid], red_idx[h][tid], k0, i0)) {
        k0 = red_key[h][tid]; v0 = red_val[h][tid]; i0 = red_idx[h][tid];
      }
    uint64_t r = row0 + tid;
    if (SPLIT) {
      if (r < n) {
        float* o = split_out + (r * gridDim.y + blockIdx.y) * 3;
        o[0] = k0;
        o[1] = v0;
        o[2] = __uint_as_float(i0);
      }
    } else if (r < n) {
      if (row_list) r = row_list[r];
      const bool ok = i0 != 0xffffffffu;
      part[r] = ok ? i0 : 0u;
      if (dist) dist[r] = ok ? v0 : __int_as_float(0x7fc00000);
      if (valid) valid[r] = ok ? 1 : 0;
    }
  }
  }  // row groups
}

// ------------------------------------------------------------------------------------------------
// (d) wide PQ kernel (16 <= ds <= 256: the reference's full order, l2.rs:57-91 / dot.rs:30-58, restated in
//   dist_exact_thread): per (row, codeword) pair the 16 lane sums in chunk order, added in lane order (t), the
//   tail ds & ~15 .. ds-1 summed left to right (s), then s + t.
//   grid = (row tiles of 64, M), 4 rows x 4 codewords per thread as in (a): lane-outer / chunk-inner, so only the
//   lane and total accumulators are live, then the tail.  The tile's rows (residuals when ivf_centroids is given)
//   and 64-codeword tiles of cbT ([M][ds][Kp], NaN pad columns, transpose_pad_kernel) are staged in shared memory.
//   Outputs, tie rule and row_valid as in (b).
// ------------------------------------------------------------------------------------------------
template <int METRIC, bool CODES>
__global__ void __launch_bounds__(256)
pq_wide_kernel(const float* __restrict__ x, uint64_t n, int ldx, int ds, const float* __restrict__ cbT, int Kp,
               const float* __restrict__ ivf_centroids, const uint32_t* __restrict__ part_ids,
               const uint8_t* __restrict__ row_valid, uint8_t* __restrict__ codes, int M,
               uint32_t* __restrict__ ids, float* __restrict__ dists, uint8_t* __restrict__ valid,
               const uint8_t* __restrict__ active) {
  const int m = blockIdx.y;
  if (active && !active[m]) return;
  extern __shared__ float smem[];
  const int ld = ds + 1;
  float* xs = smem;            // [64][ds+1]
  float* cs = smem + 64 * ld;  // [ds][64] (64 * ld floats: 16-byte aligned)
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const uint64_t row0 = (uint64_t)blockIdx.x * 64;
  // scalar loads: neither the row stride nor m * ds need be a multiple of 4
  for (int idx = tid; idx < 64 * ds; idx += 256) {
    const int r = idx / ds, t = idx - r * ds;
    float v = 0.0f;
    if (row0 + r < n) {
      v = x[(row0 + r) * (uint64_t)ldx + (uint64_t)m * ds + t];
      if (ivf_centroids)  // residual.rs:93
        v = __fsub_rn(v, ivf_centroids[(uint64_t)part_ids[row0 + r] * ldx + (uint64_t)m * ds + t]);
    }
    xs[r * ld + t] = v;
  }
  const float* cb = cbT + (size_t)m * ds * Kp;
  const float* xrow = xs + (ty * 4) * ld;
  const int nchunk = ds >> 4, n16 = ds & ~15;
  float best_val[4];
  uint32_t best_idx[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    best_val[i] = __int_as_float(0x7f800000);
    best_idx[i] = 0xffffffffu;
  }
  for (int ct = 0; ct < Kp; ct += 64) {
    __syncthreads();
    for (int idx = tid; idx < ds * 16; idx += 256) {
      const int e = idx >> 4, q = idx & 15;
      *reinterpret_cast<float4*>(cs + e * 64 + q * 4) =
          *reinterpret_cast<const float4*>(cb + (size_t)e * Kp + ct + q * 4);
    }
    __syncthreads();
    float total[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) total[i][j] = 0.0f;
    for (int l = 0; l < 16; ++l) {
      float acc[4][4];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.0f;
#pragma unroll 2
      for (int c = 0; c < nchunk; ++c) {
        const int e = c * 16 + l;
        const float4 cv = *reinterpret_cast<const float4*>(cs + e * 64 + tx * 4);
        float xv[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) xv[i] = xrow[i * ld + e];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          acc[i][0] = f_add(acc[i][0], term<METRIC>(xv[i], cv.x));
          acc[i][1] = f_add(acc[i][1], term<METRIC>(xv[i], cv.y));
          acc[i][2] = f_add(acc[i][2], term<METRIC>(xv[i], cv.z));
          acc[i][3] = f_add(acc[i][3], term<METRIC>(xv[i], cv.w));
        }
      }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) total[i][j] = f_add(total[i][j], acc[i][j]);
    }
    float s[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) s[i][j] = 0.0f;
    for (int e = n16; e < ds; ++e) {
      const float4 cv = *reinterpret_cast<const float4*>(cs + e * 64 + tx * 4);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float xv = xrow[i * ld + e];
        s[i][0] = f_add(s[i][0], term<METRIC>(xv, cv.x));
        s[i][1] = f_add(s[i][1], term<METRIC>(xv, cv.y));
        s[i][2] = f_add(s[i][2], term<METRIC>(xv, cv.z));
        s[i][3] = f_add(s[i][3], term<METRIC>(xv, cv.w));
      }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float v = finish<METRIC>(f_add(s[i][j], total[i][j]));
        const uint32_t cidx = ct + tx * 4 + j;
        if (v < best_val[i]) {  // ascending codewords, strict <: the first minimum; NaN never wins
          best_val[i] = v;
          best_idx[i] = cidx;
        }
      }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
#pragma unroll
    for (int off = 8; off >= 1; off >>= 1) {
      float ov = __shfl_xor_sync(0xffffffffu, best_val[i], off);
      uint32_t oi = __shfl_xor_sync(0xffffffffu, best_idx[i], off);
      if (better(ov, oi, best_val[i], best_idx[i])) {
        best_val[i] = ov; best_idx[i] = oi;
      }
    }
    const uint64_t r = row0 + ty * 4 + i;
    if (tx == 0 && r < n) {
      const bool ok = best_idx[i] != 0xffffffffu;
      if (CODES) {
        const bool rv = row_valid ? row_valid[r] != 0 : true;
        codes[r * (uint64_t)M + m] = (ok && rv) ? (uint8_t)best_idx[i] : (uint8_t)0;
      } else {
        ids[(uint64_t)m * n + r] = ok ? best_idx[i] : 0u;
        if (dists) dists[(uint64_t)m * n + r] = ok ? best_val[i] : __int_as_float(0x7fc00000);
        if (valid) valid[(uint64_t)m * n + r] = ok ? 1 : 0;
      }
    }
  }
}

// sub-space m of rows [0, n) as contiguous [n][ds] rows (residuals when cent is given): the route for
// sub-vectors wider than pq_wide_kernel's tile hands them to assign_f32_ex one sub-space at a time
__global__ void pq_subspace_copy_kernel(const float* __restrict__ x, uint64_t n, int ldx, int ds, int m,
                                        const float* __restrict__ cent, const uint32_t* __restrict__ part,
                                        float* __restrict__ out) {
  const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n * ds) return;
  const uint64_t r = g / ds;
  const uint64_t col = (uint64_t)m * ds + g % ds;
  const float v = x[r * ldx + col];
  out[g] = cent ? __fsub_rn(v, cent[(uint64_t)part[r] * ldx + col]) : v;  // residual.rs:93
}

// sub-space m's codes from an assignment: pq.rs:165 `unwrap_or(0)`, zero for rows row_valid drops
__global__ void pq_subspace_codes_kernel(const uint32_t* __restrict__ ids, const uint8_t* __restrict__ ok,
                                         const uint8_t* __restrict__ row_valid, uint64_t n, int M, int m,
                                         uint8_t* __restrict__ codes) {
  const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const bool rv = row_valid ? row_valid[r] != 0 : true;
  codes[r * M + m] = (ok[r] && rv) ? (uint8_t)ids[r] : (uint8_t)0;
}

// ------------------------------------------------------------------------------------------------
// host dispatch
// ------------------------------------------------------------------------------------------------
template <int METRIC, bool WRITE_ALL>
static void assign_dispatch(const float* x, uint64_t n, int d, const float* cent, int K,
                            const float* bias, uint32_t* part, float* dist,
                            uint8_t* valid, float* all_out, const uint8_t* active, TcWorkspace& ws) {
  if (n == 0) return;
  // the tile kernel reads rows as float4: a row base that is not 16-byte aligned (a view into a caller's buffer)
  // takes the scalar-load generic kernel, which returns the same bits
  if (d % 16 == 0 && d <= 256 && (reinterpret_cast<uintptr_t>(x) & 15) == 0) {
    const int Kp = (K + 63) / 64 * 64;
    DevBuf<float>& cT = ws.cT;  // no allocation per call inside a training loop / CUDA graph
    if (cT.n < (size_t)d * Kp) cT.alloc((size_t)d * Kp);
    LB2_LAUNCH("transpose_centroids", transpose_pad_kernel, cdiv((uint64_t)d * Kp, 256), 256, 0,
               cent, K, d, Kp, cT.get());
    const size_t smem = sizeof(float) * (64 * (d + 1) + (size_t)d * 64);
    const unsigned grid = cdiv(n, 64);
    set_smem(assign_tile_kernel<METRIC, WRITE_ALL, 4>, smem);
    LB2_LAUNCH("assign_exact", (assign_tile_kernel<METRIC, WRITE_ALL, 4>), grid, 256, smem, x, n, d,
               cT.get(), K, Kp, bias, part, dist, valid, all_out, active, nullptr, nullptr, 0u, 0xffffffffu);
    return;
  }
  // 16 rows per CTA halve the centroid re-reads from L2; wide vectors fall back to 8 rows
  const bool r16 = sizeof(float) * 16 * (size_t)d <= 96 * 1024;
  const size_t smem = sizeof(float) * (r16 ? 16 : 8) * (size_t)d;
  const unsigned grid = cdiv(n, r16 ? 16 : 8);
#define LB2_GENERIC(RR)                                                                                \
  do {                                                                                                 \
    if (smem_with_static(generic_kernel<METRIC, WRITE_ALL, RR>, smem) > ctx().smem_optin)              \
      fail(LB2_UNSUPPORTED, "dimension %d too large for the exact kernel", d);                         \
    set_smem(generic_kernel<METRIC, WRITE_ALL, RR>, smem);                                             \
    LB2_LAUNCH("assign_exact_generic", (generic_kernel<METRIC, WRITE_ALL, RR>), grid, 256, smem, x, n, \
               d, cent, K, bias, part, dist, valid, all_out, active, nullptr, nullptr);                \
  } while (0)
  if (r16) LB2_GENERIC(16); else LB2_GENERIC(8);
#undef LB2_GENERIC
}

// exact tile kernel over a device-side row list (count read on the device: no host sync)
void assign_rows_f32(const float* x, uint64_t n_max, int d, const float* cent, int K, int metric,
                     const float* bias, const uint32_t* row_list, const uint32_t* row_count,
                     uint32_t* part, float* dist, uint8_t* valid, const uint8_t* active,
                     TcWorkspace& ws, bool cT_ready) {
  if (metric != METRIC_L2) fail(LB2_UNSUPPORTED, "assign_rows_f32: metric not supported");
  if (!(d % 16 == 0 && d <= 256)) {
    // 8 rows per CTA: the list is short, more CTAs beat fewer centroid re-reads (measured)
    const size_t gsmem = sizeof(float) * 8 * (size_t)d;
    if (smem_with_static(generic_kernel<METRIC_L2, false, 8>, gsmem) > ctx().smem_optin)
      fail(LB2_UNSUPPORTED, "dimension %d too large for the exact kernel", d);
    // very short lists against many centroids: one CTA per (8 rows, range of centroids) + a merge
    const int gchunks = (int)std::min<uint64_t>(64, (uint64_t)K / 128);
    const uint32_t gtiny = gchunks > 1 ? (uint32_t)std::min<uint64_t>(4096, n_max + 1) : 0u;
    if (gtiny) {
      const int kchunk = ((K + gchunks - 1) / gchunks + 15) / 16 * 16;
      const int nch = (K + kchunk - 1) / kchunk;
      if (ws.split_scratch.n < (size_t)gtiny * nch * 3) ws.split_scratch.alloc((size_t)gtiny * nch * 3);
      set_smem((generic_kernel<METRIC_L2, false, 8, true>), gsmem);
      LB2_LAUNCH("assign_exact_fallback", (generic_kernel<METRIC_L2, false, 8, true>),
                 dim3((unsigned)cdiv(gtiny, 8), (unsigned)nch), 256, gsmem, x, n_max, d, cent, K, bias, part, dist,
                 valid, nullptr, active, row_list, row_count, 0u, gtiny, kchunk, ws.split_scratch.p);
      LB2_LAUNCH("assign_exact_fallback", split_merge_kernel, cdiv(gtiny, 256), 256, 0, ws.split_scratch.p, nch, row_list,
                 row_count, gtiny, part, dist, valid, active);
    }
    set_smem(generic_kernel<METRIC_L2, false, 8>, gsmem);
    LB2_LAUNCH("assign_exact_fallback", (generic_kernel<METRIC_L2, false, 8>),
               (unsigned)std::min<uint64_t>(cdiv(n_max, 8), 8 * (uint64_t)ctx().num_sms), 256, gsmem, x,
               n_max, d, cent, K, bias, part, dist, valid, nullptr, active, row_list, row_count, gtiny,
               0xffffffffu);
    return;
  }
  const int Kp = (K + 63) / 64 * 64;
  DevBuf<float>& cT = ws.cT;
  if (cT.n < (size_t)d * Kp) cT.alloc((size_t)d * Kp);
  if (!cT_ready)
    LB2_LAUNCH("transpose_centroids", transpose_pad_kernel, cdiv((uint64_t)d * Kp, 256), 256, 0, cent,
               K, d, Kp, cT.get());
  // The list length lives on the device, so every regime is launched and the ones whose range does not
  // hold the count exit at once:
  //   very short lists (< 2048 rows): 16-row tiles x one CTA per 64-centroid chunk + a merge (latency);
  //   short lists: 16-row tiles so that the work still spreads over all SMs;
  //   long lists (only worth a launch when the centroid matrix is large, K > 256): 64-row tiles.
  const int nchunks = Kp / 64;
  const uint32_t tiny = (nchunks > 1 && nchunks <= 64) ? (uint32_t)std::min<uint64_t>(2048, n_max + 1) : 0u;
  const uint32_t split = K > 256 ? 64u * 2u * (uint32_t)ctx().num_sms : 0xffffffffu;
  const size_t smem = sizeof(float) * (16 * (d + 1) + (size_t)d * 64);
  if (tiny) {
    if (ws.split_scratch.n < (size_t)tiny * nchunks * 3) ws.split_scratch.alloc((size_t)tiny * nchunks * 3);
    set_smem(assign_tile_kernel<METRIC_L2, false, 1, true>, smem);
    LB2_LAUNCH("assign_exact_fallback", (assign_tile_kernel<METRIC_L2, false, 1, true>),
               dim3((unsigned)cdiv(tiny, 16), (unsigned)nchunks), 256, smem, x, n_max, d, cT.get(), K, Kp, bias,
               part, dist, valid, nullptr, active, row_list, row_count, 0u, tiny, ws.split_scratch.p);
    LB2_LAUNCH("assign_exact_fallback", split_merge_kernel, cdiv(tiny, 256), 256, 0, ws.split_scratch.p, nchunks,
               row_list, row_count, tiny, part, dist, valid, active);
  }
  set_smem(assign_tile_kernel<METRIC_L2, false, 1>, smem);
  LB2_LAUNCH("assign_exact_fallback", (assign_tile_kernel<METRIC_L2, false, 1>),
             (unsigned)std::min<uint64_t>(cdiv(std::min<uint64_t>(n_max, split), 16), 4 * (uint64_t)ctx().num_sms), 256,
             smem, x, n_max, d, cT.get(), K, Kp, bias,
             part, dist, valid, nullptr, active, row_list, row_count, tiny, split);
  if (n_max >= split) {
    const size_t smem4 = sizeof(float) * (64 * (d + 1) + (size_t)d * 64);
    set_smem(assign_tile_kernel<METRIC_L2, false, 4>, smem4);
    LB2_LAUNCH("assign_exact_fallback", (assign_tile_kernel<METRIC_L2, false, 4>),
               (unsigned)std::min<uint64_t>(cdiv(n_max, 64), 2 * (uint64_t)ctx().num_sms), 256, smem4,
               x, n_max, d, cT.get(), K, Kp, bias, part, dist, valid, nullptr, active, row_list,
               row_count, split, 0xffffffffu);
  }
}

void assign_f32_ex(const float* x, uint64_t n, int d, const float* cent, int K, int metric,
                   const float* bias, uint32_t* part, float* dist, uint8_t* valid,
                   const uint8_t* active, TcWorkspace& ws, const void* x16, int x16_dtype) {
  if (n >= 256 && tc_assign_supported(n, d, K, metric, x)) {
    // tensor-core filter + exact re-rank: bit-identical outputs, ~10x less FP32 work
    // large inputs in chunks of <= 2^20 rows (<= 4 GB of vectors): bounds the per-call scratch (row norms,
    // verdicts, the 3x-wide refinement rows) without changing any output
    const uint64_t chunk = std::max<uint64_t>(1ull << 16, std::min<uint64_t>(1ull << 20, (1ull << 30) / (uint64_t)d));
    if (n <= chunk + chunk / 2) {
      tc_assign_f32(x, n, d, cent, K, bias, part, dist, valid, active, ws, x16, x16_dtype);
      return;
    }
    for (uint64_t r0 = 0; r0 < n; r0 += chunk) {
      const uint64_t rows = std::min(chunk, n - r0);
      tc_assign_f32(x + r0 * d, rows, d, cent, K, bias, part + r0, dist ? dist + r0 : nullptr,
                    valid ? valid + r0 : nullptr, active, ws,
                    x16 ? static_cast<const uint16_t*>(x16) + r0 * d : nullptr, x16_dtype);
    }
    return;
  }
  if (metric == METRIC_DOT)
    assign_dispatch<METRIC_DOT, false>(x, n, d, cent, K, bias, part, dist, valid, nullptr, active, ws);
  else
    assign_dispatch<METRIC_L2, false>(x, n, d, cent, K, bias, part, dist, valid, nullptr, active, ws);
}
void assign_f32(const float* x, uint64_t n, int d, const float* cent, int K, int metric,
                const float* bias, uint32_t* part, float* dist, uint8_t* valid, const void* x16, int x16_dtype) {
  TcWorkspace ws;
  assign_f32_ex(x, n, d, cent, K, metric, bias, part, dist, valid, nullptr, ws, x16, x16_dtype);
}
void centroid_distances(const float* x, uint64_t n, int d, const float* cent, int K, int metric, float* out) {
  TcWorkspace ws;
  if (metric == METRIC_DOT)
    assign_dispatch<METRIC_DOT, true>(x, n, d, cent, K, nullptr, nullptr, nullptr, nullptr, out, nullptr, ws);
  else
    assign_dispatch<METRIC_L2, true>(x, n, d, cent, K, nullptr, nullptr, nullptr, nullptr, out, nullptr, ws);
}

template <int DS, int METRIC>
static void small_d_launch(const float* x, uint64_t n, int ldx, int M, const float* codebook, int Kc,
                           const float* ivf_centroids, const uint32_t* part_ids,
                           const uint8_t* row_valid, uint8_t* codes, uint32_t* ids, float* dists,
                           uint8_t* valid, const uint8_t* active) {
  dim3 grid(cdiv(n, 64), M);
  if (codes)
    LB2_LAUNCH("pq_assign_exact", (small_d_kernel<DS, METRIC, true>), grid, 256, 0, x, n, ldx,
               codebook, Kc, ivf_centroids, part_ids, row_valid, codes, M, ids, dists, valid, active);
  else
    LB2_LAUNCH("pq_assign_exact", (small_d_kernel<DS, METRIC, false>), grid, 256, 0, x, n, ldx,
               codebook, Kc, ivf_centroids, part_ids, row_valid, codes, M, ids, dists, valid, active);
}

template <int METRIC>
static void pq_wide_launch(const float* x, uint64_t n, int ldx, int M, int ds, const float* codebook, int Kc,
                           const float* ivf_centroids, const uint32_t* part_ids, const uint8_t* row_valid,
                           uint8_t* codes, uint32_t* ids, float* dists, uint8_t* valid, const uint8_t* active,
                           PqAssignWorkspace& ws) {
  const int Kp = (Kc + 63) / 64 * 64;
  if (ws.cbT.n < (size_t)M * ds * Kp) ws.cbT.alloc((size_t)M * ds * Kp);
  LB2_LAUNCH("pq_codebook_transpose", transpose_pad_kernel, dim3(cdiv((uint64_t)ds * Kp, 256), M), 256, 0, codebook,
             Kc, ds, Kp, ws.cbT.p);
  const size_t smem = sizeof(float) * (64 * (size_t)(ds + 1) + (size_t)ds * 64);
  const dim3 grid(cdiv(n, 64), M);
#define LB2_WIDE(CODESV)                                                                                    \
  do {                                                                                                      \
    set_smem(pq_wide_kernel<METRIC, CODESV>, smem);                                                         \
    LB2_LAUNCH("pq_assign_wide", (pq_wide_kernel<METRIC, CODESV>), grid, 256, smem, x, n, ldx, ds, ws.cbT.p, \
               Kp, ivf_centroids, part_ids, row_valid, codes, M, ids, dists, valid, active);               \
  } while (0)
  if (codes) LB2_WIDE(true); else LB2_WIDE(false);
#undef LB2_WIDE
}

// sub-vectors wider than the wide kernel's tile: each sub-space's rows as a contiguous matrix through the exact IVF
// assignment (tensor-core filter + exact re-rank where it applies), which computes the same reference-order
// distances, keeps the same first minimum and marks a row without a finite winner with valid = 0
static void pq_assign_by_subspace(const float* x, uint64_t n, int ldx, int M, int ds, const float* codebook, int Kc,
                                  int metric, const float* ivf_centroids, const uint32_t* part_ids,
                                  const uint8_t* row_valid, uint8_t* codes, uint32_t* ids, float* dists,
                                  uint8_t* valid, const uint8_t* active, PqAssignWorkspace& ws) {
  const uint64_t chunk = std::min<uint64_t>(n, std::max<uint64_t>(1ull << 16, (1ull << 28) / (uint64_t)ds));  // <= 1 GB
  if (ws.sub.n < chunk * ds) ws.sub.alloc(chunk * ds);
  if (codes && ws.ids.n < chunk) {
    ws.ids.alloc(chunk);
    ws.ok.alloc(chunk);
  }
  for (uint64_t r0 = 0; r0 < n; r0 += chunk) {
    const uint64_t rows = std::min(chunk, n - r0);
    for (int m = 0; m < M; ++m) {
      LB2_LAUNCH("pq_subspace_copy", pq_subspace_copy_kernel, cdiv(rows * ds, 256), 256, 0, x + r0 * ldx, rows, ldx,
                 ds, m, ivf_centroids, part_ids ? part_ids + r0 : nullptr, ws.sub.p);
      ws.tc.norm_src = nullptr;  // the buffer holds another sub-space now: its cached row norms are stale
      const float* cb = codebook + (size_t)m * Kc * ds;
      if (codes) {
        assign_f32_ex(ws.sub.p, rows, ds, cb, Kc, metric, nullptr, ws.ids.p, nullptr, ws.ok.p, nullptr, ws.tc);
        LB2_LAUNCH("pq_subspace_codes", pq_subspace_codes_kernel, cdiv(rows, 256), 256, 0, ws.ids.p, ws.ok.p,
                   row_valid ? row_valid + r0 : nullptr, rows, M, m, codes + r0 * M);
      } else {
        const uint64_t o = (uint64_t)m * n + r0;
        assign_f32_ex(ws.sub.p, rows, ds, cb, Kc, metric, nullptr, ids + o, dists ? dists + o : nullptr,
                      valid ? valid + o : nullptr, active ? active + m : nullptr, ws.tc);
      }
    }
  }
}

void pq_assign_f32(const float* x, uint64_t n, int ldx, int M, int ds, const float* codebook, int Kc, int metric,
                   const float* ivf_centroids, const uint32_t* part_ids, const uint8_t* row_valid, uint8_t* codes,
                   uint32_t* ids, float* dists, uint8_t* valid, const uint8_t* active, PqAssignWorkspace* ws) {
  if (n == 0) return;
  if (ds >= 16) {
    PqAssignWorkspace local;  // stream-ordered frees: nothing to wait for on return
    PqAssignWorkspace& w = ws ? *ws : local;
    if (ds > PQ_WIDE_MAX_DS)
      pq_assign_by_subspace(x, n, ldx, M, ds, codebook, Kc, metric, ivf_centroids, part_ids, row_valid, codes, ids,
                            dists, valid, active, w);
    else if (metric == METRIC_DOT)
      pq_wide_launch<METRIC_DOT>(x, n, ldx, M, ds, codebook, Kc, ivf_centroids, part_ids, row_valid, codes, ids,
                                 dists, valid, active, w);
    else
      pq_wide_launch<METRIC_L2>(x, n, ldx, M, ds, codebook, Kc, ivf_centroids, part_ids, row_valid, codes, ids,
                                dists, valid, active, w);
    return;
  }
#define LB2_SD(DSV)                                                                              \
  case DSV:                                                                                      \
    if (metric == METRIC_DOT)                                                                    \
      small_d_launch<DSV, METRIC_DOT>(x, n, ldx, M, codebook, Kc, ivf_centroids, part_ids,       \
                                      row_valid, codes, ids, dists, valid, active);              \
    else                                                                                         \
      small_d_launch<DSV, METRIC_L2>(x, n, ldx, M, codebook, Kc, ivf_centroids, part_ids,        \
                                     row_valid, codes, ids, dists, valid, active);               \
    break;
  switch (ds) {
    LB2_SD(1) LB2_SD(2) LB2_SD(3) LB2_SD(4) LB2_SD(5) LB2_SD(6) LB2_SD(7) LB2_SD(8)
    LB2_SD(9) LB2_SD(10) LB2_SD(11) LB2_SD(12) LB2_SD(13) LB2_SD(14) LB2_SD(15)
    default:
      fail(LB2_INVALID_ARG, "PQ sub-vector width %d", ds);
  }
#undef LB2_SD
}

}  // namespace lb2
