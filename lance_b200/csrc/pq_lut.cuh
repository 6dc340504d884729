// pq_lut.cuh -- the PQ lookup table of a query and the row sums over it: the one definition that the IVF_PQ scan
// (pq_scan.cu) and the IVF_HNSW_PQ graph build and search (hnsw.cu) share, so that both kinds score a row from the
// same table bits.
//
// Replaces  build_distance_table_l2/_dot       lance-index/src/vector/pq/distance.rs:24-92
//           compute_pq_distance (8-bit sum)     pq/distance.rs:109-144
//           PQDistCalculator::distance          pq/storage.rs:891-919
#pragma once
#include "common.cuh"
#include "exact.cuh"

namespace lb2 {

// LUT[m][c] = dist(q_m, cb[m][c])  (pq/distance.rs:38-56).  For the common sub-vector widths the
// codeword is fetched with 128-bit loads and the reference-order sum is fully unrolled.
template <int METRIC, int DS>
__device__ __forceinline__ float lut_entry_fixed(const float* __restrict__ qm, const float* __restrict__ cw) {
  float qv[DS], cv[DS];
#pragma unroll
  for (int t = 0; t < DS; t += 4) {
    const float4 a = *reinterpret_cast<const float4*>(qm + t);
    const float4 b = __ldg(reinterpret_cast<const float4*>(cw + t));
    qv[t] = a.x; qv[t + 1] = a.y; qv[t + 2] = a.z; qv[t + 3] = a.w;
    cv[t] = b.x; cv[t + 1] = b.y; cv[t + 2] = b.z; cv[t + 3] = b.w;
  }
  if (DS < 16) {  // tail-only path (l2.rs:69-79): plain left-to-right sum
    float s = 0.0f;
#pragma unroll
    for (int t = 0; t < DS; ++t) s = f_add(s, term<METRIC>(qv[t], cv[t]));
    return finish<METRIC>(f_add(s, 0.0f));
  } else {        // DS == 16: one chunk of 16 lanes, summed lane 0..15
    float t0 = 0.0f;
#pragma unroll
    for (int t = 0; t < 16; ++t) t0 = f_add(t0, f_add(0.0f, term<METRIC>(qv[t], cv[t])));
    return finish<METRIC>(f_add(0.0f, t0));
  }
}

// the 8-bit table [M][256] of the query qr (16-byte aligned), threads tid = 0 .. NT - 1 of the caller
template <int METRIC, int NT = 256>
__device__ __forceinline__ void build_lut_smem(float* lut, const float* qr, const float* __restrict__ codebook,
                                               int M, int ds, int tid) {
  if (ds == 8) {
    for (int idx = tid; idx < M * 256; idx += NT)
      lut[idx] = lut_entry_fixed<METRIC, 8>(qr + (idx >> 8) * 8, codebook + (size_t)idx * 8);
  } else if (ds == 4) {
    for (int idx = tid; idx < M * 256; idx += NT)
      lut[idx] = lut_entry_fixed<METRIC, 4>(qr + (idx >> 8) * 4, codebook + (size_t)idx * 4);
  } else if (ds == 16) {
    for (int idx = tid; idx < M * 256; idx += NT)
      lut[idx] = lut_entry_fixed<METRIC, 16>(qr + (idx >> 8) * 16, codebook + (size_t)idx * 16);
  } else {
    for (int idx = tid; idx < M * 256; idx += NT)
      lut[idx] = dist_exact_thread<METRIC>(qr + (idx >> 8) * ds, codebook + (size_t)idx * ds, ds);
  }
}

// the table [M][2^NBITS] of the query qr: 8-bit as build_lut_smem, 4-bit one exact entry per thread and step
template <int METRIC, int NBITS, int NT = 256>
__device__ __forceinline__ void build_lut(float* lut, const float* qr, const float* __restrict__ codebook, int M,
                                          int ds, int tid) {
  if (NBITS == 8) {
    build_lut_smem<METRIC, NT>(lut, qr, codebook, M, ds, tid);
  } else {
    for (int idx = tid; idx < M * 16; idx += NT)
      lut[idx] = dist_exact_thread<METRIC>(qr + (idx / 16) * ds, codebook + (size_t)idx * ds, ds);
  }
}

// one row's 8-bit ADC distance: the reference's m-ascending f32 sum of LUT[m][code[m]] (pq/distance.rs:109-144)
__device__ __forceinline__ float pq8_row_distance(const float* lut, const uint8_t* __restrict__ rp, int M) {
  float dist = 0.0f;
  if ((M & 15) == 0) {
    const uint4* rp4 = reinterpret_cast<const uint4*>(rp);
    for (int c16 = 0; c16 < M / 16; ++c16) {
      const uint4 v = __ldg(rp4 + c16);
      const uint32_t w[4] = {v.x, v.y, v.z, v.w};
      const float* l0 = lut + c16 * 16 * 256;
#pragma unroll
      for (int aa = 0; aa < 4; ++aa)
#pragma unroll
        for (int bb = 0; bb < 4; ++bb)
          dist = f_add(dist, l0[(aa * 4 + bb) * 256 + ((w[aa] >> (8 * bb)) & 0xff)]);
    }
  } else {
    for (int m = 0; m < M; ++m) dist = f_add(dist, lut[m * 256 + rp[m]]);
  }
  return dist;
}

// PQDistCalculator::distance of 4-bit codes (pq/storage.rs:897-906): per code byte i the pair
// LUT[2i][lo] + LUT[2i + 1][hi] is formed first, then the pairs are summed in byte order (cw = M / 2 bytes).
// Not the IVF_PQ scan's exact 4-bit rule, which adds the two entries one after the other.
__device__ __forceinline__ float pq4_pair_distance(const float* lut, const uint8_t* __restrict__ rp, int cw) {
  float dist = 0.0f;
  for (int i = 0; i < cw; ++i) {
    const uint8_t c = __ldg(rp + i);
    dist = f_add(dist, f_add(lut[(2 * i) * 16 + (c & 0xF)], lut[(2 * i + 1) * 16 + (c >> 4)]));
  }
  return dist;
}

}  // namespace lb2
