// assign.cuh -- internal interface of the exact nearest-centroid kernels (assign.cu)
#pragma once
#include <stdint.h>

#include "tc_assign.cuh"
namespace lb2 {
// part/dist/valid are [n] (dist and valid nullable): each row's nearest centroid, its distance, and 0 in valid where
// no centroid is at a finite distance.  bias (nullable, [K]) is added for the comparison only (kernels.rs:92-111).
// x16 (nullable): the same rows as x in their own element type x16_dtype (LB2_F16 / LB2_BF16); the tensor-core
// filter may read them instead of x (tc_assign.cu, "native 16-bit rows").
void assign_f32(const float* x, uint64_t n, int d, const float* cent, int K, int metric,
                const float* bias, uint32_t* part, float* dist, uint8_t* valid,
                const void* x16 = nullptr, int x16_dtype = 0);
// same, with an optional device-side `active` flag (active[0] == 0 -> the kernels return immediately; used by the
// Lloyd loop) and the caller's workspace (a training loop keeps one across iterations and its CUDA graph)
void assign_f32_ex(const float* x, uint64_t n, int d, const float* cent, int K, int metric,
                   const float* bias, uint32_t* part, float* dist, uint8_t* valid,
                   const uint8_t* active, TcWorkspace& ws,
                   const void* x16 = nullptr, int x16_dtype = 0);
// the full [n][K] distance matrix, out[r * K + k] = dist(x[r], cent[k]), by the same exact kernels
void centroid_distances(const float* x, uint64_t n, int d, const float* cent, int K, int metric, float* out);
// exact tile kernel restricted to row_list[0 .. *row_count) (both on the device)
void assign_rows_f32(const float* x, uint64_t n_max, int d, const float* cent, int K, int metric,
                     const float* bias, const uint32_t* row_list, const uint32_t* row_count,
                     uint32_t* part, float* dist, uint8_t* valid, const uint8_t* active,
                     TcWorkspace& ws, bool cT_ready);
// PQ code assignment, batched over the M sub-spaces: x row stride ldx, sub-space m reads columns [m*ds,(m+1)*ds)
// (minus the same columns of ivf_centroids[part_ids[row]] when given).  Every ds >= 1 has an exact route:
// small_d_kernel below 16, pq_wide_kernel up to PQ_WIDE_MAX_DS, assign_f32_ex per sub-space beyond.
// codes != NULL -> u8 [n][M] out (PQ encode), else ids/dists/valid [M][n] (PQ training); active[m] == 0 skips
// sub-space m.  ws (nullable): scratch of the wide routes, kept by a caller that captures the call into a CUDA graph.
constexpr int PQ_WIDE_MAX_DS = 256;
struct PqAssignWorkspace {
  DevBuf<float> cbT;    // [M][ds][Kp] transposed codebooks (pq_wide_kernel)
  DevBuf<float> sub;    // one sub-space's rows, contiguous (ds > PQ_WIDE_MAX_DS)
  DevBuf<uint32_t> ids;  // ... their codewords and valid flags before the u8 codes are written
  DevBuf<uint8_t> ok;
  TcWorkspace tc;
};
void pq_assign_f32(const float* x, uint64_t n, int ldx, int M, int ds, const float* codebook, int Kc, int metric,
                   const float* ivf_centroids, const uint32_t* part_ids, const uint8_t* row_valid, uint8_t* codes,
                   uint32_t* ids, float* dists, uint8_t* valid, const uint8_t* active,
                   PqAssignWorkspace* ws = nullptr);
}  // namespace lb2
