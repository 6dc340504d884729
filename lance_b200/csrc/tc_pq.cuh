// tc_pq.cuh -- internal interface of the tensor-core (wgmma) PQ code-assignment path (tc_pq.cu)
#pragma once
#include <stdint.h>

#include "common.cuh"
namespace lb2 {
struct TcPqWorkspace {
  DevBuf<float> bm, cnh;  // codebook as a K-major 256 x d matrix; -|c|^2/2 per (m, c) + max|c|^2 per m
  DevBuf<uint32_t> fb_pairs, fb_count;
};
// what a 256-thread block needs to refresh sub-space m's share of the tensor-path operands
// (Bm column block, -|c|^2/2, max|c|^2, empty undecided-row list); used by prep_codebook_kernel and, fused,
// by the k-means epilogue so that a training iteration needs no separate preparation launch
struct TcPqPrepArgs {
  float* bm = nullptr;       // [256][d]
  float* cnh = nullptr;      // [M][256]
  float* cbmax2 = nullptr;   // [M]
  uint32_t* fb_count = nullptr;  // [M]
  int d = 0;
};
#ifdef __CUDACC__
__device__ __forceinline__ void tc_pq_prep_block(const float* __restrict__ cb_m, int m, const TcPqPrepArgs& a,
                                                 float* s_n2 /* [256] shared */) {
  const int c = threadIdx.x;  // blockDim.x == 256 codewords
  const float* src = cb_m + (size_t)c * 8;
  float n2 = 0.0f;
#pragma unroll
  for (int t = 0; t < 8; ++t) {
    const float v = src[t];
    a.bm[(size_t)c * a.d + m * 8 + t] = v;
    n2 += v * v;
  }
  a.cnh[m * 256 + c] = -0.5f * n2;
  s_n2[c] = n2;
  __syncthreads();
  if (c < 32) {
    float mx = 0.0f;
    for (int i = c; i < 256; i += 32) mx = fmaxf(mx, s_n2[i]);
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if (c == 0) a.cbmax2[m] = mx;
  }
}
#endif
bool tc_pq_supported(uint64_t n, int d, int M, int ds, int Kc, int metric, const float* x);
// r_out (nullable) = x - cent[part] (cent nullable -> plain copy skipped); rn2[n][M] = |r_m|^2
void tc_pq_residual_norms(const float* x, const float* cent, const uint32_t* part, uint64_t n, int M,
                          float* r_out, float* rn2);
// codes != NULL: u8 [n][M] (encode); else ids/dists/valid [M][n] (training). Bit-identical to
// pq_assign_f32 on the same inputs.
// prepared = the operands were already refreshed for this codebook (by the fused epilogue)
void tc_pq_assign(const float* r, const float* rn2, uint64_t n, int d, int M, const float* codebook,
                  const uint8_t* row_valid, uint8_t* codes, uint32_t* ids, float* dists,
                  uint8_t* valid, const uint8_t* active, TcPqWorkspace* ws, bool prepared = false);
// allocates the workspace for (M, d) and returns the pointers the fused preparation writes
TcPqPrepArgs tc_pq_prep_args(int M, int d, TcPqWorkspace* ws);
// whole encode of n rows (residual fused when cent/part are given), chunked to bound temp memory
void pq_encode_dev(const float* x, uint64_t n, int d, int M, int ds, const float* codebook, int metric,
                   const float* cent, const uint32_t* part, const uint8_t* row_valid, uint8_t* codes);
}  // namespace lb2
