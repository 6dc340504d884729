// tc_assign.cuh -- internal interface of the tensor-core (wgmma) filter path (tc_assign.cu)
#pragma once
#include <stdint.h>

#include "common.cuh"
namespace lb2 {
struct TcWorkspace {
  DevBuf<float> cpad, cnh, row_norm2, cT;  // cT: transposed centroids for the exact kernels
  DevBuf<uint32_t> res, fb_rows, fb_count;
  DevBuf<float> split_scratch;  // short row lists: per (row, 64-centroid chunk) partial argmins (key, val, idx)
  // refinement pass over the rows the first pass left undecided (tc_assign.cu, "refinement")
  DevBuf<float> a3, b3, rn2c;        // [cap][3d] split rows, [Kp][3d] split centroids, their |x|^2
  DevBuf<uint32_t> res2, fb_rows2;   // verdicts of the refinement pass, rows that need the full-K exact scan
  DevBuf<uint32_t> cand;             // candidate pass: [cap] counts + [cap][CAND_SLOTS] column ids
  DevBuf<float> top1_val;            // best score of the last top-3 pass, per undecided row
  DevBuf<uint16_t> cpad16;           // padded centroids as f16 / bf16 (native 16-bit operand path)
  const float* norm_src = nullptr;  // row norms are cached per (pointer, n): valid inside one call
  uint64_t norm_n = 0;
};
bool tc_assign_supported(uint64_t n, int d, int K, int metric, const float* x);
// same contract as assign_f32_ex (L2, no all_out); bit-identical outputs
void tc_assign_f32(const float* x, uint64_t n, int d, const float* cent, int K, const float* bias,
                   uint32_t* part, float* dist, uint8_t* valid, const uint8_t* active,
                   TcWorkspace& ws, const void* x16, int x16_dtype);
}  // namespace lb2
