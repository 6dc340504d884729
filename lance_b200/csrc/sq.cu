// sq.cu -- the 8-bit scalar quantizer of IVF_SQ (lance-index/src/vector/sq.rs, sq/builder.rs).
//
// Replaces  ScalarQuantizer::update_bounds   sq.rs:67-89 (the bounds of ScalarQuantizer::build, :152-182)
//           scale_to_u8                      sq.rs:263-277 (quantize / transform, and the query's codes,
//                                            sq/storage.rs:404-430)
//
// The bounds are a min / max: exact in f32 and widened to f64 afterwards, so any reduction order gives the
// reference's fold.  The encoding is restated in f64 with explicitly rounded operations (no mul-add contraction).
#include <algorithm>
#include <cfloat>
#include <vector>

#include "common.cuh"
#include "sq.cuh"

namespace lb2 {

constexpr int SQ_BOUNDS_THREADS = 256;

// per-block (min, max) of the non-NaN elements; +inf / -inf when the block saw none
__global__ void __launch_bounds__(SQ_BOUNDS_THREADS)
sq_bounds_kernel(const float* __restrict__ x, uint64_t count, float2* __restrict__ block_out) {
  float mn = __int_as_float(0x7f800000), mx = __int_as_float(0xff800000);
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (uint64_t)gridDim.x * blockDim.x) {
    const float v = x[i];
    mn = fminf(mn, v);  // fminf / fmaxf return the other operand when one is NaN, like f64::min / f64::max
    mx = fmaxf(mx, v);
  }
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) {
    mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  }
  __shared__ float s_mn[SQ_BOUNDS_THREADS / 32], s_mx[SQ_BOUNDS_THREADS / 32];
  const int warp = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) { s_mn[warp] = mn; s_mx[warp] = mx; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < SQ_BOUNDS_THREADS / 32; ++w) { mn = fminf(mn, s_mn[w]); mx = fmaxf(mx, s_mx[w]); }
    block_out[blockIdx.x] = make_float2(mn, mx);
  }
}

void sq_bounds_f32(const float* x, uint64_t count, double* lower, double* upper) {
  double lo = DBL_MAX, hi = -DBL_MAX;  // (f64::MAX, f64::MIN): what the fold starts from
  if (count) {
    const unsigned nb = (unsigned)std::min<uint64_t>(cdiv(count, SQ_BOUNDS_THREADS), 4ull * ctx().num_sms);
    DevBuf<float2> part(nb);
    std::vector<float2> h(nb);
    LB2_LAUNCH("sq_bounds", sq_bounds_kernel, nb, SQ_BOUNDS_THREADS, 0, x, count, part.p);
    d2h(h.data(), part.p, nb);
    sync_stream();
    for (const float2& b : h) {  // +inf never lowers f64::MAX, -inf never raises f64::MIN
      lo = std::min(lo, (double)b.x);
      hi = std::max(hi, (double)b.y);
    }
  }
  *lower = lo;
  *upper = hi;
}

__global__ void sq_encode_kernel(const float* __restrict__ x, uint64_t count, double lower, double upper,
                                 uint8_t* __restrict__ codes) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  if (lower == upper) {
    codes[i] = 0;
    return;
  }
  const double range = __dsub_rn(upper, lower);
  const double v = __ddiv_rn(__dmul_rn(__dsub_rn((double)x[i], lower), 255.0), range);
  // `v as u8`: NaN -> 0, truncation toward zero, saturating at 0 and 255
  codes[i] = v != v ? 0 : v <= 0.0 ? 0 : v >= 255.0 ? 255 : (uint8_t)v;
}

void sq_encode_f32(const float* x, uint64_t count, double lower, double upper, uint8_t* codes) {
  if (count) LB2_LAUNCH("sq_encode", sq_encode_kernel, cdiv(count, 256), 256, 0, x, count, lower, upper, codes);
}

}  // namespace lb2
