// sq.cuh -- internal interface of sq.cu: the 8-bit scalar quantizer (lance-index/src/vector/sq.rs)
#pragma once
#include <stdint.h>

#include "exact.cuh"
namespace lb2 {
// The SQ distance of two code rows (the IVF_SQ scan, and the IVF_HNSW_SQ graph build and search): an exact u32 sum
// over 4-byte words of codes -- l2_distance_uint_scalar (lance-linalg/src/distance/l2.rs:44-49) for L2 / cosine, the
// u8 dot (dot.rs:152-161) for dot -- so any split over lanes and any order gives the reference's integer; then
// inverse_scalar_dist (sq.rs:279-287) in f32: (f * r2) / 255^2 with f = s as f32 (dot: 1 - s as f32), r2 = rf * rf.
template <int METRIC>
__device__ __forceinline__ uint32_t sq_word(uint32_t x, uint32_t q, uint32_t acc) {
  if (METRIC == METRIC_DOT) return __dp4a(x, q, acc);
  const uint32_t df = __vabsdiffu4(x, q);
  return __dp4a(df, df, acc);
}
template <int METRIC>
__device__ __forceinline__ float sq_distance(uint32_t acc, float r2) {
  float f = __uint2float_rn(acc);
  if (METRIC == METRIC_DOT) f = __fsub_rn(1.0f, f);
  return __fdiv_rn(__fmul_rn(f, r2), 65025.0f);
}

// ScalarQuantizer::update_bounds (sq.rs:67-89): the fold of every element of x[count] (f32 values) as f64 from
// (f64::MAX, f64::MIN) with f64::min / f64::max, so NaN elements are ignored.  Blocks until the bounds are known.
void sq_bounds_f32(const float* x, uint64_t count, double* lower, double* upper);
// scale_to_u8 (sq.rs:263-277) of x[count]: ((v - lower) * 255 / (upper - lower)) in f64, `as u8` (truncation toward
// zero, saturating, NaN -> 0); every code is 0 when lower == upper.  Stream-ordered, no synchronisation.
void sq_encode_f32(const float* x, uint64_t count, double lower, double upper, uint8_t* codes);
// codes: the index's SQ codes [n][d] in partition order; qcodes: the queries' codes [nq][d] under the same bounds;
// r2 = rf * rf with rf = (float)(upper - lower); s.queries: f32 (normalised for cosine), for the probe selection
struct IvfSearch;
void ivfsq_search(const IvfSearch& s, const uint8_t* codes, float r2, const uint8_t* qcodes);
}  // namespace lb2
