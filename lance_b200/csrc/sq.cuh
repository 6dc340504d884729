// sq.cuh -- internal interface of sq.cu: the 8-bit scalar quantizer (lance-index/src/vector/sq.rs)
#pragma once
#include <stdint.h>
namespace lb2 {
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
