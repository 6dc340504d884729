// flat_search.cuh -- internal interface of flat_search.cu: flat KNN over one vector column, batched over queries
#pragma once
#include <stdint.h>

#include "common.cuh"

namespace lb2 {
// What flat_knn lets through (scanner.rs:3336-3411): rows whose bit is set in `allow` (nullable; bit i = row i in
// input order) and whose exact distance d has lower <= d < upper (SQL comparisons: a NaN distance fails either bound).
struct FlatFilter {
  const uint64_t* allow = nullptr;
  int has_lower = 0, has_upper = 0;
  float lower = 0.0f, upper = 0.0f;
};

// Refuses k > 1024 and a dimension whose query tile does not fit shared memory (LB2_UNSUPPORTED), before anything
// else happens.
void flat_search_check(int d, lb2_dtype dt, int metric, int k);
// The k smallest (distance, row id) pairs of every query over the n rows of `vectors` ([n][d] in element type dt,
// host or device memory: device rows are read in place, host rows are staged chunk by chunk).  queries: [nq][d] f32 on
// the device, holding values of type dt; row_ids (device, nullable = 0..n): distinct; outputs on the device: [nq][k]
// ascending, unused slots (~0, +inf), counts [nq].
void flat_search(const float* queries, uint64_t nq, int d, int metric, const void* vectors, uint64_t n, lb2_dtype dt,
                 const uint64_t* row_ids, const FlatFilter& flt, int k, uint64_t* out_ids, float* out_dists,
                 uint32_t* out_counts);
}  // namespace lb2
