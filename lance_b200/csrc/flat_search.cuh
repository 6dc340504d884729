// flat_search.cuh -- internal interface of flat_search.cu: flat KNN over one vector column, batched over queries
#pragma once
#include <stdint.h>

#include <vector>

#include "common.cuh"

namespace lb2 {
// What flat_knn lets through (scanner.rs:3336-3411): rows whose bit is set in `allow` (nullable; bit i = row i in
// input order) and whose exact distance d has lower <= d < upper (SQL comparisons: a NaN distance fails either bound).
struct FlatFilter {
  const uint64_t* allow = nullptr;
  int has_lower = 0, has_upper = 0;
  float lower = 0.0f, upper = 0.0f;
};

// One query of a batch whose queries differ in k and filter (flat_search_batch), on the device: allow is a device
// bitmap (or null), k its own list length.
struct FlatQuery {
  FlatFilter flt;
  int k = 0;
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
// the FlatQuery table of a batch (P: lb2_flat_query_params or lb2_query_params): query q's k and range, and the staged
// bitmap bm[filter_q] (bm: device pointers, one per filter), or `none` for a query without a filter
template <class P>
std::vector<FlatQuery> flat_queries(const P* params, uint64_t nq, const std::vector<const uint64_t*>& bm,
                                    const uint64_t* none) {
  std::vector<FlatQuery> fq(nq);
  for (uint64_t q = 0; q < nq; ++q) {
    const P& p = params[q];
    fq[q].flt.allow = p.filter == UINT32_MAX ? none : bm[p.filter];
    fq[q].flt.has_lower = p.has_lower_bound != 0;
    fq[q].flt.has_upper = p.has_upper_bound != 0;
    fq[q].flt.lower = p.lower_bound;
    fq[q].flt.upper = p.upper_bound;
    fq[q].k = (int)p.k;
  }
  return fq;
}
// flat_search_check for flat_search_batch, whose largest k is kmax
void flat_search_batch_check(int d, lb2_dtype dt, int metric, int kmax);
// flat_search with every query's own k and filter: fq_host [nq] (host; its bitmaps on the device).  Row q of the
// outputs ([nq][k_stride], device) is flat_search of query q alone with fq_host[q], slots k_q.. (~0, +inf); out_counts
// nullable.  The launches depend on n, nq and the chunking, not on how many distinct (k, filter) sets the batch holds.
void flat_search_batch(const float* queries, uint64_t nq, int d, int metric, const void* vectors, uint64_t n,
                       lb2_dtype dt, const uint64_t* row_ids, const FlatQuery* fq_host, int k_stride,
                       uint64_t* out_ids, float* out_dists, uint32_t* out_counts);
}  // namespace lb2
