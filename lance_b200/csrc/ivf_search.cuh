// ivf_search.cuh -- what an IVF search is, for the index (which fills one IvfSearch) and the scan drivers of the
// four index kinds (which run it with their own scan); internal interface of ivf_search.cu
#pragma once
#include <stdint.h>
#include <string.h>

#include "common.cuh"
#include "probe.cuh"
namespace lb2 {
// what FlatIndex::search lets into its heap (flat/index.rs:97-165): the prefilter bitmap over storage
// positions (nullable) and the [lower, upper) range in f32::total_cmp order as signed order keys
struct ScanFilter {
  const uint64_t* allow = nullptr;
  int range = 0;
  int32_t lo_key = 0, hi_key = 0;
};
// total-order key of a float on the host (graph.rs:80-84: f32::total_cmp)
inline int32_t host_total_key(float f) {
  int32_t b;
  memcpy(&b, &f, 4);
  return b ^ (int32_t)((uint32_t)(b >> 31) >> 1);
}
inline ScanFilter make_filter(const uint64_t* allow, int has_lower, float lower, int has_upper, float upper) {
  ScanFilter f;
  f.allow = allow;
  f.range = (has_lower || has_upper) ? 1 : 0;
  // flat/index.rs:101-102: lower_bound.unwrap_or(f32::MIN), upper_bound.unwrap_or(f32::MAX)
  f.lo_key = host_total_key(has_lower ? lower : -3.40282347e+38f);
  f.hi_key = host_total_key(has_upper ? upper : 3.40282347e+38f);
  return f;
}

// One query of a batch whose queries differ in their parameters (lb2_index_search_batch), on the device.  A scan
// kernel reads its slot's query here; a search without the array gives every query IvfSearch::k and ::flt.
struct QueryParam {
  ScanFilter flt;        // the query's prefilter (device bitmap, nullable) and range
  int k;                 // k' = k * max(1, refine_factor): the query's list length (<= IvfSearch::k, the list stride)
  uint32_t ef;           // IVF_HNSW_*: the graph search's ef, >= k'
  const uint32_t* acnt;  // IVF_HNSW_*: allowed rows per partition under the query's prefilter (null: no prefilter)
};

// One search of an IVF index, whatever its kind: the coarse model, the partition layout, the queries (f32,
// normalised for cosine), what to return and where.  pr (nullable): search with the probe rule instead of nprobes
// (k is then k * refine_factor, pr->k the query's k).
// qp (nullable, device [nq]): per-query k' and filter; k is then the largest k', nprobes the largest probe count,
// qnp (device [nq]) each query's own min(nprobes, K), and `filtering` tells whether any query filters.  The merge
// writes query q's k'_q best at out[q * k], padded to k.  With per-query probe rules (pr->qpr) any_range tells whether
// any query has a range, and the candidate lists are held in sub-slabs of about 256 MB.
struct IvfSearch {
  const float* centroids; int K, d, metric;
  const uint64_t* part_offsets; const uint64_t* row_ids;
  const float* queries; uint64_t nq; int k; int nprobes;
  uint64_t* out_ids; float* out_dists; uint32_t* out_counts;
  ScanFilter flt; const ProbeRule* pr;
  const QueryParam* qp = nullptr; const uint32_t* qnp = nullptr; bool any_filter = false, any_range = false;
  const QueryParam* qp_host = nullptr;  // the same table on the host (route choices), with qp
  bool filtering() const { return qp ? any_filter : (flt.allow != nullptr || flt.range != 0); }
  // the per-query values of the queries from q0 on (null without them)
  const QueryParam* qp_at(uint64_t q0) const { return qp ? qp + q0 : nullptr; }
};

// What a scan is asked to fill: the candidate lists of queries [q0, q0 + qn) (at most SEARCH_SLAB of them: the
// grid.y limit), np slots per query.  Slot (q, pi) probes partition probe_ids[q * np + pi] of `offsets` (the
// index's, or with a probe rule its copy with one more, empty, partition); probe_dists are the distances of the
// probed centroids (dist_q_c).  The arrays start at query q0's first slot.
struct ScanSlots {
  uint64_t q0, qn; int np;
  const uint64_t* offsets; const uint32_t* probe_ids; const float* probe_dists;
  float* cand_d; uint64_t* cand_id; uint32_t* cand_cnt;
};
constexpr uint64_t SEARCH_SLAB = 32768;

// a reference to a driver's scan (a lambda over ScanSlots) that lives as long as the call it is passed to
class ScanRef {
  const void* obj;
  void (*call)(const void*, const ScanSlots&);

 public:
  template <class F>
  ScanRef(const F& f) : obj(&f), call([](const void* o, const ScanSlots& s) { (*static_cast<const F*>(o))(s); }) {}
  void operator()(const ScanSlots& s) const { call(obj, s); }
};

// What every driver settles before it launches anything: false when the search is empty; refuses k > 1024, and a
// search whose largest kernel needs more than the device's shared memory (`need` bytes, static included) with the
// driver's own text, which formats `refusal_arg` with one %zu.
bool ivf_search_begin(const IvfSearch& s, size_t need, const char* refusal, size_t refusal_arg);
// the fixed-nprobes skeleton (probe selection, scan, per-query merge), or with a probe rule the per-query one
void run_ivf_search(const IvfSearch& s, ScanRef scan);

void find_partitions_f32(const float* centroids, int K, int d, int metric, const float* queries,
                         uint64_t nq, int nprobes, uint32_t* ids, float* dists);
// np lists of <= k candidates per query -> the k smallest by (distance, row id) per query, ascending; unused slots
// (~0, +inf).  List pi of query q: distances at cand_d[pi * stride_p_d + q * stride_q], ids likewise, count at
// cand_cnt[pi * cnt_stride_p + q * cnt_stride_q].  nl > np: the query's nl lists are merged in groups of np
// (output row q * ceil(nl / np) + group).
// qp (nullable, nl == np): query q keeps its own qp[q].k best (<= k), padded to k.
void merge_lists(const char* name, uint64_t nq, const float* cand_d, const uint64_t* cand_id, const uint32_t* cand_cnt,
                 int np, int k, size_t stride_p_d, size_t stride_p_id, size_t stride_q, size_t cnt_stride_p,
                 size_t cnt_stride_q, uint64_t* out_ids, float* out_dists, uint32_t* out_counts, int nl = 0,
                 const QueryParam* qp = nullptr);
// [nq][nl][k] lists (counts [nq][nl]) -> [nq][k], any nl >= 1, by rank-counting merges only
void merge_list_tree(const char* name, uint64_t nq, const float* cand_d, const uint64_t* cand_id,
                     const uint32_t* cand_cnt, int nl, int k, uint64_t* out_ids, float* out_dists,
                     uint32_t* out_counts);
// all ranks' [nq][k] results of a row-sharded index -> the global top-k by (distance, row id) on every rank
void merge_sharded_topk(const uint64_t* ids, const float* dists, const uint32_t* counts, uint64_t nq, int k,
                        uint64_t* out_ids, float* out_dists, uint32_t* out_counts);
}  // namespace lb2
