// probe.cuh -- the per-query probe count of a search with minimum / maximum nprobes (probe.cu)
#pragma once
#include <stdint.h>
namespace lb2 {
struct QueryProbe;
// Query::minimum_nprobes / maximum_nprobes and the prefilter's allow list as ANNIvfSubIndexExec sees them
// (rust/lance/src/io/exec/knn.rs:714-882, 1108-1130).  k is the query's k, not k * refine_factor.
struct ProbeRule {
  uint32_t min_np = 1, max_np = 0;  // max_np 0: every partition
  uint32_t late_width = 1;          // partitions the late search keeps in flight
  uint32_t k = 0;
  int has_max_len = 0;
  uint64_t max_len = 0;
  const uint64_t* mask_ids = nullptr;  // device, ascending; null: the allow list is not iterable (no shortcut)
  uint64_t num_mask_ids = 0;
  uint32_t* nprobes_out = nullptr;     // device [nq] partitions searched, nullable
  // a batch (lb2_index_search_batch): each query's own rule, device [nq]; the fields above then describe the batch:
  // max_np its largest L (0: K), mask_ids non-null when any query may take the shortcut
  const QueryProbe* qpr = nullptr;
};
// one query's probe rule in a batch: its bounds (L = min(max_np or K, K)), k, k' = kc, its allow list's max_len and
// ids, and cpart = the rows of each partition its prefilter keeps (uncapped; every row without one).  ranged: the query
// has a range, so its c_p are its scan's list counts; a query without one keeps c_p from cpart even when the batch
// scans first (an IVF_HNSW_* list may hold fewer rows than its partition admits)
struct QueryProbe {
  uint32_t min_np, L, k, kc;
  int ranged, has_max_len;
  uint64_t max_len;
  const uint64_t* mask_ids;  // null: not iterable
  uint64_t num_mask_ids;
  const uint32_t* cpart;
};
// partitions whose distances fit one block's shared-memory sort; more are sorted in tiles and merged
constexpr int RANK_TILE = 8192;
// dists [nq][K] -> the L smallest (total order of the distance, partition id) per query, ascending: ids / pd [nq][L]
void rank_probes(const float* dists, uint64_t nq, int K, int L, uint32_t* ids, float* pd);
// c[p] = min(kc, rows of partition p the allow bitmap keeps (every row without one))
void partition_counts(const uint64_t* part_offsets, int K, const uint64_t* allow, uint32_t kc, uint32_t* c);
// c[f][p] = rows of partition p that bitmap allows[f] keeps (uncapped), for nf bitmaps (allows: device [nf]), one launch
void partition_counts_table(const uint64_t* part_offsets, int K, const uint64_t* const* allows, int nf, uint32_t* c);
// Per query of a slab: early pruning, min_np and the late-search cutoff -> nsearch[q] partitions to search and
// shortcut[q]; *nmax = max(*nmax, nsearch[q]).  c_p comes from cpart[probe id], or (cpart null) from the scan's own
// list counts cslot[q * slot_stride + t], whose lists past the cutoff are then emptied.  nprobes_out: [nq] or null.
// qpr (nullable; the slab's): per-query rules, whose own cpart (capped by the query's k') replaces `cpart` unless the
// counts come from the scan (cslot) and the query has a range.
void probe_cutoff(const ProbeRule& r, uint64_t nq, int L, const uint32_t* pids, const float* pd, const uint32_t* cpart,
                  uint32_t* cslot, int slot_stride, uint32_t* nsearch, uint32_t* shortcut, uint32_t* nmax,
                  uint32_t* nprobes_out, const QueryProbe* qpr = nullptr);
// probe slots [nq][nl]: slot t < nsearch[q] (< L; all L when nsearch is null) is P[t], every other one the empty
// partition `sentinel`; qpr (nullable, the slab's): without nsearch, slot t < the query's own L
void gather_probes(uint64_t nq, int L, const uint32_t* pids, const float* pd, const uint32_t* nsearch, int nl,
                   uint32_t sentinel, uint32_t* out_ids, float* out_pd, const QueryProbe* qpr = nullptr);
// list nl - 1 of every query with shortcut[q]: the first kc mask ids (ascending) that none of the query's lists
// 0 .. nl - 2 holds, at +inf; an empty list for the other queries.  qpr (nullable, the slab's): each query's own
// mask ids and k' (kc is then the lists' stride)
void shortcut_lists(uint64_t nq, const uint32_t* shortcut, const uint64_t* mask_ids, uint64_t num_mask_ids, int nl,
                    int kc, float* cand_d, uint64_t* cand_id, uint32_t* cand_cnt, const QueryProbe* qpr = nullptr);
}  // namespace lb2
