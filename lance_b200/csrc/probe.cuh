// probe.cuh -- the per-query probe count of a search with minimum / maximum nprobes (probe.cu)
#pragma once
#include <stdint.h>
namespace lb2 {
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
};
// partitions whose distances fit one block's shared-memory sort; more are sorted in tiles and merged
constexpr int RANK_TILE = 8192;
// dists [nq][K] -> the L smallest (total order of the distance, partition id) per query, ascending: ids / pd [nq][L]
void rank_probes(const float* dists, uint64_t nq, int K, int L, uint32_t* ids, float* pd);
// c[p] = min(kc, rows of partition p the allow bitmap keeps (every row without one))
void partition_counts(const uint64_t* part_offsets, int K, const uint64_t* allow, uint32_t kc, uint32_t* c);
// Per query of a slab: early pruning, min_np and the late-search cutoff -> nsearch[q] partitions to search and
// shortcut[q]; *nmax = max(*nmax, nsearch[q]).  c_p comes from cpart[probe id], or (cpart null) from the scan's own
// list counts cslot[q * slot_stride + t], whose lists past the cutoff are then emptied.  nprobes_out: [nq] or null.
void probe_cutoff(const ProbeRule& r, uint64_t nq, int L, const uint32_t* pids, const float* pd, const uint32_t* cpart,
                  uint32_t* cslot, int slot_stride, uint32_t* nsearch, uint32_t* shortcut, uint32_t* nmax,
                  uint32_t* nprobes_out);
// probe slots [nq][nl]: slot t < nsearch[q] (< L; all L when nsearch is null) is P[t], every other one the empty
// partition `sentinel`
void gather_probes(uint64_t nq, int L, const uint32_t* pids, const float* pd, const uint32_t* nsearch, int nl,
                   uint32_t sentinel, uint32_t* out_ids, float* out_pd);
// list nl - 1 of every query with shortcut[q]: the first kc mask ids (ascending) that none of the query's lists
// 0 .. nl - 2 holds, at +inf; an empty list for the other queries
void shortcut_lists(uint64_t nq, const uint32_t* shortcut, const uint64_t* mask_ids, uint64_t num_mask_ids, int nl,
                    int kc, float* cand_d, uint64_t* cand_id, uint32_t* cand_cnt);
}  // namespace lb2
