// search.cuh -- internal interface of search.cu
#pragma once
#include <stdint.h>
#include <string.h>

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
void find_partitions_f32(const float* centroids, int K, int d, int metric, const float* queries,
                         uint64_t nq, int nprobes, uint32_t* ids, float* dists);
void ivfpq_search_f32(const float* centroids, int K, int d, int metric, const float* codebook, int M,
                      int nbits, const uint64_t* part_offsets, const uint8_t* codes,
                      const uint64_t* row_ids, const float* queries, uint64_t nq, int k, int nprobes,
                      uint64_t* out_ids, float* out_dists, uint32_t* out_counts,
                      const ScanFilter& flt = ScanFilter(), const uint64_t* slab_off = nullptr,
                      const uint8_t* skew = nullptr, const ProbeRule* pr = nullptr);
// the conflict-free scan's copy of the codes (8-bit, 16 sub-spaces of 8 dimensions): per 512-row slab and lane the
// lane's 16 rows as one byte stream delayed by lane mod 16 bytes, in 17 coalesced 16-byte units
bool skew_layout_applies(int M, int d, int nbits);
size_t skew_bytes_bound(uint64_t n, int K);
void build_skew_codes(const uint64_t* part_offsets, int K, const uint8_t* codes, uint64_t n, uint64_t* slab_off,
                      uint8_t* skew);
// vectors: the index's rows in element type vdt (lb2_dtype: f32 / f16 / bf16)
void ivfflat_search_f32(const float* centroids, int K, int d, int metric, const uint64_t* part_offsets,
                        const void* vectors, int vdt, const uint64_t* row_ids, const float* queries, uint64_t nq,
                        int k, int nprobes, uint64_t* out_ids, float* out_dists, uint32_t* out_counts,
                        const ScanFilter& flt = ScanFilter(), const ProbeRule* pr = nullptr);
// codes: the index's SQ codes [n][d] in partition order; qcodes: the queries' codes [nq][d] under the same bounds;
// r2 = rf * rf with rf = (float)(upper - lower); queries: f32 (normalised for cosine), for the probe selection
void ivfsq_search_f32(const float* centroids, int K, int d, int metric, const uint64_t* part_offsets,
                      const uint8_t* codes, const uint64_t* row_ids, float r2, const float* queries,
                      const uint8_t* qcodes, uint64_t nq, int k, int nprobes, uint64_t* out_ids, float* out_dists,
                      uint32_t* out_counts, const ScanFilter& flt = ScanFilter(), const ProbeRule* pr = nullptr);
// pr (nullable): search with the probe rule instead of nprobes (the search's k is k * refine_factor, pr->k the
// query's k)
// IVF_RQ: rotation [code_dim][code_dim]; codes [n][code_dim / 8] and the add / scale factors [n] in partition order;
// queries: f32 (normalised for cosine).  rq_scan_fits: the scan's tables and a k-slot fit shared memory.
bool rq_scan_fits(int code_dim, int k);
void ivfrq_search_f32(const float* centroids, int K, int d, int metric, const float* rotation, int code_dim,
                      const uint64_t* part_offsets, const uint8_t* codes, const float* add, const float* scale,
                      const uint64_t* row_ids, const float* queries, uint64_t nq, int k, int nprobes,
                      uint64_t* out_ids, float* out_dists, uint32_t* out_counts, const ScanFilter& flt = ScanFilter(),
                      const ProbeRule* pr = nullptr);
// all ranks' [nq][k] results of a row-sharded index -> the global top-k by (distance, row id) on every rank
void merge_sharded_topk(const uint64_t* ids, const float* dists, const uint32_t* counts, uint64_t nq, int k,
                        uint64_t* out_ids, float* out_dists, uint32_t* out_counts);
// bit i of bitmap = RowIdMask::selected(row_ids[i]) (lance-core/src/utils/mask.rs:84-93); lists sorted
void row_mask_f32(const uint64_t* row_ids, uint64_t n, const uint64_t* allow, uint64_t n_allow, bool has_allow,
                  const uint64_t* block, uint64_t n_block, bool has_block, uint64_t* bitmap);
void refine_f32(const float* queries, uint64_t nq, int d, int metric, const void* vectors, int vdt,
                uint64_t num_vectors, const uint64_t* cand_id, const uint32_t* cand_cnt, int kc, int k,
                uint64_t* out_id, float* out_d, uint32_t* out_cnt, int has_lower = 0, float lower = 0.0f,
                int has_upper = 0, float upper = 0.0f);
void build_lut_f32(const float* codebook, int M, int nbits, int d, int metric, const float* query,
                   float* lut);
void pq_scan_transposed_f32(const float* lut, int M, int metric, const uint8_t* codes_t, uint64_t n,
                            float* out);
void pq_scan_4bit_f32(const float* lut, int M, int metric, const uint8_t* codes_t, uint64_t n, uint64_t k_hint,
                      float* out);
void pack_nibbles(const uint8_t* codes, uint64_t n, int M, uint8_t* out);
void flat_topk_f32(const float* dists, const uint64_t* row_ids, uint64_t n, int k, const ScanFilter& flt,
                   uint64_t* out_id, float* out_d, uint32_t* out_cnt);
}  // namespace lb2
