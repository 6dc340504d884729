// scan.cuh -- internal interface of pq_scan.cu and flat_scan.cu (the IVF_SQ and IVF_RQ scans: sq.cuh, rq.cuh)
#pragma once
#include <stdint.h>

#include "ivf_search.cuh"
namespace lb2 {
// ---- pq_scan.cu ----
// codes: [n][M] (8-bit) or [n][M / 2] (4-bit) in partition order; slab_off / skew: the skewed copy, or null
void ivfpq_search(const IvfSearch& s, const float* codebook, int M, int nbits, const uint8_t* codes,
                  const uint64_t* slab_off, const uint8_t* skew);
// the conflict-free scan's copy of the codes (8-bit, 16 sub-spaces of 8 dimensions): per 512-row slab and lane the
// lane's 16 rows as one byte stream delayed by lane mod 16 bytes, in 17 coalesced 16-byte units
bool skew_layout_applies(int M, int d, int nbits);
size_t skew_bytes_bound(uint64_t n, int K);
void build_skew_codes(const uint64_t* part_offsets, int K, const uint8_t* codes, uint64_t n, uint64_t* slab_off,
                      uint8_t* skew);
void build_lut_f32(const float* codebook, int M, int nbits, int d, int metric, const float* query,
                   float* lut);
void pq_scan_transposed_f32(const float* lut, int M, int metric, const uint8_t* codes_t, uint64_t n,
                            float* out);
void pq_scan_4bit_f32(const float* lut, int M, int metric, const uint8_t* codes_t, uint64_t n, uint64_t k_hint,
                      float* out);
void pack_nibbles(const uint8_t* codes, uint64_t n, int M, uint8_t* out);
// ---- flat_scan.cu ----
// vectors: the index's rows in element type vdt (lb2_dtype: f32 / f16 / bf16)
void ivfflat_search(const IvfSearch& s, const void* vectors, int vdt);
void refine_f32(const float* queries, uint64_t nq, int d, int metric, const void* vectors, int vdt,
                uint64_t num_vectors, const uint64_t* cand_id, const uint32_t* cand_cnt, int kc, int k,
                uint64_t* out_id, float* out_d, uint32_t* out_cnt, int has_lower = 0, float lower = 0.0f,
                int has_upper = 0, float upper = 0.0f);
// the finish of a batch with per-query values (lb2_index_search_batch), one block per query: query q's merged
// candidates (cand_* [nq][kc], its own k' = qo[q].kc of them at most) -> its k = qo[q].k results in rows of k_stride,
// re-ranked by exact distance within its range when qo[q].refine (refine_f32), else its first k as they are
struct QueryOut {
  int kc, k, refine, has_lower, has_upper;
  float lower, upper;
};
void refine_batch_f32(const float* queries, uint64_t nq, int d, int metric, const void* vectors, int vdt,
                      uint64_t num_vectors, const float* cand_d, const uint64_t* cand_id, const uint32_t* cand_cnt,
                      int kc, const QueryOut* qo, int k_stride, uint64_t* out_id, float* out_d, uint32_t* out_cnt,
                      const uint64_t* positions = nullptr);
// positions [nq][kc] (lb2_index_refine_taken): candidate c of query q is row positions[q][c] of the num_vectors rows
// in `vectors`, not row cand_id[q][c]; the same kernel, only the row source differs
void candidate_rows(const uint64_t* cid, const float* cdist, const uint32_t* ccnt, uint64_t nq, int kc,
                    const QueryOut* qo, int stride, uint64_t* out_id, float* out_d, uint32_t* out_cnt);
// ---- distinct.cu ----
// the ascending distinct values of ids[0, n) below limit into distinct (capacity n; the rest UINT64_MAX), their
// count m into *num_distinct (device), and positions[i] = the index of ids[i] in that list (UINT64_MAX for a value
// at or above limit)
void distinct_ids(const uint64_t* ids, uint64_t n, uint64_t* distinct, uint64_t* num_distinct, uint64_t* positions,
                  uint64_t limit = ~0ull);
void flat_topk_f32(const float* dists, const uint64_t* row_ids, uint64_t n, int k, const ScanFilter& flt,
                   uint64_t* out_id, float* out_d, uint32_t* out_cnt);
// lb2_distance_batch with the reference's per-type rule: u8 L2 / dot (exact integer sums) and f16 / bf16 dot
// (32 lanes); `from` is the f32 view of one row, `to` n rows of element type dt (lb2_dtype)
bool distance_batch_typed_applies(int dt, int metric);
void distance_batch_typed(const float* from, const void* to, int dt, uint64_t n, int d, int metric, float* out);
}  // namespace lb2
