// index.cuh -- the device-resident index handle and what the builds need to fill one
#pragma once
#include <memory>

#include "hnsw.cuh"
#include "partition_index.cuh"
#include "staging.cuh"

namespace lb2 {
enum class IndexKind { PQ, FLAT, SQ, RQ };
}  // namespace lb2

// the handle
struct lb2_index {
  lb2::IndexKind kind = lb2::IndexKind::PQ;
  lb2_dtype dtype = LB2_F32;  // element type of the vectors / queries the caller passes
  // IVF_FLAT: the (normalised for cosine) vectors in partition order, in the vectors' own element type
  // (f32 / f16 / bf16; u8 columns are held as f32, the reference's model type for them, ivf.rs:1917-1929)
  lb2::DevBuf<uint8_t> vectors;
  lb2_dtype vdtype() const { return dtype == LB2_U8 ? LB2_F32 : dtype; }
  int K = 0, d = 0, M = 0, nbits = 0, metric = 0;
  uint64_t n = 0;
  lb2::DevBuf<float> centroids, codebook;
  lb2::DevBuf<uint64_t> part_offsets, row_ids;
  lb2::DevBuf<uint8_t> codes;
  // the conflict-free scan's skewed copy of `codes` (pq_scan.cu: ivfpq_scan_skew_kernel); empty for other shapes
  lb2::DevBuf<uint64_t> slab_off;
  lb2::DevBuf<uint8_t> codes_skew;
  // IVF_SQ: `codes` are the 8-bit scalar codes [n][d] of the (normalised for cosine) vectors, under the bounds
  // [sq_lower, sq_upper] (sq/storage.rs:38-45)
  double sq_lower = 0.0, sq_upper = 0.0;
  // IVF_RQ: `codes` are the sign codes [n][code_dim / 8] of the rotated residuals (num_bits = nbits, code_dim =
  // d * nbits), with the per-row factors rq_add / rq_scale [n] and the rotation rq_rot [code_dim][code_dim]
  // (bq/storage.rs:110-121)
  lb2::DevBuf<float> rq_rot, rq_add, rq_scale;
  // IVF_HNSW_SQ / IVF_HNSW_PQ / IVF_HNSW_FLAT: an IVF_SQ / IVF_PQ / IVF_FLAT index with an HNSW graph per partition
  // over its codes or vectors (hnsw.cuh), searched through the graphs instead of the partition scan
  std::unique_ptr<lb2::HnswGraph> hnsw;
  // how rows are assigned to partitions (lb2_partition_index_mode, partition_index.cuh): the mode, the graph's level
  // seed and insert_batch, and the graph over the centroids when the mode resolves to one (null: the exact scan).
  // lb2_index_transform, IVF_RQ's split transform and the indexes optimize / split / join return follow it.
  uint32_t pi_mode = LB2_PARTITION_INDEX_EXACT;
  uint64_t pi_seed = 0;
  uint32_t pi_batch = 1;
  lb2::PartitionIndexPtr pidx;
  int code_dim() const { return d * nbits; }
  size_t codebook_len() const { return ((size_t)1 << nbits) * d; }
  // a row's payload in partition order: IVF_FLAT's vectors, the codes of every other kind
  lb2::DevBuf<uint8_t>& payload() { return kind == lb2::IndexKind::FLAT ? vectors : codes; }
  const lb2::DevBuf<uint8_t>& payload() const { return kind == lb2::IndexKind::FLAT ? vectors : codes; }
  // bytes per row of payload() (PQ: pq.rs:168-173; SQ: one per dimension; RQ: one bit per code dimension)
  size_t row_bytes() const {
    switch (kind) {
      case lb2::IndexKind::FLAT: return (size_t)d * (vdtype() == LB2_F32 ? 4 : 2);
      case lb2::IndexKind::SQ: return d;
      case lb2::IndexKind::RQ: return code_dim() / 8;
      case lb2::IndexKind::PQ: break;
    }
    return nbits == 4 ? M / 2 : M;
  }
};

namespace lb2 {

// an index of `kind` with room for K centroids and nothing else; M and nbits are 0
std::unique_ptr<lb2_index> make_index(IndexKind kind, uint32_t K, uint32_t d, int metric, lb2_dtype dtype);
// a partition id >= K (a corrupted / mismatched shuffle file) would index device memory out of bounds
void check_part_ids(const uint32_t* part_ids, uint64_t n, uint32_t K, const char* what);
// stable grouping of n rows' payloads (row_bytes() each: codes, or IVF_FLAT's stored rows) by partition; rows with
// valid[r] == 0 are dropped; rq_add / rq_scale (IVF_RQ only): the rows' factors, grouped with their codes
void index_load_dev(lb2_index* ix, const uint32_t* part_ids, const uint8_t* codes, const uint64_t* row_ids,
                    uint64_t n, const uint8_t* valid = nullptr, const float* rq_add = nullptr,
                    const float* rq_scale = nullptr);
// IVF_FLAT storage from the caller's matrix (normalised when `normalize`)
void index_load_flat_src(lb2_index* ix, const uint32_t* part_ids, Source& src, const uint64_t* row_ids,
                         const uint8_t* valid, bool normalize);

// the model of `from` in `to`, an index of the same kind from make_index: the centroids (or new_centroids, in the
// model type of the index), M, nbits, and the codebook, SQ bounds or RQ rotation
void copy_model(const lb2_index* from, lb2_index* to, const void* new_centroids = nullptr);
// the name of the graph kind over an index of `kind` in messages: IVF_HNSW_SQ, IVF_HNSW_PQ or IVF_HNSW_FLAT
const char* hnsw_kind_name(IndexKind kind);
// an empty graph of these parameters (hnsw/builder.rs:63-72; max_level and m range-checked) over an index of `kind`;
// insert_batch 0 or 1 is the serial build, and what a loaded graph records
std::unique_ptr<HnswGraph> new_graph(IndexKind kind, uint32_t max_level, uint32_t m, uint32_t ef_construction,
                                     uint32_t insert_batch = 1);
// the graphs of ix built (hnsw_build, under the hnsw_build tag; `keep`: the partitions spliced from an older graph)
// and attached; an IVF_PQ index's skewed code copy is released, as only the IVF_PQ scan reads it
void attach_graph(lb2_index* ix, uint32_t max_level, uint32_t m, uint32_t ef_construction, uint32_t insert_batch,
                  uint64_t seed, const HnswKeep* keep = nullptr);
// ix's partition rule: mode, level seed and insert_batch recorded, and the graph over ix's centroids built when the
// mode resolves to one (lb2_index_set_partition_index, the builds, and the indexes optimize / split / join return)
void set_partition_index(lb2_index* ix, uint32_t mode, uint64_t seed, uint32_t insert_batch);
// lb2_index_optimize's merge into a new index; add_valid (nullable, device [n_add]): added rows with 0 are left out
std::unique_ptr<lb2_index> index_merge(const lb2_index* old, const lb2_optimize_params& p, const char* what,
                                       const uint8_t* add_valid = nullptr);

}  // namespace lb2
