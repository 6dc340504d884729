// hnsw.cuh -- the per-partition HNSW graphs of IVF_HNSW_SQ, IVF_HNSW_PQ and IVF_HNSW_FLAT
// (lance-index/src/vector/hnsw/builder.rs) and their device layout; internal interface of hnsw.cu
#pragma once
#include <stdint.h>

#include <vector>

#include "common.cuh"
namespace lb2 {
struct IvfSearch;

// One graph per partition over the partition's storage order (node i = storage position off_p + i).
//   level 0, dense over every row:  cnt0[n], nbr0[n][2m] (partition-local node ids), dst0[n][2m]
//   levels 1.., compact:            a node with L levels owns rows up_base[row] .. up_base[row] + L - 2, one per
//                                   level 1 .. L-1, each cntu, nbru[m], dstu[m]
// Lists keep the reference's order of level_neighbors_ranked (graph/builder.rs:33-48); the distances are those of
// the ranked list.  Node 0 of every partition has max_level levels and is the entry point (builder.rs:354-376).
struct HnswGraph {
  const char* kind = "IVF_HNSW_SQ";  // the index kind's name in messages: IVF_HNSW_SQ, IVF_HNSW_PQ or IVF_HNSW_FLAT
  int max_level = 0, m = 0, ef_construction = 0;
  uint32_t insert_batch = 1;  // B of the batched build (1: serial; a loaded graph records 1)
  uint64_t max_part = 0;      // rows of the largest partition (scratch sizing)
  uint64_t n_up = 0;      // upper-level rows
  DevBuf<uint8_t> nlev;
  DevBuf<uint32_t> up_base, cnt0, nbr0, cntu, nbru;
  DevBuf<float> dst0, dstu;
};

// The level thresholds of random_level (builder.rs:386-393): node i >= 1 of a partition gets 1 + #{l in 1 ..
// max_level - 1 : u < thr[l]} levels, u the u32 draw of hnsw_level_draw; thr[l] = floor(2^32 / m^l), so P(level >= l)
// is m^-l as in the reference's -ln(r) / ln(m).  thr[0] is unused.
void hnsw_level_thresholds(int m, int max_level, uint64_t* thr);
// the counter-based draw of node i of partition p (splitmix64 of seed + (p << 32 | i) * golden ratio, high half)
inline uint32_t hnsw_level_draw(uint64_t seed, uint32_t p, uint32_t i) {
  uint64_t x = seed + ((((uint64_t)p << 32) | i) * 0x9E3779B97F4A7C15ull);
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  x ^= x >> 31;
  return (uint32_t)(x >> 32);
}

// The partitions of a rebuilt index whose graphs are kept from an older graph of the same parameters: new partition
// p takes old partition src[p]'s graph verbatim when src[p] >= 0 (its rows are all of src[p]'s rows, in order; node
// ids are partition-local, so levels, lists and distances carry over), and is built from its storage otherwise.
struct HnswKeep {
  const HnswGraph* old = nullptr;
  std::vector<uint64_t> old_off;  // the old index's part_offsets [old K + 1]
  std::vector<int64_t> src;       // [new K]: old partition id, or -1 = build this partition
};

// HNSW::index_vectors (builder.rs:742-775) of every partition, nodes inserted 1 .. n_p - 1 in ascending order, or in
// rounds of up to g.insert_batch concurrent inserts when it is above 1 (the round definition of include/lance_b200.h);
// codes [n][d] in partition order, part_offsets on the device.  Fills g (its parameters set by the caller).  With
// `keep`, only the partitions keep->src marks -1 are built; the others are spliced from keep->old.
void hnsw_build(HnswGraph& g, const uint64_t* part_offsets, int K, const uint8_t* codes, int d, int metric, float r2,
                uint64_t seed, const HnswKeep* keep = nullptr);
// the same over PQ codes [n][cw] (cw = M, or M / 2 for 4-bit codes) with the codebook [M][2^nbits][d / M]: a node's
// descent, beam searches and lists use the table of its decoded codes, the heuristic the decoded rows' distance with
// the rule of `dtype` (pq/storage.rs:675-841)
void hnsw_build_pq(HnswGraph& g, const uint64_t* part_offsets, int K, const uint8_t* codes, const float* codebook,
                   int d, int M, int nbits, int metric, lb2_dtype dtype, uint64_t seed, const HnswKeep* keep = nullptr);
// the same over IVF_FLAT's stored rows [n][d] in element type `vdt` (f32, f16 or bf16): every distance, cosine
// included, is the IVF_FLAT scan's rule (flat/storage.rs:345-410)
void hnsw_build_flat(HnswGraph& g, const uint64_t* part_offsets, int K, const void* vectors, int vdt, int d, int metric,
                     uint64_t seed, const HnswKeep* keep = nullptr);
// a graph from the caller's arrays in the layout above (host or device memory), checked against the partitions
void hnsw_load(HnswGraph& g, const uint64_t* part_offsets, int K, const uint8_t* levels, const uint32_t* counts0,
               const uint32_t* nbr0, const float* dist0, const uint32_t* counts_up, const uint32_t* nbr_up,
               const float* dist_up);
// out[0] = 0, out[i + 1] = in[0] + .. + in[i] for i < n, on the device (out has n + 1 entries)
void scan_u64(const uint64_t* in, uint64_t n, uint64_t* out);
// The graphs in the reference's storage layout (HNSW::to_batch / HNSW::load, builder.rs:579-640,788-833), every
// partition's level batches back to back (include/lance_b200.h, lb2_index_storage).  hnsw_storage_edges: the number
// of list entries.  hnsw_to_storage: every output a device pointer or NULL; level_offsets [K][max_level + 1],
// vector_id [rows], list_offsets [rows + 1] (global), neighbors / distances [edges], rows = n + g.n_up.
uint64_t hnsw_storage_edges(const HnswGraph& g, uint64_t n);
void hnsw_to_storage(const HnswGraph& g, const uint64_t* part_offsets, int K, uint64_t n, uint64_t* level_offsets,
                     uint32_t* vector_id, uint64_t* list_offsets, uint32_t* neighbors, float* distances);
// the inverse into g (max_level, m, ef_construction, kind set by the caller; device inputs): the storage checks on the
// device, then hnsw_load of the dense layout.  LB2_INVALID_ARG on malformed input, before g is filled.
void hnsw_from_storage(HnswGraph& g, const uint64_t* part_offsets, int K, uint64_t n, const uint32_t* entry_point,
                       const uint64_t* level_offsets, const uint32_t* vector_id, const uint64_t* list_offsets,
                       const uint32_t* neighbors, const float* distances, uint64_t rows, uint64_t edges);
// HNSW::search (builder.rs:678-739) as the scan of every probed partition; ef = 0: k' + k' / 2 (builder.rs:563-573)
void hnsw_search(const IvfSearch& s, const HnswGraph& g, const uint8_t* codes, float r2, const uint8_t* qcodes,
                 uint32_t ef);
// the same over PQ codes: each slot's table is the IVF_PQ scan's table of the (residual) query
void hnsw_search_pq(const IvfSearch& s, const HnswGraph& g, const float* codebook, int M, int nbits,
                    const uint8_t* codes, uint32_t ef);
// the same over IVF_FLAT's stored rows: each slot scores rows with the IVF_FLAT scan's rule for the (normalised) query
void hnsw_search_flat(const IvfSearch& s, const HnswGraph& g, const void* vectors, int vdt, uint32_t ef);
}  // namespace lb2
