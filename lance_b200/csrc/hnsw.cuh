// hnsw.cuh -- the per-partition HNSW graphs of IVF_HNSW_SQ, IVF_HNSW_PQ and IVF_HNSW_FLAT
// (lance-index/src/vector/hnsw/builder.rs) and their device layout; internal interface of hnsw.cu
#pragma once
#include <stdint.h>

#include <vector>

#include "common.cuh"
struct lb2_index;
namespace lb2 {
struct IvfSearch;

// One graph per partition over the partition's storage order (node i = storage position off_p + i).
//   level 0, dense over every row:  cnt0[n], nbr0[n][2m] (partition-local node ids), dst0[n][2m]
//   levels 1.., compact:            a node with L levels owns rows up_base[row] .. up_base[row] + L - 2, one per
//                                   level 1 .. L-1, each cntu, nbru[m], dstu[m]
// Lists keep the reference's order of level_neighbors_ranked (graph/builder.rs:33-48); the distances are those of
// the ranked list.  Node 0 of every partition has max_level levels and is the entry point (builder.rs:354-376).
struct HnswGraph {
  const char* kind = nullptr;  // the index kind's name in messages (hnsw_kind_name)
  int max_level = 0, m = 0, ef_construction = 0;
  uint32_t insert_batch = 1;  // B of the batched build (1: serial; a loaded graph records 1)
  uint64_t max_part = 0;      // rows of the largest partition (scratch sizing)
  uint64_t n_up = 0;      // upper-level rows
  DevBuf<uint8_t> nlev;
  DevBuf<uint32_t> up_base, cnt0, nbr0, cntu, nbru;
  DevBuf<float> dst0, dstu;
};

// the layout as the kernels see it
struct GraphDev {
  const uint8_t* nlev;
  const uint32_t* up_base;
  uint32_t *cnt0, *nbr0, *cntu, *nbru;
  float *dst0, *dstu;
  int m, max_level;
};
inline GraphDev dev_view(const HnswGraph& g) {
  return GraphDev{g.nlev.p, g.up_base.p, g.cnt0.p, g.nbr0.p, g.cntu.p, g.nbru.p, g.dst0.p, g.dstu.p, g.m, g.max_level};
}
struct ListRef {
  uint32_t* cnt;
  uint32_t* ids;
  float* dist;
};
// the list of global row `row` at `level`
__device__ __forceinline__ ListRef list_of(const GraphDev& g, uint64_t row, int level) {
  if (level == 0) return {g.cnt0 + row, g.nbr0 + row * 2 * g.m, g.dst0 + row * 2 * g.m};
  const uint64_t r = (uint64_t)g.up_base[row] + (level - 1);
  return {g.cntu + r, g.nbru + r * g.m, g.dstu + r * g.m};
}

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

// HNSW::index_vectors (builder.rs:742-775) of every partition of ix over its payload (codes or rows in partition
// order), nodes inserted 1 .. n_p - 1 in ascending order, or in rounds of up to g.insert_batch concurrent inserts when
// it is above 1 (the round definition of include/lance_b200.h), with the distances of ix's kind (hnsw.cu: SqDist,
// PqDist, FlatDist).  Fills g (its parameters set by the caller).  With `keep`, only the partitions keep->src marks -1
// are built; the others are spliced from keep->old.
void hnsw_build(HnswGraph& g, const lb2_index& ix, uint64_t seed, const HnswKeep* keep = nullptr);
// the same build over one partition of n f32 rows on the device (d % 4 == 0), with IVF_HNSW_FLAT's f32 distances
// under L2 (METRIC_L2) or dot (METRIC_DOT): the graph over the centroids of a partition index (partition_index.cu)
void hnsw_build_rows(HnswGraph& g, const float* rows, uint64_t n, int d, int metric, uint64_t seed);
// a graph from the caller's arrays in the layout above (host or device memory), checked against the partitions
void hnsw_load(HnswGraph& g, const uint64_t* part_offsets, int K, const uint8_t* levels, const uint32_t* counts0,
               const uint32_t* nbr0, const float* dist0, const uint32_t* counts_up, const uint32_t* nbr_up,
               const float* dist_up);
// HNSW::search (builder.rs:678-739) as the scan of every probed partition, through ix's graphs with the distances of
// ix's kind: the IVF_SQ scan's on sq_query_codes (s's queries encoded, IVF_HNSW_SQ only), the IVF_PQ scan's tables or
// the IVF_FLAT scan's rule.  ef = 0: k' + k' / 2 (builder.rs:563-573)
void hnsw_search(const IvfSearch& s, const lb2_index& ix, const uint8_t* sq_query_codes, uint32_t ef);
}  // namespace lb2
