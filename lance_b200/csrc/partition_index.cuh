// partition_index.cuh -- the partition index (an HNSW graph over the IVF centroids, partition_index.cu) as the builds
// and the index handle use it; internal interface of partition_index.cu
#pragma once
#include <stdint.h>

#include <memory>

#include "../../include/lance_b200.h"

namespace lb2 {

struct PartitionIndexDeleter {
  void operator()(lb2_partition_index* p) const;
};
using PartitionIndexPtr = std::unique_ptr<lb2_partition_index, PartitionIndexDeleter>;

// may_train_index's rule (utils.rs:67-91): does `mode` give a k x d model over columns of `dtype` a graph?
bool partition_index_uses_graph(uint64_t k, uint32_t d, lb2_dtype dtype, uint32_t mode);
// the graph over the f32 device centroids [k][d] under `metric` (METRIC_L2 / METRIC_DOT; a cosine index passes L2, its
// rows are normalised first) when the mode resolves to it for a column of `dtype`, else null; the refusals of
// lb2_partition_index_build
PartitionIndexPtr partition_index_make(const float* centroids, uint32_t k, uint32_t d, lb2_dtype dtype, int metric,
                                       uint32_t mode, uint64_t seed, uint32_t insert_batch);
// SimpleIndex::search of the f32 device rows x [n][pi.d] (dist / valid nullable)
void partition_index_assign(const lb2_partition_index& pi, const float* x, uint64_t n, uint32_t* part, float* dist,
                            uint8_t* valid);

// The graph's level seed of a build with seed `seed`: distinct from the seeds the build already draws from
// (the IVF sample, k-means, PQ training and the HNSW kinds' levels all take `seed` itself or its PQ offset).
inline uint64_t partition_index_seed(uint64_t seed) { return seed ^ 0x7061727469646978ull; }  // "partidix"

}  // namespace lb2
