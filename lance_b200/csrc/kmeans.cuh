// kmeans.cuh -- internal interface of the Lloyd loop (lloyd.cu) and the k-means entry (kmeans.cu)
#pragma once
#include <stdint.h>

#include <vector>

#include "../../include/lance_b200.h"
#include "common.cuh"
namespace lb2 {

// what every Lloyd run of one training shares
struct LloydParams {
  int metric;
  float balance_factor;  // the post-division value (kmeans.rs:1344)
  int max_iters;
  double tolerance;
  uint64_t seed;
};

// B independent Lloyd problems over the columns [b*ds, (b+1)*ds) of x (row stride ldx).  centroids: device [B][K][ds].
void lloyd_train(const float* x, uint64_t n, int ldx, int B, int ds, int K, const LloydParams& p, const float* init_dev,
                 float* centroids, std::vector<double>* loss_out, std::vector<uint32_t>* iters_out);
// k > 256: the reference's hierarchical scheme (kmeans.rs:746-1003); the loss is not meaningful (0)
void hierarchical_train(const float* x, uint64_t n, int d, int K, const LloydParams& p, int hk, float* centroids_out);

// kmeans.rs:1027: the hierarchical tree trains k > 256 centroids that have no initial values
inline bool kmeans_uses_tree(int K, const lb2_kmeans_params& kp, const float* init) {
  return K > 256 && kp.hierarchical_k > 1 && !init;
}
// KMeans::new_with_params on this rank's n rows (every rank of the current communicator passes its own): the balance
// factor divided by the global row count, then the tree or one flat Lloyd run.  loss and iters get one entry each,
// 0 for the tree.
void train_kmeans(const float* x, uint64_t n, int d, int K, int metric, const lb2_kmeans_params& kp, const float* init,
                  float* centroids, std::vector<double>* loss, std::vector<uint32_t>* iters);
}  // namespace lb2
