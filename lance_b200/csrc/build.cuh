// build.cuh -- the parts of the index builds that the stand-alone primitives and the index handle share
#pragma once
#include "staging.cuh"

struct lb2_index;

namespace lb2 {

// x - centroid of its partition, row by row (x and out may alias: the in-place residual of the PQ training sample)
__global__ void residual_kernel(const float* x, const float* __restrict__ cent, const uint32_t* __restrict__ part,
                                uint64_t n, int d, float* out);

// What a ProductQuantizer of M sub-vectors and num_bits codes needs: M divides d (pq/utils.rs:25) and num_bits is 4
// or 8 (ENCODE, i.e. wherever codes exist: M is even for 4-bit codes, pq.rs:132-140).  Every sub-vector width has
// an exact encode route (pq_assign_f32).
enum class PqUse { TRAIN, ENCODE };
void check_pq_shape(uint32_t d, uint32_t M, uint32_t nbits, PqUse use);
void check_redos(uint32_t redos, float balance_factor);
void pq_train_dev(const float* data, uint64_t n, int d, int metric, const lb2_pq_params* p, float* codebook,
                  std::vector<uint32_t>* iters);
void pq_encode_any(const float* x, uint64_t n, int d, int M, int ds, const float* codebook, int metric,
                   const float* cent, const uint32_t* part, const uint8_t* row_valid, int nbits, uint8_t* codes);
void sq_check_dim(uint32_t d);
void rq_check(uint32_t d, lb2_dtype dtype, uint32_t num_bits);
// the transform of every row of `src` with the model and partition rule of `index`, for the builds, the stand-alone
// transforms and a split (every output nullable, device; IVF_FLAT's NULL payload is not written; synchronises only
// for scratch); given_part (nullable): the rows' partitions are given, and IVF_PQ takes its residuals to them
void index_transform_rows(const lb2_index* index, Source& src, const uint32_t* given_part, uint32_t* part_out,
                          uint8_t* payload_out, float* add_out, float* scale_out, uint8_t* valid_out);

}  // namespace lb2
