// rq.cuh -- internal interface of rq.cu (the RaBitQ quantizer of IVF_RQ)
#pragma once
#include <stdint.h>
namespace lb2 {
// a code_dim x code_dim orthogonal matrix, row-major, f32: the Q factor of a Householder QR of a standard-normal
// f64 matrix drawn with Philox from `seed`, cast with round to nearest even
void rq_rotation_f32(int code_dim, uint64_t seed, float* out);
// Y[m][j] = dot(R[j, :d], X[m]) for j < code_dim, in the reference's 16-lane f32 order (dot.rs:30-58);
// R is [code_dim][code_dim], X is [m][d]
void rq_rotate_f32(const float* R, int code_dim, int d, const float* X, uint64_t m, float* Y);
// out[i] = x[i] - centroids[part[i]], elementwise f32 (residual.rs:86-95); rows with valid[i] == 0 become zero
void rq_residual_f32(const float* x, uint64_t m, int d, const float* centroids, const uint32_t* part,
                     const uint8_t* valid, float* out);
// norm_squared_fsl (lance-linalg/src/distance/norm_l2.rs:141-157): sequential f32 sum of squares per row
void rq_norm_sq_f32(const float* x, uint64_t m, int d, float* out);
// RQTransformer::transform (bq/transform.rs:70-220) from the rotated residuals: sign codes [m][code_dim / 8]
// (LSB-first), add and scale factors.  metric: METRIC_L2 (cosine is L2 on normalised rows) or METRIC_DOT.
// dist_v_c: the assignment's distance; cnorm_sq: |c|^2 per centroid (dot only).  Rows with valid == 0 get zeros.
void rq_encode_f32(const float* rot, const float* residual, const float* dist_v_c, const uint32_t* part,
                   const float* cnorm_sq, const uint8_t* valid, uint64_t m, int d, int num_bits, int metric,
                   uint8_t* codes, float* add, float* scale);
// IVF_RQ: rotation [code_dim][code_dim]; codes [n][code_dim / 8] and the add / scale factors [n] in partition order;
// s.queries: f32 (normalised for cosine).  rq_scan_fits: the scan's tables and a k-slot fit shared memory.
struct IvfSearch;
bool rq_scan_fits(int code_dim, int k);
void ivfrq_search(const IvfSearch& s, const float* rotation, int code_dim, const uint8_t* codes, const float* add,
                  const float* scale);
}  // namespace lb2
