// rq.cu -- the RaBitQ quantizer of IVF_RQ (lance-index/src/vector/bq/{builder,transform}.rs).
//
// Replaces  random_orthogonal / householder_qr   bq/builder.rs:309-367 (the rotation of RabitQuantizer::new)
//           RabitQuantizer::transform            bq/builder.rs:143-181 (the sign codes)
//           codes_res_dot_dists                  bq/builder.rs:100-141 (the per-row |rot| sum)
//           RQTransformer::transform             bq/transform.rs:70-220 (add / scale factors)
//
// Exactness: the reference rotates data rows with an ndarray GEMM whose summation order is unspecified.  Here the
// rotation of a row is defined as the query side's rotation, the 16-lane f32 `dot` (dot.rs:30-58, the order of
// dist_exact_thread<METRIC_DOT> in exact.cuh), and the |rot| sum as a sequential sum.  Codes, factors and the search
// are then bit-identical to a CPU restatement; against the reference's GEMM a code bit can only differ where the
// rotated component lies below that GEMM's rounding bound.
//
// The rotation matrix: the reference draws it from an unseeded rng, so no bit-level parity exists; any orthogonal
// matrix is an equally valid model.  Ours is the Q factor of a Householder QR of a Philox standard-normal f64
// matrix, with the reference's sign convention; each reflection is applied as a rank-1 update (O(n^3)), never
// formed as a matrix.
#include <curand_kernel.h>

#include <cfloat>

#include "common.cuh"
#include "exact.cuh"
#include "rq.cuh"

namespace lb2 {

__global__ void rq_normal_kernel(uint64_t count, uint64_t seed, double* __restrict__ a) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  curandStatePhilox4_32_10_t st;
  curand_init(seed, i, 0, &st);
  a[i] = curand_normal_double(&st);
}

__global__ void rq_eye_kernel(int n, double* __restrict__ q) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < (uint64_t)n * n) q[i] = (i / n == i % n) ? 1.0 : 0.0;
}

__device__ __forceinline__ double block_sum_256(double v, double* red) {
  const int tid = threadIdx.x;
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((tid & 31) == 0) red[tid >> 5] = v;
  __syncthreads();
  double s = 0.0;
  for (int w = 0; w < 8; ++w) s += red[w];
  __syncthreads();
  return s;
}

// step k: u = the unit Householder vector of column k of A below the diagonal (builder.rs:323-334);
// ok = 0 when that column's norm is below f64::EPSILON (the step is skipped)
__global__ void __launch_bounds__(256) rq_hh_vector_kernel(const double* __restrict__ a, int n, int k,
                                                           double* __restrict__ u, int* __restrict__ ok) {
  __shared__ double red[8];
  const int len = n - k, tid = threadIdx.x;
  double s = 0.0;
  for (int i = tid; i < len; i += 256) {
    const double x = a[(size_t)(k + i) * n + k];
    s += x * x;
  }
  const double xnorm = sqrt(block_sum_256(s, red));
  if (xnorm < DBL_EPSILON) {
    if (tid == 0) *ok = 0;
    return;
  }
  const double x0 = a[(size_t)k * n + k];
  const double x0n = x0 + (x0 >= 0.0 ? 1.0 : -1.0) * xnorm;
  s = 0.0;
  for (int i = tid; i < len; i += 256) {
    const double x = i == 0 ? x0n : a[(size_t)(k + i) * n + k];
    s += x * x;
  }
  const double unorm = sqrt(block_sum_256(s, red));
  for (int i = tid; i < len; i += 256) u[i] = (i == 0 ? x0n : a[(size_t)(k + i) * n + k]) / unorm;
  if (tid == 0) *ok = 1;
}

// w[j] = sum_i u[i] A[k + i][k + j] (j < n - k): the row vector u^T A[k.., k..]
__global__ void rq_hh_w_kernel(const double* __restrict__ a, int n, int k, const double* __restrict__ u,
                               const int* __restrict__ ok, double* __restrict__ w) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (!*ok || j >= n - k) return;
  double s = 0.0;
  for (int i = 0; i < n - k; ++i) s += u[i] * a[(size_t)(k + i) * n + k + j];
  w[j] = s;
}

// v[i] = sum_j Q[i][k + j] u[j] (i < n): Q[.., k..] u, one warp per row
__global__ void rq_hh_v_kernel(const double* __restrict__ q, int n, int k, const double* __restrict__ u,
                               const int* __restrict__ ok, double* __restrict__ v) {
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (!*ok || i >= n) return;
  double s = 0.0;
  for (int j = lane; j < n - k; j += 32) s += q[(size_t)i * n + k + j] * u[j];
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) v[i] = s;
}

// A[k.., k..] = H A[k.., k..] and Q[.., k..] = Q[.., k..] H with H = I - 2 u u^T, as rank-1 updates
__global__ void rq_hh_update_kernel(double* __restrict__ a, double* __restrict__ q, int n, int k,
                                    const double* __restrict__ u, const double* __restrict__ w,
                                    const double* __restrict__ v, const int* __restrict__ ok) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x, i = blockIdx.y;
  if (!*ok || j >= n - k) return;
  q[(size_t)i * n + k + j] -= 2.0 * v[i] * u[j];
  if (i >= k) a[(size_t)i * n + k + j] -= 2.0 * u[i - k] * w[j];
}

__global__ void rq_cast_kernel(const double* __restrict__ q, uint64_t count, float* __restrict__ out) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < count) out[i] = __double2float_rn(q[i]);
}

void rq_rotation_f32(int n, uint64_t seed, float* out) {
  const uint64_t nn = (uint64_t)n * n;
  DevBuf<double> a(nn), q(nn), u(n), w(n), v(n);
  DevBuf<int> ok(1);
  LB2_LAUNCH("rq_normal", rq_normal_kernel, cdiv(nn, 256), 256, 0, nn, seed, a.p);
  LB2_LAUNCH("rq_eye", rq_eye_kernel, cdiv(nn, 256), 256, 0, n, q.p);
  for (int k = 0; k + 1 < n; ++k) {  // k in 0..min(n, m - 1) (builder.rs:318)
    LB2_LAUNCH("rq_householder", rq_hh_vector_kernel, 1, 256, 0, a.p, n, k, u.p, ok.p);
    LB2_LAUNCH("rq_householder", rq_hh_w_kernel, cdiv(n - k, 128), 128, 0, a.p, n, k, u.p, ok.p, w.p);
    LB2_LAUNCH("rq_householder", rq_hh_v_kernel, cdiv((uint64_t)n * 32, 256), 256, 0, q.p, n, k, u.p, ok.p, v.p);
    LB2_LAUNCH("rq_householder", rq_hh_update_kernel, dim3(cdiv(n - k, 128), (unsigned)n), 128, 0, a.p, q.p, n, k,
               u.p, w.p, v.p, ok.p);
  }
  LB2_LAUNCH("rq_cast", rq_cast_kernel, cdiv(nn, 256), 256, 0, q.p, nn, out);
  sync_stream();
}

// ---- Y[m][j] = dot(R[j, :d], X[m]) in the reference's order --------------------------------------------------
// One output per thread: the d % 16 tail summed first, then 16 lane accumulators over the 16-wide chunks, folded
// 0..15, then tail + fold (dot.rs:30-58).  A CTA computes RT_M rows x RT_J outputs; tiles of RT_K columns of R and
// X are staged in shared memory so that one R tile serves RT_M rows and one X tile RT_J outputs.
constexpr int RT_J = 32, RT_M = 8, RT_K = 64;

__global__ void __launch_bounds__(256) rq_rotate_kernel(const float* __restrict__ R, int code_dim, int d,
                                                        const float* __restrict__ X, uint64_t m,
                                                        float* __restrict__ Y) {
  __shared__ float rs[RT_J][RT_K + 1];
  __shared__ float xs[RT_M][RT_K];
  const int tj = threadIdx.x & 31, tm = threadIdx.x >> 5;
  const uint64_t r0 = (uint64_t)blockIdx.x * RT_M;
  const int j0 = blockIdx.y * RT_J;
  const int n16 = d & ~15;
  float acc[16];
#pragma unroll
  for (int l = 0; l < 16; ++l) acc[l] = 0.0f;
  for (int c0 = 0; c0 < n16; c0 += RT_K) {
    const int kc = min(RT_K, n16 - c0);  // a multiple of 16
    for (int t = threadIdx.x; t < RT_J * RT_K; t += 256) {
      const int jj = t / RT_K, cc = t % RT_K;
      rs[jj][cc] = (j0 + jj < code_dim && cc < kc) ? R[(size_t)(j0 + jj) * code_dim + c0 + cc] : 0.0f;
    }
    for (int t = threadIdx.x; t < RT_M * RT_K; t += 256) {
      const int mm = t / RT_K, cc = t % RT_K;
      xs[mm][cc] = (r0 + mm < m && cc < kc) ? X[(r0 + mm) * d + c0 + cc] : 0.0f;
    }
    __syncthreads();
#pragma unroll
    for (int cb = 0; cb < RT_K; cb += 16) {
      if (cb < kc) {
#pragma unroll
        for (int l = 0; l < 16; ++l) acc[l] = __fadd_rn(acc[l], __fmul_rn(rs[tj][cb + l], xs[tm][cb + l]));
      }
    }
    __syncthreads();
  }
  const int j = j0 + tj;
  const uint64_t r = r0 + tm;
  if (j >= code_dim || r >= m) return;
  const float* xr = X + r * d;
  const float* rr = R + (size_t)j * code_dim;
  float s = 0.0f;
  for (int i = n16; i < d; ++i) s = __fadd_rn(s, __fmul_rn(rr[i], xr[i]));
  float t = 0.0f;
#pragma unroll
  for (int l = 0; l < 16; ++l) t = __fadd_rn(t, acc[l]);
  Y[r * code_dim + j] = __fadd_rn(s, t);
}

void rq_rotate_f32(const float* R, int code_dim, int d, const float* X, uint64_t m, float* Y) {
  if (m == 0) return;
  LB2_LAUNCH("rq_rotate", rq_rotate_kernel, dim3(cdiv(m, RT_M), cdiv(code_dim, RT_J)), 256, 0, R, code_dim, d, X, m,
             Y);
}

__global__ void rq_residual_kernel(const float* __restrict__ x, uint64_t m, int d, const float* __restrict__ cent,
                                   const uint32_t* __restrict__ part, const uint8_t* __restrict__ valid,
                                   float* __restrict__ out) {
  const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= m * d) return;
  const uint64_t r = g / d;
  out[g] = (valid && !valid[r]) ? 0.0f : __fsub_rn(x[g], cent[(size_t)part[r] * d + g % d]);
}

void rq_residual_f32(const float* x, uint64_t m, int d, const float* centroids, const uint32_t* part,
                     const uint8_t* valid, float* out) {
  if (m) LB2_LAUNCH("rq_residual", rq_residual_kernel, cdiv(m * d, 256), 256, 0, x, m, d, centroids, part, valid, out);
}

__global__ void rq_norm_sq_kernel(const float* __restrict__ x, uint64_t m, int d, float* __restrict__ out) {
  const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= m) return;
  float s = 0.0f;
  for (int i = 0; i < d; ++i) s = __fadd_rn(s, __fmul_rn(x[r * d + i], x[r * d + i]));
  out[r] = s;
}

void rq_norm_sq_f32(const float* x, uint64_t m, int d, float* out) {
  if (m) LB2_LAUNCH("rq_norm_sq", rq_norm_sq_kernel, cdiv(m, 128), 128, 0, x, m, d, out);
}

// One warp per row.  Bit j of a row = rot[j].is_sign_positive(), LSB-first (BitVec<u8, Lsb0>, builder.rs:170-173):
// lane l of a ballot over rot[32 w + l] is bit l of the little-endian word w, i.e. bytes 4w .. 4w + 3.
// ip = (sequential sum of |rot[j]|) / sqrt(code_dim); res_norm_sq = dist_v_c (L2) or the sequential sum of
// squares of the residual (dot); add = res_norm_sq (L2) or dist_v_c + |c|^2 (dot); scale = (-2 res_norm_sq) / ip (L2)
// or -(res_norm_sq / ip) (dot), where a zero ip gives a zero quotient (div_checked(..).unwrap_or_default()).
__global__ void rq_encode_kernel(const float* __restrict__ rot, const float* __restrict__ res,
                                 const float* __restrict__ dvc, const uint32_t* __restrict__ part,
                                 const float* __restrict__ cn, const uint8_t* __restrict__ valid, uint64_t m, int d,
                                 int code_dim, float sqrt_d, int metric, uint8_t* __restrict__ codes,
                                 float* __restrict__ add, float* __restrict__ scale) {
  const uint64_t row = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= m) return;  // warp-uniform
  const int cb = code_dim >> 3;
  uint8_t* co = codes + row * cb;
  if (valid && !valid[row]) {
    for (int b = lane; b < cb; b += 32) co[b] = 0;
    if (lane == 0) add[row] = scale[row] = 0.0f;
    return;
  }
  const float* rr = rot + row * code_dim;
  float ip = 0.0f;
  for (int j0 = 0; j0 < code_dim; j0 += 32) {
    const bool in = j0 + lane < code_dim;
    const float v = in ? rr[j0 + lane] : 0.0f;
    const unsigned bits = __ballot_sync(0xffffffffu, in && !signbit(v));
    if (lane < min(4, (code_dim - j0) >> 3)) co[(j0 >> 3) + lane] = (uint8_t)(bits >> (8 * lane));
    const int cnt = min(32, code_dim - j0);
    for (int i = 0; i < cnt; ++i) ip = __fadd_rn(ip, fabsf(__shfl_sync(0xffffffffu, v, i)));
  }
  ip = __fdiv_rn(ip, sqrt_d);
  float rns = 0.0f;
  if (metric == METRIC_DOT) {
    const float* xr = res + row * d;
    for (int i0 = 0; i0 < d; i0 += 32) {
      const float x = i0 + lane < d ? xr[i0 + lane] : 0.0f;
      const int cnt = min(32, d - i0);
      for (int i = 0; i < cnt; ++i) {
        const float xi = __shfl_sync(0xffffffffu, x, i);
        rns = __fadd_rn(rns, __fmul_rn(xi, xi));
      }
    }
  } else {
    rns = dvc[row];
  }
  if (lane) return;
  if (metric == METRIC_DOT) {
    add[row] = __fadd_rn(dvc[row], cn[part[row]]);
    scale[row] = -(ip == 0.0f ? 0.0f : __fdiv_rn(rns, ip));
  } else {
    add[row] = rns;
    scale[row] = ip == 0.0f ? 0.0f : __fdiv_rn(__fmul_rn(-2.0f, rns), ip);
  }
}

void rq_encode_f32(const float* rot, const float* residual, const float* dist_v_c, const uint32_t* part,
                   const float* cnorm_sq, const uint8_t* valid, uint64_t m, int d, int num_bits, int metric,
                   uint8_t* codes, float* add, float* scale) {
  if (m == 0) return;
  const int code_dim = d * num_bits;
  const float sqrt_d = sqrtf((float)d * (float)num_bits);  // (dim as f32 * num_bits as f32).sqrt(), builder.rs:137
  LB2_LAUNCH("rq_encode", rq_encode_kernel, cdiv(m * 32, 256), 256, 0, rot, residual, dist_v_c, part, cnorm_sq, valid,
             m, d, code_dim, sqrt_d, metric, codes, add, scale);
}

}  // namespace lb2
