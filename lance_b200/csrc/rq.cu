// rq.cu -- the RaBitQ quantizer of IVF_RQ (lance-index/src/vector/bq/{builder,transform}.rs).
//
// Replaces  random_orthogonal / householder_qr   bq/builder.rs:309-367 (the rotation of RabitQuantizer::new)
//           RabitQuantizer::transform            bq/builder.rs:143-181 (the sign codes)
//           codes_res_dot_dists                  bq/builder.rs:100-141 (the per-row |rot| sum)
//           RQTransformer::transform             bq/transform.rs:70-220 (add / scale factors)
//           RabitDistCalculator                  bq/storage.rs:160-445 (the partition scan of a search)
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

#include <algorithm>
#include <cfloat>

#include "common.cuh"
#include "exact.cuh"
#include "ivf_search.cuh"
#include "rq.cuh"
#include "topk.cuh"

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

// ------------------------------------------------------------------------------------------------
// IVF_RQ: RabitDistCalculator (lance-index/src/vector/bq/storage.rs:160-445) + top-k, one CTA per (probe, query).
// rq = the slot's rotated residual query (dot(R[i, :d], q - c_p), storage.rs:130-156).  In shared memory:
//   - the code_dim / 4 sub-tables of 16 entries by the lowbit chain t[j] = t[j - lowbit(j)] + rq[4s + ctz(j)]
//     (storage.rs:210-245), which fixes the rounding order;
//   - sum_q = the sequential f32 sum of rq from -0.0 (Rust's float Sum);
//   - the table quantised to u8 with qmin / qmax over the whole table in total_cmp order (storage.rs:249-267).
// distance_all (storage.rs:319-369): the rows before the partition's last n_p % 32 sum u8 entries in 16-bit lanes
// that wrap mod 2^16, as the x86 kernels do (dist_table.rs:96-160, dist_table.c) -- an exact u32 sum & 0xffff --
// and are dequantised as q * ((qmax - qmin) / 255) + (code_dim / 4) * qmin; the last n_p % 32 rows take the exact
// f32 sum of the pairs t_lo[lo] + t_hi[hi] from 0.0.  With a prefilter every row takes DistCalculator::distance
// (storage.rs:297-316), the same pair sums from -0.0; no table entry is -0.0 (t[0] = +0.0 and x + y is -0.0 only
// when both are), so the start does not matter.  Then ((2 dist - sum_q) / sqrt_d) * scale + add + q_factor, each
// operation rounded on its own.  Codes are row-major [n][code_dim / 8]; the 32-row rule uses the partition-local row.
// ------------------------------------------------------------------------------------------------
static size_t rq_scan_smem_bytes(int code_dim, int k) {
  return (size_t)code_dim * 4 * (sizeof(float) + 1) + slot_smem_bytes(k);
}

__global__ void __launch_bounds__(256)
ivfrq_scan_kernel(const float* __restrict__ rq, int code_dim, float sqrt_d, int q_minus_one,
                  const uint32_t* __restrict__ probe_ids, const float* __restrict__ probe_dists, int np,
                  const uint64_t* __restrict__ part_offsets, const uint8_t* __restrict__ codes,
                  const float* __restrict__ add, const float* __restrict__ scale, const uint64_t* __restrict__ row_ids,
                  int k, float* __restrict__ cand_d, uint64_t* __restrict__ cand_id, uint32_t* __restrict__ cand_cnt,
                  const ScanFilter flt0, const QueryParam* __restrict__ qp) {
  extern __shared__ float rq_smem[];
  const int nt = code_dim >> 2;  // sub-tables of 16 entries
  float* tab = rq_smem;                                      // [nt * 16] f32
  uint8_t* qt = reinterpret_cast<uint8_t*>(tab + nt * 16);  // [nt * 16] u8 (code_dim % 8 == 0: 4-byte aligned end)
  __shared__ int32_t s_mn, s_mx;
  __shared__ float s_sum_q;
  const int tid = threadIdx.x;
  size_t qi, slot;
  uint32_t p, n_p;
  uint64_t off;
  if (!slot_partition(probe_ids, np, part_offsets, cand_cnt, qi, slot, p, off, n_p)) return;
  const int kq = query_k(qp, qi, k);  // k: the lists' stride
  const ScanFilter flt = query_filter(qp, qi, flt0);
  const SlotSmem s(qt + nt * 16, kq + 1);
  const float* r = rq + slot * (size_t)code_dim;
  if (tid == 0) { s_mn = 0x7fffffff; s_mx = (int32_t)0x80000000; }
  for (int st = tid; st < nt; st += 256) {
    float t[16];
    t[0] = 0.0f;
#pragma unroll
    for (int j = 1; j < 16; ++j) {
      const int ctz = (j & 1) ? 0 : (j & 2) ? 1 : (j & 4) ? 2 : 3;
      t[j] = __fadd_rn(t[j - (j & -j)], r[4 * st + ctz]);
    }
#pragma unroll
    for (int j = 0; j < 16; ++j) tab[st * 16 + j] = t[j];
  }
  __syncthreads();
  int32_t mn = 0x7fffffff, mx = (int32_t)0x80000000;
  for (int i = tid; i < nt * 16; i += 256) {
    const int32_t kv = total_order_key(tab[i]);
    mn = min(mn, kv);
    mx = max(mx, kv);
  }
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) {
    mn = min(mn, __shfl_xor_sync(0xffffffffu, mn, o));
    mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  }
  if ((tid & 31) == 0) { atomicMin(&s_mn, mn); atomicMax(&s_mx, mx); }
  if (tid == 0) {
    float sq = -0.0f;
    for (int i = 0; i < code_dim; ++i) sq = __fadd_rn(sq, r[i]);
    s_sum_q = sq;
  }
  __syncthreads();
  const float qmin = key_to_float(s_mn), qmax = key_to_float(s_mx);
  if (flt.allow == nullptr) {
    const bool flat = qmin == qmax;  // e.g. a zero residual query: all codes 0
    const float factor = flat ? 0.0f : __fdiv_rn(255.0f, __fsub_rn(qmax, qmin));
    for (int i = tid; i < nt * 16; i += 256) {
      const float v = flat ? 0.0f : roundf(__fmul_rn(__fsub_rn(tab[i], qmin), factor));  // f32::round
      qt[i] = (v != v) ? 0 : v <= 0.0f ? 0 : v >= 255.0f ? 255 : (uint8_t)v;           // `as u8`
    }
  }
  __syncthreads();
  const float range = __fdiv_rn(__fsub_rn(qmax, qmin), 255.0f), sum_min = __fmul_rn((float)nt, qmin);
  const float sum_q = s_sum_q, dqc = probe_dists[slot];
  const float q_factor = q_minus_one ? __fsub_rn(dqc, 1.0f) : dqc;  // storage.rs:427-434
  const int cb = code_dim >> 3;
  const uint8_t* pc = codes + off * cb;
  const uint32_t n_quant = flt.allow ? 0u : n_p - n_p % 32;
  auto fill = [&](uint32_t c0, uint32_t clen) {
    for (uint32_t j = tid; j < clen; j += 256) {
      const uint32_t row = c0 + j;
      const uint8_t* rp = pc + (size_t)row * cb;
      float dist;
      if (row < n_quant) {
        uint32_t qs = 0;
        for (int i = 0; i < cb; ++i) {
          const uint32_t c = __ldg(rp + i);
          qs += (uint32_t)qt[(2 * i) * 16 + (c & 15)] + (uint32_t)qt[(2 * i + 1) * 16 + (c >> 4)];
        }
        dist = __fadd_rn(__fmul_rn(__uint2float_rn(qs & 0xffffu), range), sum_min);
      } else {
        dist = 0.0f;
        for (int i = 0; i < cb; ++i) {
          const uint32_t c = __ldg(rp + i);
          dist = __fadd_rn(dist, __fadd_rn(tab[(2 * i) * 16 + (c & 15)], tab[(2 * i + 1) * 16 + (c >> 4)]));
        }
      }
      const float dvq = __fdiv_rn(__fsub_rn(__fmul_rn(2.0f, dist), sum_q), sqrt_d);
      float out = __fadd_rn(__fadd_rn(__fmul_rn(dvq, scale[off + row]), add[off + row]), q_factor);
      // x86's default NaN (0xFFC00000, ordered before every number): with finite rows a NaN only comes from invalid
      // operations, e.g. on a normalised zero query under cosine, and the reference runs on x86
      if (out != out) out = __int_as_float(0xffc00000);
      s.ukey[j] = (uint32_t)total_order_key(out) ^ 0x80000000u;
    }
  };
  const uint32_t cnt = slot_topk(s, n_p, kq, flt, off, false, fill);
  write_slot(s, cnt, slot, k, off, row_ids, cand_d, cand_id, cand_cnt);
}

// residual queries of `nq` queries x np probes: out[(q np + pi) d + t] = queries[q d + t] - c_{probe}[t]
// (a probe id >= K is an empty slot of a search with minimum / maximum nprobes: its residual is 0)
__global__ void rq_query_residual_kernel(const float* __restrict__ queries, uint64_t nq, int np, int d,
                                         const float* __restrict__ centroids, int K,
                                         const uint32_t* __restrict__ probe_ids, float* __restrict__ out) {
  const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= nq * np * d) return;
  const uint64_t sl = g / d;
  const int t = (int)(g % d);
  const uint32_t p = probe_ids[sl];
  out[g] = p < (uint32_t)K ? __fsub_rn(queries[(sl / np) * d + t], centroids[(size_t)p * d + t]) : 0.0f;
}

bool rq_scan_fits(int code_dim, int k) {
  return smem_with_static(ivfrq_scan_kernel, rq_scan_smem_bytes(code_dim, k)) <= ctx().smem_optin;
}

void ivfrq_search(const IvfSearch& s, const float* rotation, int code_dim, const uint8_t* codes, const float* add,
                  const float* scale) {
  const int d = s.d, k = s.k;
  const size_t smem = rq_scan_smem_bytes(code_dim, k);
  if (!ivf_search_begin(s, smem_with_static(ivfrq_scan_kernel, smem),
                        "IVF_RQ: the tables of code_dim %zu do not fit the scan's shared memory", (size_t)code_dim))
    return;
  const float sqrt_d = sqrtf((float)code_dim);  // (dim as f32 * num_bits as f32).sqrt(): the product is exact
  const int q_minus_one = s.metric != METRIC_L2;  // the storage's metric: cosine / dot -> dist_q_c - 1.0
  run_ivf_search(s, [&](const ScanSlots& sl) {
    const int np = sl.np;
    // the (query, probe) residuals are rotated in groups of queries that keep both buffers near 256 MB
    const uint64_t per_q = (uint64_t)np * (d + code_dim) * sizeof(float);
    const uint64_t qc = std::max<uint64_t>(1, std::min<uint64_t>(sl.qn, (256ull << 20) / per_q));
    DevBuf<float> res(qc * np * d), rot(qc * np * code_dim);
    set_smem(ivfrq_scan_kernel, smem);
    for (uint64_t a = 0; a < sl.qn; a += qc) {
      const uint64_t b = std::min(qc, sl.qn - a);
      LB2_LAUNCH("rq_query_residual", rq_query_residual_kernel, cdiv(b * np * d, 256), 256, 0,
                 s.queries + (sl.q0 + a) * d, b, np, d, s.centroids, s.K, sl.probe_ids + a * np, res.p);
      rq_rotate_f32(rotation, code_dim, d, res.p, b * np, rot.p);
      LB2_LAUNCH("rq_scan", ivfrq_scan_kernel, dim3(np, (unsigned)b), 256, smem, rot.p, code_dim, sqrt_d, q_minus_one,
                 sl.probe_ids + a * np, sl.probe_dists + a * np, np, sl.offsets, codes, add, scale, s.row_ids, k,
                 sl.cand_d + a * np * k, sl.cand_id + a * np * k, sl.cand_cnt + a * np, s.flt, s.qp_at(sl.q0 + a));
    }
  });
}

}  // namespace lb2
