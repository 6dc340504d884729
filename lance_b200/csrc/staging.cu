// staging.cu -- element-type conversion, the staging cache of host-sourced builds and training samples
#include "staging.cuh"

namespace lb2 {

// kernels.rs:141-146: norm = sqrt(sum x^2) accumulated sequentially in f32, then x / norm
// (x and out may be the same buffer: a row is read completely before it is written)
__global__ void normalize_kernel(const float* x, uint64_t n, int d, float* out) {
  const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const float* v = x + r * d;
  float s = 0.0f;
  for (int i = 0; i < d; ++i) s = f_add(s, __fmul_rn(v[i], v[i]));
  const float norm = __fsqrt_rn(s);
  for (int i = 0; i < d; ++i) out[r * d + i] = __fdiv_rn(v[i], norm);
}

// KeepFiniteVectors (lance-index/src/vector/transform.rs:86-159) / the is_finite filter applied to the training
// sample (rust/lance/src/index/vector/builder.rs:436); warp per row.  flag[r] = every element of row r is finite,
// or with clear_only: flag[r] = 0 for a row with a non-finite element, other flags left as they are
__global__ void finite_rows_kernel(const float* __restrict__ x, uint64_t n, int d, uint8_t* __restrict__ flag,
                                   int clear_only) {
  const uint64_t w = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= n) return;
  bool ok = true;
  for (int e = lane; e < d; e += 32) ok &= isfinite(x[w * d + e]);
  ok = __all_sync(0xffffffffu, ok);
  if (lane == 0 && !(clear_only && ok)) flag[w] = ok ? 1 : 0;
}

__global__ void to_f32_kernel(const void* __restrict__ in, int dt, size_t count, float* __restrict__ out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  if (dt == LB2_F16) out[i] = __half2float(reinterpret_cast<const __half*>(in)[i]);
  else if (dt == LB2_BF16) out[i] = __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(in)[i]);
  else out[i] = (float)reinterpret_cast<const uint8_t*>(in)[i];
}
__global__ void from_f32_kernel(const float* __restrict__ in, int dt, size_t count, void* __restrict__ out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  if (dt == LB2_F16) reinterpret_cast<__half*>(out)[i] = __float2half_rn(in[i]);
  else reinterpret_cast<__nv_bfloat16*>(out)[i] = __float2bfloat16_rn(in[i]);
}

// gather rows of a matrix of any element type into f32 (training samples, fallback rows)
__global__ void gather_rows_typed_kernel(const void* __restrict__ x, int dt, const uint64_t* __restrict__ rows,
                                         uint64_t s, int d, float* __restrict__ out) {
  const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= s * d) return;
  const size_t src = (size_t)rows[g / d] * d + g % d;
  float v;
  if (dt == LB2_F32) v = reinterpret_cast<const float*>(x)[src];
  else if (dt == LB2_F16) v = __half2float(reinterpret_cast<const __half*>(x)[src]);
  else if (dt == LB2_BF16) v = __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(x)[src]);
  else v = (float)reinterpret_cast<const uint8_t*>(x)[src];
  out[g] = v;
}
// The same gather for f32 rows with d % 4 == 0 as a SMALL grid-stride kernel (16 bytes per thread and step): it is
// run on the copy stream while the first training uses the SMs, so it must not occupy them -- 64 CTAs keep
// 256 KB of reads in flight, more than the PCIe bandwidth-latency product of the zero-copy path it reads from.
__global__ void __launch_bounds__(256)
gather_rows_f32x4_kernel(const float4* __restrict__ x, const uint64_t* __restrict__ rows, uint64_t s, int d4,
                         float4* __restrict__ out) {
  const uint64_t total = s * (uint64_t)d4, stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += stride)
    out[g] = x[rows[g / d4] * (uint64_t)d4 + g % d4];
}
// values of an f32 buffer rounded to what element type `dt` can hold (f16 / bf16 models: the reference keeps
// centroids and codebooks in the vectors' own type, kmeans.rs:405-418, pq/builder.rs:139-157)
__global__ void round_to_dtype_kernel(float* __restrict__ v, size_t count, int dt) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  if (dt == LB2_F16) v[i] = __half2float(__float2half_rn(v[i]));
  else if (dt == LB2_BF16) v[i] = __bfloat162float(__float2bfloat16_rn(v[i]));
}
void round_model(float* v, size_t count, lb2_dtype dt) {
  if ((dt == LB2_F16 || dt == LB2_BF16) && count)
    LB2_LAUNCH("round_model", round_to_dtype_kernel, cdiv(count, 256), 256, 0, v, count, (int)dt);
}

void normalize_rows(const float* x, uint64_t n, int d, float* out) {
  if (n) LB2_LAUNCH("normalize", normalize_kernel, cdiv(n, 128), 128, 0, x, n, d, out);
}

thread_local std::map<int, StagingCache> g_staging;
void staging_cache_release() {
  auto it = g_staging.find(ctx().device);
  if (it == g_staging.end() || it->second.in_use) return;
  StagingCache& sc = it->second;
  if (sc.copy_stream) { cudaStreamSynchronize(sc.copy_stream); cudaStreamDestroy(sc.copy_stream); }
  if (sc.copied) cudaEventDestroy(sc.copied);
  if (sc.flags_ready) cudaEventDestroy(sc.flags_ready);
  if (sc.flags_host) cudaFreeHost(sc.flags_host);
  if (sc.buf) cudaFreeAsync(sc.buf, ctx().stream);
  g_staging.erase(it);
}

// Training sample of a build: rows `rows` (ascending) of x, minus the rows that are not finite
// (rust/lance/src/index/vector/builder.rs:436 keeps `is_finite` rows only; under cosine a zero vector
// has become NaN by then).  Returns the number of rows kept in `out` ([rows.size()][d]).
uint64_t gather_finite_sample(Source& src, std::vector<uint64_t>& rows, bool normalize, DevBuf<float>& out) {
  const int d = src.d();
  uint64_t s = rows.size();
  out.alloc(std::max<uint64_t>(1, s * d));
  if (s == 0) return 0;
  DevBuf<uint8_t> flag(s);
  std::vector<uint8_t> hf(s);
  for (int pass = 0; pass < 2; ++pass) {
    src.gather_f32(rows, out.p);
    if (normalize)  // cosine: NormalizeTransformer first (ivf.rs:158-166); a zero vector becomes NaN and is dropped
      normalize_rows(out.p, s, d, out.p);
    if (pass == 1) break;
    LB2_LAUNCH("finite_rows", finite_rows_kernel, cdiv(s * 32, 256), 256, 0, out.p, s, d, flag.p, 0);
    d2h(hf.data(), flag.p, s);
    sync_stream();
    uint64_t kept = 0;
    for (uint64_t i = 0; i < s; ++i)
      if (hf[i]) rows[kept++] = rows[i];
    if (kept == s) break;
    rows.resize(kept);  // rare: gather again without the dropped rows (order preserved)
    s = kept;
    if (!s) break;
  }
  sync_stream();
  return s;
}

// s distinct rows out of n, ascending: one uniformly random row from each of s equal strata
// (the reference draws a random subset through Dataset::sample, rust/lance/src/index/vector/utils.rs:
// 202-209, with an unseeded rng -> the selection is unpinned; ours is O(s), seeded, already sorted)
std::vector<uint64_t> sample_rows(uint64_t n, uint64_t s, uint64_t seed) {
  std::vector<uint64_t> out;
  if (s >= n) {
    out.resize(n);
    for (uint64_t i = 0; i < n; ++i) out[i] = i;
    return out;
  }
  SplitMix64 rng(seed);
  out.resize(s);
  // stratum i = [floor(i n / s), floor((i + 1) n / s)): the quotients are carried incrementally (i n = q s + r),
  // not recomputed with two 128-bit divisions per row -- this loop is host time in front of every build
  const uint64_t qn = n / s, rn = n % s;
  uint64_t lo = 0, rem = 0;
  for (uint64_t i = 0; i < s; ++i) {
    uint64_t hi = lo + qn;
    rem += rn;
    if (rem >= s) { rem -= s; ++hi; }
    out[i] = lo + rng.next() % (hi - lo);
    lo = hi;
  }
  return out;
}

}  // namespace lb2
