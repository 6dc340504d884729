// api.cu -- the extern "C" surface declared in include/lance_b200.h, the per-thread runtime
// context, the device-resident index handle and the whole-index builder.
#include <chrono>
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <algorithm>
#include <cmath>
#include <memory>

#include "assign.cuh"
#include "comm.cuh"
#include "common.cuh"
#include "exact.cuh"
#include "kmeans.cuh"
#include "rq.cuh"
#include "search.cuh"
#include "sq.cuh"
#include "tc_assign.cuh"
#include "tc_pq.cuh"

namespace lb2 {

// ------------------------------------------------------------------------------------------------
// runtime context
// ------------------------------------------------------------------------------------------------
static thread_local std::string g_last_error;
static thread_local Ctx* g_ctx = nullptr;
static thread_local int g_requested_device = 0;

void set_last_error(const std::string& m) { g_last_error = m; }

static int usable_devices() {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return n;
}

Ctx& ctx() {
  if (g_ctx && g_ctx->device == g_requested_device) {
    return *g_ctx;
  }
  if (usable_devices() <= 0)
    fail(LB2_NO_DEVICE, "no CUDA device: lance_b200 has no CPU fallback (needs an sm_90a GPU)");
  LB2_CUDA(cudaSetDevice(g_requested_device));
  Ctx* c = new Ctx();  // one per (thread, device); lives for the thread's lifetime
  c->device = g_requested_device;
  LB2_CUDA(cudaStreamCreateWithFlags(&c->own_stream, cudaStreamNonBlocking));
  c->stream = c->own_stream;
  LB2_CUDA(cudaEventCreate(&c->t0));
  LB2_CUDA(cudaEventCreate(&c->t1));
  cudaDeviceProp prop;
  LB2_CUDA(cudaGetDeviceProperties(&prop, c->device));
  c->num_sms = prop.multiProcessorCount;
  c->smem_optin = prop.sharedMemPerBlockOptin;
  // keep freed blocks in the pool: the training loop allocates per iteration
  cudaMemPool_t pool;
  if (cudaDeviceGetDefaultMemPool(&pool, c->device) == cudaSuccess) {
    uint64_t thr = ~0ull;
    cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
  }
  g_ctx = c;
  return *c;
}

void Ctx::flush_profile() {
  if (pending.empty()) return;
  cudaStreamSynchronize(stream);
  for (auto& e : pending) {
    float ms = 0.f;
    cudaEventElapsedTime(&ms, e.second.first, e.second.second);
    auto& pe = prof[e.first];
    pe.launches++;
    pe.total_ms += ms;
    cudaEventDestroy(e.second.first);
    cudaEventDestroy(e.second.second);
  }
  pending.clear();
}

bool is_device_ptr(const void* p) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
}

// ------------------------------------------------------------------------------------------------
// small elementwise kernels
// ------------------------------------------------------------------------------------------------
// x and out may alias (in-place residual of the PQ training sample)
__global__ void residual_kernel(const float* x, const float* __restrict__ cent,
                                const uint32_t* __restrict__ part, uint64_t n, int d, float* out) {
  const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n * d) return;
  const uint64_t r = g / d;
  const int t = g % d;
  out[g] = __fsub_rn(x[g], cent[(size_t)part[r] * d + t]);  // residual.rs:93
}

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

__global__ void gather_rows_kernel(const float* __restrict__ x, const uint64_t* __restrict__ rows,
                                   uint64_t s, int d, float* __restrict__ out) {
  const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= s * d) return;
  out[g] = x[rows[g / d] * d + g % d];
}

__global__ void group_kernel(const uint32_t* __restrict__ members, uint64_t n, int M,
                             const uint8_t* __restrict__ codes, const uint64_t* __restrict__ row_ids,
                             uint8_t* __restrict__ codes_out, uint64_t* __restrict__ row_ids_out) {
  const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n) return;
  const uint32_t src = members[g];
  row_ids_out[g] = row_ids ? row_ids[src] : (uint64_t)src;
  for (int m = 0; m < M; ++m) codes_out[g * M + m] = codes[(size_t)src * M + m];
}

__global__ void group_vectors_kernel(const uint32_t* __restrict__ members, uint64_t n, int d,
                                     const float* __restrict__ vectors, const uint64_t* __restrict__ row_ids,
                                     float* __restrict__ vectors_out, uint64_t* __restrict__ row_ids_out) {
  const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;  // one float4 per thread
  const int d4 = d >> 2;
  if (g >= n * d4) return;
  const uint64_t r = g / d4;
  const int c = g % d4;
  const uint32_t src = members[r];
  reinterpret_cast<float4*>(vectors_out)[g] = reinterpret_cast<const float4*>(vectors)[(uint64_t)src * d4 + c];
  if (c == 0) row_ids_out[r] = row_ids ? row_ids[src] : (uint64_t)src;
}

// row-major codes [n][cw] of one partition -> the reference's storage layout [cw][n] (pq/storage.rs:430-450)
__global__ void transpose_codes_kernel(const uint8_t* __restrict__ codes, uint64_t n, int cw, uint8_t* __restrict__ out) {
  const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n * cw) return;
  const uint64_t j = g % n;
  const int m = (int)(g / n);
  out[g] = codes[j * cw + m];
}

__global__ void widen_offsets_kernel(const uint32_t* __restrict__ off32, int K,
                                     uint64_t* __restrict__ off64) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i <= K) off64[i] = off32[i];
}

// largest partition id of a caller-supplied id column (range check before it indexes device memory)
__global__ void max_u32_kernel(const uint32_t* __restrict__ v, uint64_t n, uint32_t* __restrict__ out) {
  uint32_t m = 0;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
    m = max(m, v[i]);
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m) atomicMax(out, m);
}

// KeepFiniteVectors (lance-index/src/vector/transform.rs:112-159) / the is_finite filter applied to the
// training sample (rust/lance/src/index/vector/builder.rs:436): flag[r] = every element of row r is finite
__global__ void finite_rows_kernel(const float* __restrict__ x, uint64_t n, int d, uint8_t* __restrict__ flag) {
  const uint64_t w = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= n) return;
  bool ok = true;
  for (int e = lane; e < d; e += 32) ok &= isfinite(x[w * d + e]);
  ok = __all_sync(0xffffffffu, ok);
  if (lane == 0) flag[w] = ok ? 1 : 0;
}

// valid[w] = 0 for a row with a non-finite element (KeepFiniteVectors, transform.rs:86-150); warp per row
__global__ void drop_nonfinite_rows_kernel(const float* __restrict__ x, uint64_t n, int d, uint8_t* __restrict__ valid) {
  const uint64_t w = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= n) return;
  bool ok = true;
  for (int e = lane; e < d; e += 32) ok &= isfinite(x[w * d + e]);
  ok = __all_sync(0xffffffffu, ok);
  if (lane == 0 && !ok) valid[w] = 0;
}

// l2_distance_uint_scalar (lance-linalg/src/distance/l2.rs:44-49, impl L2 for u8 :93-98): sum of |x - y|^2 in
// u32 (wrapping, like Rust's release-mode `sum::<u32>()`), then `as f32` (round to nearest even); warp per row
__global__ void l2_u8_kernel(const uint8_t* __restrict__ from, const uint8_t* __restrict__ to, uint64_t n, int d,
                             float* __restrict__ out) {
  const uint64_t w = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= n) return;
  uint32_t s = 0;
  for (int e = lane; e < d; e += 32) {
    const int df = (int)from[e] - (int)to[w * d + e];
    s += (uint32_t)(df * df);
  }
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) out[w] = __uint2float_rn(s);
}
// cosine_distance_batch (cosine.rs:143-174,266-290): 1 - xy / |x| / sqrt(yy) with f32 FMA lanes; the
// reference's own lane order is ISA specific, so parity is the reference's tolerance (cosine.rs:361-393)
__global__ void cosine_f32_kernel(const float* __restrict__ from, const float* __restrict__ to, uint64_t n, int d,
                                  float* __restrict__ out) {
  const uint64_t w = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= n) return;
  float xx = 0.0f, xy = 0.0f, yy = 0.0f;
  for (int e = lane; e < d; e += 32) {
    const float x = from[e], y = to[w * d + e];
    xx = fmaf(x, x, xx);
    xy = fmaf(x, y, xy);
    yy = fmaf(y, y, yy);
  }
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) {
    xx += __shfl_xor_sync(0xffffffffu, xx, o);
    xy += __shfl_xor_sync(0xffffffffu, xy, o);
    yy += __shfl_xor_sync(0xffffffffu, yy, o);
  }
  if (lane == 0) out[w] = 1.0f - xy / sqrtf(xx) / sqrtf(yy);
}

// ---- element types ---------------------------------------------------------------------------------
// f16 / bf16 / u8 buffers are converted to f32 on the device at the boundary and every loop runs
// with the reference's f32 semantics (what the reference itself does for Int8 vectors,
// rust/lance/src/index/vector/ivf.rs:1917-1929; its f16 paths accumulate in f16 / use a -ffast-math
// C kernel, so for f16 inputs parity with the reference is by tolerance, see DESIGN.md).
// Model outputs (centroids, codebook, residuals, normalised vectors) use the input's element type,
// except for u8 inputs, whose model is f32.
static size_t dtype_size(lb2_dtype dt) { return dt == LB2_F32 ? 4 : (dt == LB2_U8 ? 1 : 2); }
static lb2_dtype model_dtype(lb2_dtype dt) { return dt == LB2_U8 ? LB2_F32 : dt; }

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

// typed input: device f32 view of a (host or device) buffer of `dt` elements
struct VecIn {
  InArg<float> f32;
  InArg<uint8_t> raw;
  DevBuf<float> conv;
  const float* p = nullptr;
  VecIn() = default;
  VecIn(const void* ptr, size_t count, lb2_dtype dt) { set(ptr, count, dt); }
  void set(const void* ptr, size_t count, lb2_dtype dt) {
    if (!ptr || !count) { p = nullptr; return; }
    if (dt == LB2_F32) { f32.set(ptr, count); p = f32.get(); return; }
    raw.set(ptr, count * dtype_size(dt));
    conv.alloc(count);
    LB2_LAUNCH("convert_to_f32", to_f32_kernel, cdiv(count, 256), 256, 0, raw.get(), (int)dt, count, conv.p);
    p = conv.p;
  }
  const float* get() const { return p; }
};
// typed output: kernels write f32; commit() converts to `dt` and copies to the caller's buffer
struct VecOut {
  OutArg<float> f32;
  OutArg<uint8_t> raw;
  DevBuf<float> tmp;
  lb2_dtype dt = LB2_F32;
  size_t count = 0;
  float* p = nullptr;
  VecOut(void* ptr, size_t cnt, lb2_dtype d) : dt(d), count(cnt) {
    if (!ptr || !cnt) return;
    if (dt == LB2_F32) { f32.set(ptr, cnt); p = f32.get(); return; }
    raw.set(ptr, cnt * dtype_size(dt));
    tmp.alloc(cnt);
    p = tmp.p;
  }
  float* get() const { return p; }
  void commit() {
    if (!p) return;
    if (dt == LB2_F32) { f32.commit(); return; }
    LB2_LAUNCH("convert_from_f32", from_f32_kernel, cdiv(count, 256), 256, 0, tmp.p, (int)dt, count, raw.get());
    raw.commit();
  }
};

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
static void round_model(float* v, size_t count, lb2_dtype dt) {
  if ((dt == LB2_F16 || dt == LB2_BF16) && count)
    LB2_LAUNCH("round_model", round_to_dtype_kernel, cdiv(count, 256), 256, 0, v, count, (int)dt);
}

// ---- a caller's n x d matrix, in its own element type, wherever it lives ----------------------------------
// The kernels never see an f32 copy of the WHOLE matrix.  Device-resident rows are used where they are;
// host rows are either copied once, in their native type, on a second stream while training runs (when they
// fit the budget), or streamed chunk by chunk through two staging slots during the per-row pass.  f32 views
// exist for one chunk of rows at a time (zero-copy when the rows already are f32 on the device).
// What a host-sourced build needs every time, kept per (thread, device) between calls: the copy stream, its
// event and the device-side landing buffer of the bulk copy.  Re-creating them per build -- above all a fresh
// 512 MB cudaMallocAsync, which the pool serves by mapping new physical memory whenever its free blocks are
// fragmented -- costs host time at random before the copy can even start (tools/e2e_trace.py shows it); with
// the cache the copy is issued right after the sample gathers.  Only buffers <= LB2_STAGING_CACHE_MB (default 1024) are retained;
// lb2_trim_memory() gives everything back.
struct StagingCache {
  cudaStream_t copy_stream = nullptr;
  cudaEvent_t copied = nullptr;
  void* buf = nullptr;
  size_t bytes = 0;
  uint8_t* flags_host = nullptr;  // pinned: the finite-row flags of a sample gathered on the copy stream
  size_t flags_cap = 0;
  cudaEvent_t flags_ready = nullptr;
  bool in_use = false;
};
static thread_local std::map<int, StagingCache> g_staging;
static size_t staging_cache_cap() {
  static const size_t cap = [] {
    const char* e = getenv("LB2_STAGING_CACHE_MB");
    return (size_t)(e && *e ? strtoull(e, nullptr, 10) : 1024ull) << 20;
  }();
  return cap;
}
static void staging_cache_release() {  // the calling thread's cache on the current device
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

class Source {
 public:
  Source(const void* p, uint64_t n, int d, lb2_dtype dt) : host_(p), n_(n), d_(d), dt_(dt), es_(dtype_size(dt)) {
    cudaPointerAttributes pa;
    const bool ok = cudaPointerGetAttributes(&pa, p) == cudaSuccess;
    if (!ok) cudaGetLastError();
    if (ok && (pa.type == cudaMemoryTypeDevice || pa.type == cudaMemoryTypeManaged)) {
      dev_native_ = p;
    } else if (ok && pa.type == cudaMemoryTypeHost && pa.devicePointer) {
      static const bool no_zc = getenv("LB2_NO_ZERO_COPY") && *getenv("LB2_NO_ZERO_COPY");  // diagnostics
      if (!no_zc) zero_copy_ = pa.devicePointer;  // pinned: the device can read it over PCIe
    }
  }
  ~Source() {
    if (cache_) {  // stream, event and (maybe) the buffer go back to the thread's cache
      cudaStreamSynchronize(copy_stream_);
      cudaEventRecord(copied_, ctx().stream);  // the buffer's last reader: the next bulk copy waits for it
      cache_->in_use = false;
      copy_stream_ = nullptr;
      copied_ = nullptr;
    }
    if (copy_stream_) { cudaStreamSynchronize(copy_stream_); cudaStreamDestroy(copy_stream_); }
    if (copied_) cudaEventDestroy(copied_);
    for (auto& e : slot_ready_) if (e) cudaEventDestroy(e);
    for (auto& e : slot_free_) if (e) cudaEventDestroy(e);
  }
  Source(const Source&) = delete;
  uint64_t rows_per_chunk() const {  // <= 1 GB of f32 per chunk, 64 Ki .. 1 Mi rows
    // LB2_CHUNK_ROWS=r replaces the rule (no floor): small inputs then take the multi-chunk paths.  Read on
    // every call, so that a test can set it for one call.
    const char* e = getenv("LB2_CHUNK_ROWS");
    const uint64_t r = e && *e ? strtoull(e, nullptr, 10) : 0;
    if (r >= 1) return r;
    return std::max<uint64_t>(1ull << 16, std::min<uint64_t>(1ull << 20, (1ull << 28) / (uint64_t)d_));
  }
  // training sample: rows `rows` (ascending) as f32 [rows.size()][d] -- straight out of the caller's memory
  void gather_f32(const std::vector<uint64_t>& rows, float* out) {
    const uint64_t s = rows.size();
    if (!s) return;
    // (once a bulk copy has been started the rows are read from it: zero-copy reads starve behind the copy engine)
    const void* src = dev_native_ ? dev_native_ : (bulk_p_ ? native_device() : zero_copy_);
    if (src) {
      DevBuf<uint64_t> rows_d(s);
      h2d(rows_d.p, rows.data(), s);
      LB2_LAUNCH("gather_rows", gather_rows_typed_kernel, cdiv(s * d_, 256), 256, 0, src, (int)dt_, rows_d.p, s, d_, out);
      sync_stream();
      return;
    }
    // pageable host memory: pack the rows on the host, one copy, convert on the device
    std::vector<uint8_t> pack((size_t)s * d_ * es_);
    for (uint64_t i = 0; i < s; ++i)
      memcpy(pack.data() + (size_t)i * d_ * es_, static_cast<const uint8_t*>(host_) + (size_t)rows[i] * d_ * es_, (size_t)d_ * es_);
    if (dt_ == LB2_F32) {
      LB2_CUDA(cudaMemcpyAsync(out, pack.data(), pack.size(), cudaMemcpyHostToDevice, ctx().stream));
    } else {
      DevBuf<uint8_t> raw(pack.size());
      LB2_CUDA(cudaMemcpyAsync(raw.p, pack.data(), pack.size(), cudaMemcpyHostToDevice, ctx().stream));
      LB2_LAUNCH("convert_to_f32", to_f32_kernel, cdiv((size_t)s * d_, 256), 256, 0, raw.p, (int)dt_, (size_t)s * d_, out);
    }
    sync_stream();
  }
  // A second training sample gathered on the COPY stream, in front of the bulk copy, while the first training
  // already runs on the library's stream (pinned f32 rows only).  Enqueues: rows -> device, the bounded-grid
  // gather into `out`, the finite-row flags, their copy into pinned host memory, an event.  Returns false when
  // the preconditions do not hold (the caller then gathers synchronously).  finish_async_sample() tells whether
  // every row was finite.
  bool gather_f32_async(const std::vector<uint64_t>& rows, float* out) {
    const uint64_t s = rows.size();
    if (!zero_copy_ || dt_ != LB2_F32 || d_ % 4 != 0 || s == 0 || ctx().profiling) return false;
    if ((reinterpret_cast<uintptr_t>(zero_copy_) & 15) != 0) return false;
    if (!acquire_cache()) return false;
    StagingCache& sc = *cache_;
    if (sc.flags_cap < s) {
      if (sc.flags_host) cudaFreeHost(sc.flags_host);
      sc.flags_host = nullptr;
      sc.flags_cap = 0;
      LB2_CUDA(cudaMallocHost(reinterpret_cast<void**>(&sc.flags_host), s));
      sc.flags_cap = s;
    }
    if (!sc.flags_ready) LB2_CUDA(cudaEventCreateWithFlags(&sc.flags_ready, cudaEventDisableTiming));
    async_rows_.alloc(s);   // (allocated on the library's stream, used on the copy stream behind the event below)
    async_flag_.alloc(s);
    cudaStream_t cs = copy_stream_;
    LB2_CUDA(cudaEventRecord(copied_, ctx().stream));
    LB2_CUDA(cudaStreamWaitEvent(cs, copied_, 0));
    LB2_CUDA(cudaMemcpyAsync(async_rows_.p, rows.data(), s * sizeof(uint64_t), cudaMemcpyHostToDevice, cs));
    ctx().launches += 2;
    gather_rows_f32x4_kernel<<<64, 256, 0, cs>>>(static_cast<const float4*>(zero_copy_), async_rows_.p, s, d_ / 4,
                                                 reinterpret_cast<float4*>(out));
    finite_rows_kernel<<<(unsigned)cdiv(s * 32, 256), 256, 0, cs>>>(out, s, d_, async_flag_.p);
    LB2_CUDA(cudaGetLastError());
    LB2_CUDA(cudaMemcpyAsync(sc.flags_host, async_flag_.p, s, cudaMemcpyDeviceToHost, cs));
    LB2_CUDA(cudaEventRecord(sc.flags_ready, cs));
    async_s_ = s;
    return true;
  }
  // after gather_f32_async(): waits for the gather, orders the library's stream behind it; true = all rows finite
  bool finish_async_sample() {
    StagingCache& sc = *cache_;
    LB2_CUDA(cudaEventSynchronize(sc.flags_ready));
    LB2_CUDA(cudaStreamWaitEvent(ctx().stream, sc.flags_ready, 0));
    bool all = true;
    for (uint64_t i = 0; i < async_s_; ++i) all &= sc.flags_host[i] != 0;
    async_rows_.release();
    async_flag_.release();
    return all;
  }
  // Host rows that fit: one bulk copy in the NATIVE type on a second stream (call after the sample gathers --
  // zero-copy reads get no PCIe bandwidth while the copy engine streams).  Otherwise chunks are staged on demand.
  void start_resident_copy() {
    if (dev_native_ || n_ == 0) return;
    const size_t bytes = (size_t)n_ * d_ * es_;
    acquire_cache();  // (a second Source alive on the same thread falls back to private resources)
    // LB2_MAX_RESIDENT_MB=m: a matrix of more than m MB is streamed (0 = always); read on every call, and
    // ahead of the warm-cache shortcut below, which would otherwise skip every size test
    const char* cap_e = getenv("LB2_MAX_RESIDENT_MB");
    if (cap_e && *cap_e && bytes > ((size_t)strtoull(cap_e, nullptr, 10) << 20)) return;
    StagingCache& sc = g_staging[ctx().device];
    const bool cached_buf = cache_ && bytes <= staging_cache_cap();
    if (!(cached_buf && sc.bytes >= bytes)) {
      size_t free_b = 0, total_b = 0;
      cudaMemGetInfo(&free_b, &total_b);
      if (bytes > (free_b + (cached_buf ? sc.bytes : 0)) / 2) return;  // streamed (issue_copy uses the stream too)
      if (cached_buf) {
        if (sc.buf) cudaFreeAsync(sc.buf, ctx().stream);
        sc.buf = nullptr;
        sc.bytes = 0;
        LB2_CUDA(cudaMallocAsync(&sc.buf, bytes, ctx().stream));
        sc.bytes = bytes;
      } else {
        bulk_.alloc(bytes);
      }
    }
    bulk_p_ = cached_buf ? static_cast<uint8_t*>(sc.buf) : bulk_.p;
    if (!cache_) {
      if (!copy_stream_) LB2_CUDA(cudaStreamCreateWithFlags(&copy_stream_, cudaStreamNonBlocking));
      if (!copied_) LB2_CUDA(cudaEventCreateWithFlags(&copied_, cudaEventDisableTiming));
    }
    // after the cached buffer's last reader (acquire_cache), the allocation and the gathers
    LB2_CUDA(cudaEventRecord(copied_, ctx().stream));
    LB2_CUDA(cudaStreamWaitEvent(copy_stream_, copied_, 0));
    LB2_CUDA(cudaMemcpyAsync(bulk_p_, host_, bytes, cudaMemcpyHostToDevice, copy_stream_));
    LB2_CUDA(cudaEventRecord(copied_, copy_stream_));
    bulk_pending_ = true;
  }
  // device pointer to ALL rows in their native type, or nullptr when the matrix is streamed
  const void* native_device() {
    if (dev_native_) return dev_native_;
    if (bulk_p_) {
      if (bulk_pending_) { LB2_CUDA(cudaStreamWaitEvent(ctx().stream, copied_, 0)); bulk_pending_ = false; }
      return bulk_p_;
    }
    return nullptr;
  }
  // f32 view of rows [r0, r0 + rows) on the library's stream; valid until the second-next call (two slots)
  const float* rows_f32(uint64_t r0, uint64_t rows) {
    const void* nat = native_device();
    const size_t off = (size_t)r0 * d_ * es_, cnt = (size_t)rows * d_;
    last_native_ = nat ? static_cast<const uint8_t*>(nat) + off : nullptr;
    if (nat && dt_ == LB2_F32) return reinterpret_cast<const float*>(static_cast<const uint8_t*>(nat) + off);
    const int slot = (int)(calls_++ & 1);
    if (!nat && dt_ != LB2_F32) last_native_ = nullptr;  // set below once the slot is known
    if (nat) {
      if (f32_[slot].n < cnt) f32_[slot].alloc(cnt);
      LB2_LAUNCH("convert_to_f32", to_f32_kernel, cdiv(cnt, 256), 256, 0, static_cast<const uint8_t*>(nat) + off,
                 (int)dt_, cnt, f32_[slot].p);
      return f32_[slot].p;
    }
    // streamed from the host: the copy runs on the copy stream (issued by prefetch() while the previous chunk's
    // kernels execute, or here), the conversion on the library's stream
    if (!(staged_[slot] && staged_r0_[slot] == r0)) issue_copy(slot, r0, rows);
    staged_[slot] = false;
    LB2_CUDA(cudaStreamWaitEvent(ctx().stream, slot_ready_[slot], 0));
    if (dt_ != LB2_F32) {
      LB2_LAUNCH("convert_to_f32", to_f32_kernel, cdiv(cnt, 256), 256, 0, raw_[slot].p, (int)dt_, cnt, f32_[slot].p);
      last_native_ = raw_[slot].p;
    }
    return f32_[slot].p;
  }
  // where the rows of the last rows_f32() view lie on the device in their own element type (nullptr: f32 itself)
  const void* last_native() const { return last_native_; }
  // start the host-to-device copy of the NEXT chunk; call right after rows_f32() of the current chunk and
  // BEFORE launching the current chunk's kernels (the slot being refilled was last read by the chunk before it)
  void prefetch(uint64_t r0, uint64_t rows) {
    if (rows == 0 || native_device() != nullptr) return;
    issue_copy((int)(calls_ & 1), r0, rows);
  }

  bool has_bulk() const { return bulk_p_ != nullptr; }

 private:
  // take the thread's cached copy stream / event (and with them the right to the cached landing buffer); the copy
  // stream is first ordered behind the buffer's last reader, recorded by the previous holder's destructor
  bool acquire_cache() {
    if (cache_) return true;
    if (copy_stream_) return false;  // already on private resources
    StagingCache& sc = g_staging[ctx().device];
    if (sc.in_use) return false;
    if (!sc.copy_stream) LB2_CUDA(cudaStreamCreateWithFlags(&sc.copy_stream, cudaStreamNonBlocking));
    if (!sc.copied) LB2_CUDA(cudaEventCreateWithFlags(&sc.copied, cudaEventDisableTiming));
    sc.in_use = true;
    cache_ = &sc;
    copy_stream_ = sc.copy_stream;
    copied_ = sc.copied;
    LB2_CUDA(cudaStreamWaitEvent(copy_stream_, copied_, 0));
    return true;
  }
  void issue_copy(int slot, uint64_t r0, uint64_t rows) {
    const size_t off = (size_t)r0 * d_ * es_, cnt = (size_t)rows * d_;
    if (!copy_stream_) LB2_CUDA(cudaStreamCreateWithFlags(&copy_stream_, cudaStreamNonBlocking));
    if (!slot_ready_[slot]) {
      LB2_CUDA(cudaEventCreateWithFlags(&slot_ready_[slot], cudaEventDisableTiming));
      LB2_CUDA(cudaEventCreateWithFlags(&slot_free_[slot], cudaEventDisableTiming));
    }
    if (f32_[slot].n < cnt) f32_[slot].alloc(cnt);
    uint8_t* dst = reinterpret_cast<uint8_t*>(f32_[slot].p);
    if (dt_ != LB2_F32) {
      if (raw_[slot].n < cnt * es_) raw_[slot].alloc(cnt * es_);
      dst = raw_[slot].p;
    }
    LB2_CUDA(cudaEventRecord(slot_free_[slot], ctx().stream));  // everything issued so far is done with the slot
    LB2_CUDA(cudaStreamWaitEvent(copy_stream_, slot_free_[slot], 0));
    // profiling: one "stage_rows" entry per staged chunk (timed on the copy stream; not a kernel launch)
    Ctx& c = ctx();
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    if (c.profiling) {
      LB2_CUDA(cudaEventCreate(&e0));
      LB2_CUDA(cudaEventCreate(&e1));
      LB2_CUDA(cudaEventRecord(e0, copy_stream_));
    }
    LB2_CUDA(cudaMemcpyAsync(dst, static_cast<const uint8_t*>(host_) + off, cnt * es_, cudaMemcpyHostToDevice, copy_stream_));
    if (e0) {
      LB2_CUDA(cudaEventRecord(e1, copy_stream_));
      c.pending.push_back({c.tag.empty() ? std::string("stage_rows") : c.tag + ":stage_rows", {e0, e1}});
    }
    LB2_CUDA(cudaEventRecord(slot_ready_[slot], copy_stream_));
    staged_[slot] = true;
    staged_r0_[slot] = r0;
  }

 public:
  uint64_t n() const { return n_; }
  int d() const { return d_; }
  lb2_dtype dtype() const { return dt_; }
  size_t row_bytes() const { return (size_t)d_ * es_; }

 private:
  bool staged_[2] = {false, false};
  uint64_t staged_r0_[2] = {0, 0};
  const void* last_native_ = nullptr;
  const void* host_;
  uint64_t n_;
  int d_;
  lb2_dtype dt_;
  size_t es_;
  const void* dev_native_ = nullptr;
  const void* zero_copy_ = nullptr;
  DevBuf<uint8_t> bulk_, raw_[2];
  DevBuf<uint64_t> async_rows_;     // gather_f32_async: the row list and the finite flags on the device
  DevBuf<uint8_t> async_flag_;
  uint64_t async_s_ = 0;
  uint8_t* bulk_p_ = nullptr;       // landing buffer of the bulk copy: bulk_ (private) or the thread's cached one
  StagingCache* cache_ = nullptr;   // non-null while this Source holds the thread's cached stream / event / buffer
  DevBuf<float> f32_[2];
  cudaStream_t copy_stream_ = nullptr;
  cudaEvent_t copied_ = nullptr, slot_ready_[2] = {nullptr, nullptr}, slot_free_[2] = {nullptr, nullptr};
  bool bulk_pending_ = false;
  uint64_t calls_ = 0;
};

static void require_f32(lb2_dtype dt, const char* what) {
  if (dt != LB2_F32)
    fail(LB2_UNSUPPORTED, "%s: element type %d is not implemented on the device yet (f32 only)", what,
         (int)dt);
}
static int metric_of(lb2_metric m) {
  switch (m) {
    case LB2_L2: return METRIC_L2;
    case LB2_COSINE: return METRIC_COSINE;
    case LB2_DOT: return METRIC_DOT;
  }
  fail(LB2_INVALID_ARG, "unknown metric %d", (int)m);
}

}  // namespace lb2

using namespace lb2;

// the handle
struct lb2_index {
  int kind = 0;  // 0 = IVF_PQ, 1 = IVF_FLAT, 2 = IVF_SQ, 3 = IVF_RQ
  lb2_dtype dtype = LB2_F32;  // element type of the vectors / queries the caller passes
  // IVF_FLAT: the (normalised for cosine) vectors in partition order, in the vectors' own element type
  // (f32 / f16 / bf16; u8 columns are held as f32, the reference's model type for them, ivf.rs:1917-1929)
  DevBuf<uint8_t> vectors;
  lb2_dtype vdtype() const { return dtype == LB2_U8 ? LB2_F32 : dtype; }
  size_t vrow_bytes() const { return (size_t)d * (vdtype() == LB2_F32 ? 4 : 2); }
  int K = 0, d = 0, M = 0, nbits = 8, metric = 0;
  uint64_t n = 0;
  DevBuf<float> centroids, codebook;
  DevBuf<uint64_t> part_offsets, row_ids;
  DevBuf<uint8_t> codes;
  // the conflict-free scan's skewed copy of `codes` (search.cu: ivfpq_scan_skew_kernel); empty for other shapes
  DevBuf<uint64_t> slab_off;
  DevBuf<uint8_t> codes_skew;
  // IVF_SQ: `codes` are the 8-bit scalar codes [n][d] of the (normalised for cosine) vectors, under the bounds
  // [sq_lower, sq_upper] (sq/storage.rs:38-45)
  double sq_lower = 0.0, sq_upper = 0.0;
  // IVF_RQ: `codes` are the sign codes [n][code_dim / 8] of the rotated residuals (num_bits = nbits, code_dim =
  // d * nbits), with the per-row factors rq_add / rq_scale [n] and the rotation rq_rot [code_dim][code_dim]
  // (bq/storage.rs:110-121)
  DevBuf<float> rq_rot, rq_add, rq_scale;
  int code_dim() const { return d * nbits; }
  // bytes per row of `codes` (PQ: pq.rs:168-173; SQ: one per dimension; RQ: one bit per code dimension)
  int code_bytes() const { return kind == 3 ? code_dim() / 8 : kind == 2 ? d : (nbits == 4 ? M / 2 : M); }
  size_t codebook_len() const { return ((size_t)1 << nbits) * d; }
};

namespace lb2 {

// a partition id >= K (a corrupted / mismatched shuffle file) would index device memory out of bounds
static void check_part_ids(const uint32_t* part_ids, uint64_t n, uint32_t K, const char* what) {
  if (n == 0) return;
  DevBuf<uint32_t> mx(1);
  mx.zero();
  LB2_LAUNCH("check_part_ids", max_u32_kernel, (unsigned)std::min<uint64_t>(cdiv(n, 1024), 1024), 256, 0, part_ids, n, mx.p);
  uint32_t h = 0;
  d2h(&h, mx.p, 1);
  sync_stream();
  if (h >= K) fail(LB2_INVALID_ARG, "%s: partition id %u out of range (the index has %u partitions)", what, h, K);
}

// stable grouping of the kept rows by partition; rows with valid[r] == 0 (KeepFiniteVectors,
// transform.rs:112-159: NaN / Inf rows, zero vectors under cosine) never enter the index
static uint64_t member_sort_index(MemberSort& ms, lb2_index* ix, const uint32_t* part_ids, const uint8_t* valid,
                                  uint64_t n) {
  LB2_REQUIRE(n < 0xffffffffull, "more than 2^32-1 rows per index shard");
  ms.run(part_ids, valid, n, ix->K, 1, nullptr);
  ix->part_offsets.alloc(ix->K + 1);
  if (n == 0) {
    ix->part_offsets.zero();
    return 0;
  }
  LB2_LAUNCH("widen_offsets", widen_offsets_kernel, cdiv(ix->K + 1, 256), 256, 0, ms.offsets.p,
             ix->K, ix->part_offsets.p);
  uint32_t kept = 0;
  d2h(&kept, ms.offsets.p + ix->K, 1);
  sync_stream();
  return kept;
}

__global__ void gather_f32_kernel(const uint32_t* __restrict__ members, uint64_t n, const float* __restrict__ src,
                                  float* __restrict__ dst) {
  const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g < n) dst[g] = src[members[g]];
}

// rq_add / rq_scale (IVF_RQ only): the rows' factors, grouped with their codes
static void index_load_dev(lb2_index* ix, const uint32_t* part_ids, const uint8_t* codes,
                           const uint64_t* row_ids, uint64_t n, const uint8_t* valid = nullptr,
                           const float* rq_add = nullptr, const float* rq_scale = nullptr) {
  MemberSort ms;
  const uint64_t kept = member_sort_index(ms, ix, part_ids, valid, n);
  ix->codes.alloc(std::max<uint64_t>(1, kept * ix->code_bytes()));
  ix->row_ids.alloc(std::max<uint64_t>(1, kept));
  if (kept)
    LB2_LAUNCH("group_by_partition", group_kernel, cdiv(kept, 256), 256, 0, ms.members.p, kept, ix->code_bytes(),
               codes, row_ids, ix->codes.p, ix->row_ids.p);
  if (ix->kind == 3) {
    ix->rq_add.alloc(std::max<uint64_t>(1, kept));
    ix->rq_scale.alloc(std::max<uint64_t>(1, kept));
    if (kept) {
      LB2_LAUNCH("group_by_partition", gather_f32_kernel, cdiv(kept, 256), 256, 0, ms.members.p, kept, rq_add, ix->rq_add.p);
      LB2_LAUNCH("group_by_partition", gather_f32_kernel, cdiv(kept, 256), 256, 0, ms.members.p, kept, rq_scale,
                 ix->rq_scale.p);
    }
  }
  ix->n = kept;
  if (kept && skew_layout_applies(ix->M, ix->d, ix->nbits)) {
    ix->slab_off.alloc(ix->K + 1);
    ix->codes_skew.alloc(skew_bytes_bound(kept, ix->K));
    build_skew_codes(ix->part_offsets.p, ix->K, ix->codes.p, kept, ix->slab_off.p, ix->codes_skew.p);
  } else {
    ix->slab_off.release();
    ix->codes_skew.release();
  }
  sync_stream();
}

__global__ void copy_row_ids_kernel(const uint32_t* __restrict__ members, uint64_t n, const uint64_t* __restrict__ row_ids,
                                    uint64_t* __restrict__ out) {
  const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g < n) out[g] = row_ids ? row_ids[members[g]] : (uint64_t)members[g];
}
__global__ void members_to_u64_kernel(const uint32_t* __restrict__ members, uint64_t n, uint64_t* __restrict__ out) {
  const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g < n) out[g] = members[g];
}

// IVF_FLAT storage: the kept rows grouped by partition (stable), normalised when the metric is cosine
// (IvfTransformer::new_flat, lance-index/src/vector/ivf.rs:149-185), written in the index's element type.
// Rows are pulled from the caller's matrix in chunks of output positions (never a whole-matrix f32 copy).
// rows `members[i]` of a matrix in its own element type -> consecutive rows (16 bytes per thread)
__global__ void gather_rows_native_kernel(const uint4* __restrict__ src, uint32_t vec_per_row,
                                          const uint32_t* __restrict__ members, uint64_t kept, uint4* __restrict__ dst) {
  const uint64_t total = kept * vec_per_row;
  for (uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t i = g / vec_per_row;
    const uint32_t v = (uint32_t)(g % vec_per_row);
    dst[g] = src[(uint64_t)members[i] * vec_per_row + v];
  }
}

static void index_load_flat_src(lb2_index* ix, const uint32_t* part_ids, Source& src, const uint64_t* row_ids,
                                const uint8_t* valid, bool normalize) {
  const uint64_t n = src.n();
  MemberSort ms;
  const uint64_t kept = member_sort_index(ms, ix, part_ids, valid, n);
  const lb2_dtype vdt = ix->vdtype();
  ix->vectors.alloc(std::max<size_t>(1, kept * ix->vrow_bytes()));
  ix->row_ids.alloc(std::max<uint64_t>(1, kept));
  ix->n = kept;
  if (!kept) { sync_stream(); return; }
  LB2_LAUNCH("group_row_ids", copy_row_ids_kernel, cdiv(kept, 256), 256, 0, ms.members.p, kept, row_ids, ix->row_ids.p);
  const void* nat = src.native_device();
  if (!nat) fail(LB2_OOM, "IVF_FLAT keeps a copy of the vectors: the %llu x %d matrix must fit in device memory",
                 (unsigned long long)n, ix->d);
  const int d = ix->d;
  if (!normalize && vdt == src.dtype() && ix->vrow_bytes() % 16 == 0 && (reinterpret_cast<uintptr_t>(nat) & 15) == 0) {
    // stored type == column type: one pass, no f32 round trip (a C4 shard: 2 x 19 GB of bf16 at HBM speed)
    const uint32_t vpr = (uint32_t)(ix->vrow_bytes() / 16);
    LB2_LAUNCH("group_vectors", gather_rows_native_kernel, (unsigned)std::min<uint64_t>(cdiv(kept * vpr, 256), 64ull * ctx().num_sms),
               256, 0, static_cast<const uint4*>(nat), vpr, ms.members.p, kept, reinterpret_cast<uint4*>(ix->vectors.p));
    sync_stream();
    return;
  }
  const uint64_t chunk = src.rows_per_chunk();
  DevBuf<uint64_t> rows64(std::min(chunk, kept));
  DevBuf<float> tmp, tmp2;
  const bool direct = vdt == LB2_F32 && !normalize;
  if (!direct) tmp.alloc(std::min(chunk, kept) * d);
  if (normalize && vdt == LB2_F32) {
  } else if (normalize) {
    tmp2.alloc(std::min(chunk, kept) * d);
  }
  for (uint64_t p0 = 0; p0 < kept; p0 += chunk) {
    const uint64_t rows = std::min(chunk, kept - p0);
    LB2_LAUNCH("group_vectors", members_to_u64_kernel, cdiv(rows, 256), 256, 0, ms.members.p + p0, rows, rows64.p);
    uint8_t* dst = ix->vectors.p + p0 * ix->vrow_bytes();
    float* g = direct ? reinterpret_cast<float*>(dst) : tmp.p;
    LB2_LAUNCH("group_vectors", gather_rows_typed_kernel, cdiv(rows * d, 256), 256, 0, nat, (int)src.dtype(), rows64.p, rows, d, g);
    if (normalize) {
      float* o = vdt == LB2_F32 ? reinterpret_cast<float*>(dst) : tmp2.p;
      LB2_LAUNCH("normalize", normalize_kernel, cdiv(rows, 128), 128, 0, g, rows, d, o);
      g = o;
    }
    if (vdt != LB2_F32)
      LB2_LAUNCH("convert_from_f32", from_f32_kernel, cdiv(rows * d, 256), 256, 0, g, (int)vdt, (size_t)rows * d, (void*)dst);
  }
  sync_stream();
}

// Training sample of a build: rows `rows` (ascending) of x, minus the rows that are not finite
// (rust/lance/src/index/vector/builder.rs:436 keeps `is_finite` rows only; under cosine a zero vector
// has become NaN by then).  Returns the number of rows kept in `out` ([rows.size()][d]).
static uint64_t gather_finite_sample(Source& src, std::vector<uint64_t>& rows, bool normalize, DevBuf<float>& out) {
  const int d = src.d();
  uint64_t s = rows.size();
  out.alloc(std::max<uint64_t>(1, s * d));
  if (s == 0) return 0;
  DevBuf<uint8_t> flag(s);
  std::vector<uint8_t> hf(s);
  for (int pass = 0; pass < 2; ++pass) {
    src.gather_f32(rows, out.p);
    if (normalize)  // cosine: NormalizeTransformer first (ivf.rs:158-166); a zero vector becomes NaN and is dropped
      LB2_LAUNCH("normalize", normalize_kernel, cdiv(s, 128), 128, 0, out.p, s, d, out.p);
    if (pass == 1) break;
    LB2_LAUNCH("finite_rows", finite_rows_kernel, cdiv(s * 32, 256), 256, 0, out.p, s, d, flag.p);
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

// ProductQuantizer::transform_impl for either code width (pq.rs:116-191): 8-bit -> [n][M] through the
// tensor path where it applies; 4-bit -> 16 codewords per sub-space, exact kernel, two codes per byte
static void pq_encode_any(const float* x, uint64_t n, int d, int M, int ds, const float* codebook, int metric,
                          const float* cent, const uint32_t* part, const uint8_t* row_valid, int nbits,
                          uint8_t* codes) {
  if (nbits == 8) {
    pq_encode_dev(x, n, d, M, ds, codebook, metric, cent, part, row_valid, codes);
    return;
  }
  if (n == 0) return;
  DevBuf<uint8_t> wide((size_t)n * M);
  small_d_assign_f32(x, n, d, M, ds, codebook, 16, metric, cent, part, row_valid, wide.p, nullptr, nullptr,
                     nullptr, nullptr);
  pack_nibbles(wide.p, n, M, codes);
  sync_stream();  // `wide` is freed on return
}

// KMeansParams::redos (kmeans.rs:643-716).  Every redo starts from `rng.clone()` of the same generator
// (kmeans.rs:645-653), i.e. from the SAME initial centroids; the only state carried from one redo to the
// next is cluster_sizes / adjusted_balance_factor, which only enter through the balance bias.  With
// balance_factor == 0 (every PQ codebook, pq/builder.rs:100) all redos are therefore identical and
// "best of redos" is the single run; with a balance bias the redo loop is not implemented -> UNSUPPORTED.
static void check_redos(uint32_t redos, float balance_factor) {
  if (redos == 0) fail(LB2_INVALID_ARG, "KMeans: redos must be at least 1");
  if (redos > 1 && balance_factor != 0.0f)
    fail(LB2_UNSUPPORTED, "KMeans: redos = %u with a balance factor is not implemented (redos = 1 only)", redos);
}

static void pq_train_dev(const float* data, uint64_t n, int d, int metric, const lb2_pq_params* p,
                         float* codebook, std::vector<uint32_t>* iters) {
  const int M = p->num_sub_vectors, K = 1 << p->num_bits;
  LB2_REQUIRE(M > 0 && d % M == 0, "num_sub_vectors must divide vector dimension %d, but got %d", d, M);
  if (p->num_bits != 8 && p->num_bits != 4)  // pq/builder.rs: only 4 and 8 exist in the reference
    fail(LB2_INVALID_ARG, "PQ: num_bits must be 4 or 8, got %u", p->num_bits);
  check_redos(p->kmeans_redos, 0.0f);
  LB2_REQUIRE(current_comm() || n >= (uint64_t)K, "Not enough rows to train PQ. Requires %d rows but only %llu available",
              K, (unsigned long long)n);
  // free fn train_kmeans (kmeans.rs:1328-1340): first sample_rate*k rows (per-rank share when sharded)
  const uint64_t nranks = current_comm() ? current_comm()->nranks : 1;
  const uint64_t cap = (p->sample_rate * K + nranks - 1) / nranks;
  const uint64_t rows = n > cap ? cap : n;
  InArg<float> init(p->codebook, (size_t)M * K * (d / M));
  lloyd_train(data, rows, d, M, d / M, K, metric == METRIC_DOT ? METRIC_DOT : METRIC_L2, 0.0f,
              (int)p->max_iters, 1e-4, p->seed, init.get(), codebook, nullptr, iters);
}

// s distinct rows out of n, ascending: one uniformly random row from each of s equal strata
// (the reference draws a random subset through Dataset::sample, rust/lance/src/index/vector/utils.rs:
// 202-209, with an unseeded rng -> the selection is unpinned; ours is O(s), seeded, already sorted)
static std::vector<uint64_t> sample_rows(uint64_t n, uint64_t s, uint64_t seed) {
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

// one pass over a caller's matrix in chunks of rows: f(xf, xnat, r0, rows) with xf = the chunk as f32 on the device
// and xnat = the same rows in the column's own type (for assign_f32: tc_assign.cu, "native 16-bit rows")
template <class F>
static void for_each_chunk(Source& src, F&& f) {
  const uint64_t n = src.n(), chunk = src.rows_per_chunk();
  // (a little more than one chunk is not split: SIFT-1M is one call)
  const uint64_t step = n <= chunk + chunk / 2 ? std::max<uint64_t>(n, 1) : chunk;
  for (uint64_t r0 = 0; r0 < n; r0 += step) {
    const uint64_t rows = std::min(step, n - r0);
    const float* xf = src.rows_f32(r0, rows);
    if (r0 + rows < n) src.prefetch(r0 + rows, std::min(step, n - r0 - rows));
    f(xf, src.last_native(), r0, rows);
  }
}

// IvfTransformer::transform over one chunk of rows already on the device as f32 (lance-index/src/vector/ivf.rs:
// 188-236,357): [normalise if cosine] -> partition id -> residual -> PQ code.  The quantizer of an index build is
// trained -- and therefore encodes -- with L2 whatever the index metric is: Q::build(&training_data,
// DistanceType::L2, ..) (rust/lance/src/index/vector/builder.rs:460); the index metric only decides the partition
// assignment, whether residuals are taken (not for dot, PQBuildParams::use_residual) and the query-time table.
// xnat / dtype: the chunk's rows in their own type (for_each_chunk); a normalised chunk is assigned from f32 only
static void transform_chunk(const float* xf, const void* xnat, int dtype, uint64_t rows, int d, int m, const float* cent,
                            int K, const float* codebook, int M, int nbits, DevBuf<float>& normbuf, uint32_t* part,
                            uint8_t* codes, uint8_t* valid) {
  const float* xp = xf;
  if (m == METRIC_COSINE) {
    if (normbuf.n < (size_t)rows * d) normbuf.alloc((size_t)rows * d);
    LB2_LAUNCH("normalize", normalize_kernel, cdiv(rows, 128), 128, 0, xf, rows, d, normbuf.p);
    xp = normbuf.p;
    xnat = nullptr;
  }
  const int am = m == METRIC_DOT ? METRIC_DOT : METRIC_L2;
  assign_f32(xp, rows, d, cent, K, am, nullptr, part, nullptr, valid, nullptr, xnat, dtype);
  pq_encode_any(xp, rows, d, M, d / M, codebook, METRIC_L2, am == METRIC_DOT ? nullptr : cent,
                am == METRIC_DOT ? nullptr : part, valid, nbits, codes);
}

}  // namespace lb2

extern "C" {

const char* lb2_version(void) { return "lance_b200 0.1.0 (sm_90a)"; }

size_t lb2_last_error(char* buf, size_t len) {
  if (buf && len) {
    size_t c = std::min(len - 1, g_last_error.size());
    memcpy(buf, g_last_error.data(), c);
    buf[c] = 0;
  }
  return g_last_error.size();
}

int lb2_device_count(void) { return usable_devices(); }

lb2_status lb2_set_device(int device) {
  LB2_API_BEGIN
  int n = usable_devices();
  if (n <= 0) fail(LB2_NO_DEVICE, "no CUDA device");
  LB2_REQUIRE(device >= 0 && device < n, "device %d out of range (0..%d)", device, n - 1);
  g_requested_device = device;
  LB2_CUDA(cudaSetDevice(device));
  ctx();
  LB2_API_END
}
lb2_status lb2_synchronize(void) {
  LB2_API_BEGIN
  sync_stream();
  LB2_API_END
}
lb2_status lb2_trim_memory(void) {
  LB2_API_BEGIN
  sync_stream();
  staging_cache_release();
  sync_stream();
  cudaMemPool_t pool;
  if (cudaDeviceGetDefaultMemPool(&pool, ctx().device) == cudaSuccess) cudaMemPoolTrimTo(pool, 0);
  LB2_API_END
}
lb2_status lb2_set_stream(void* cuda_stream) {
  LB2_API_BEGIN
  Ctx& c = ctx();
  c.flush_profile();  // pending profile events belong to the stream they were recorded on
  c.stream = cuda_stream ? static_cast<cudaStream_t>(cuda_stream) : c.own_stream;
  LB2_API_END
}
lb2_status lb2_malloc(void** ptr, size_t bytes) {
  LB2_API_BEGIN
  ctx();
  LB2_CUDA(cudaMalloc(ptr, bytes ? bytes : 1));
  LB2_API_END
}
lb2_status lb2_free(void* ptr) {
  LB2_API_BEGIN
  ctx();
  LB2_CUDA(cudaFree(ptr));
  LB2_API_END
}
lb2_status lb2_malloc_host(void** ptr, size_t bytes) {
  LB2_API_BEGIN
  ctx();
  LB2_CUDA(cudaMallocHost(ptr, bytes ? bytes : 1));
  LB2_API_END
}
lb2_status lb2_free_host(void* ptr) {
  LB2_API_BEGIN
  ctx();
  LB2_CUDA(cudaFreeHost(ptr));
  LB2_API_END
}
lb2_status lb2_memcpy(void* dst, const void* src, size_t bytes) {
  LB2_API_BEGIN
  LB2_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDefault, ctx().stream));
  sync_stream();
  LB2_API_END
}
lb2_status lb2_launch_count(uint64_t* count, int reset) {
  LB2_API_BEGIN
  if (count) *count = ctx().launches;
  if (reset) ctx().launches = 0;
  LB2_API_END
}
lb2_status lb2_profile_enable(int on) {
  LB2_API_BEGIN
  ctx().flush_profile();
  ctx().profiling = on != 0;
  LB2_API_END
}
lb2_status lb2_profile_get(const char* name, uint64_t* launches, double* total_ms) {
  LB2_API_BEGIN
  ctx().flush_profile();
  auto it = ctx().prof.find(name ? name : "");
  if (launches) *launches = it == ctx().prof.end() ? 0 : it->second.launches;
  if (total_ms) *total_ms = it == ctx().prof.end() ? 0.0 : it->second.total_ms;
  LB2_API_END
}
lb2_status lb2_profile_reset(void) {
  LB2_API_BEGIN
  ctx().flush_profile();
  ctx().prof.clear();
  LB2_API_END
}
size_t lb2_profile_dump(char* buf, size_t len) {
  std::string out;
  try {
    ctx().flush_profile();
    for (auto& kv : ctx().prof) {
      char line[256];
      snprintf(line, sizeof(line), "%s\t%llu\t%.6f\n", kv.first.c_str(),
               (unsigned long long)kv.second.launches, kv.second.total_ms);
      out += line;
    }
  } catch (...) {
  }
  if (buf && len) {
    size_t c = std::min(len - 1, out.size());
    memcpy(buf, out.data(), c);
    buf[c] = 0;
  }
  return out.size();
}
lb2_status lb2_timer_start(void) {
  LB2_API_BEGIN
  LB2_CUDA(cudaEventRecord(ctx().t0, ctx().stream));
  LB2_API_END
}
lb2_status lb2_timer_stop(float* ms_out) {
  LB2_API_BEGIN
  LB2_CUDA(cudaEventRecord(ctx().t1, ctx().stream));
  LB2_CUDA(cudaEventSynchronize(ctx().t1));
  float ms = 0.f;
  LB2_CUDA(cudaEventElapsedTime(&ms, ctx().t0, ctx().t1));
  if (ms_out) *ms_out = ms;
  LB2_API_END
}

void lb2_kmeans_params_default(lb2_kmeans_params* p) {
  p->max_iters = 50;
  p->tolerance = 1e-4;
  p->redos = 1;
  p->balance_factor = 0.0f;
  p->hierarchical_k = 16;
  p->sample_rate = 256;
  p->seed = 0;
  p->init_centroids = nullptr;
  p->metric = LB2_L2;
}
void lb2_pq_params_default(lb2_pq_params* p) {
  p->num_sub_vectors = 16;
  p->num_bits = 8;
  p->max_iters = 50;
  p->kmeans_redos = 1;
  p->sample_rate = 256;
  p->codebook = nullptr;
  p->seed = 0;
}
void lb2_ivfpq_build_params_default(lb2_ivfpq_build_params* p) {
  p->num_partitions = 256;
  lb2_kmeans_params_default(&p->ivf);
  p->ivf.balance_factor = 1.0f;  // rust/lance/src/index/vector/ivf.rs:1858
  lb2_pq_params_default(&p->pq);
  p->seed = 0;
}

lb2_status lb2_distance_batch(const void* from, const void* to, uint64_t n, uint32_t d,
                              lb2_dtype dtype, lb2_metric metric, float* out) {
  LB2_API_BEGIN
  const int m = metric_of(metric);
  LB2_REQUIRE(d > 0, "dimension must be positive");
  LB2_REQUIRE(n < (1ull << 31), "too many rows");
  OutArg<float> o(out, n);
  if (dtype == LB2_U8 && m == METRIC_L2) {  // integer arithmetic (l2.rs:44-49)
    InArg<uint8_t> f8(from, d), t8(to, (size_t)n * d);
    if (n) LB2_LAUNCH("l2_u8", l2_u8_kernel, cdiv(n * 32, 256), 256, 0, f8.get(), t8.get(), n, (int)d, o.get());
    o.commit();
    sync_stream();
    return LB2_OK;
  }
  VecIn f(from, d, dtype), t(to, (size_t)n * d, dtype);
  if (m == METRIC_COSINE) {
    if (n) LB2_LAUNCH("cosine_batch", cosine_f32_kernel, cdiv(n * 32, 256), 256, 0, f.get(), t.get(), n, (int)d, o.get());
    o.commit();
    sync_stream();
    return LB2_OK;
  }
  assign_f32(f.get(), 1, d, t.get(), (int)n, m, nullptr, nullptr, nullptr, nullptr, o.get());
  o.commit();
  sync_stream();
  LB2_API_END
}

lb2_status lb2_normalize(const void* vectors, uint64_t n, uint32_t d, lb2_dtype dtype, void* out) {
  LB2_API_BEGIN
  VecIn x(vectors, (size_t)n * d, dtype);
  VecOut o(out, (size_t)n * d, model_dtype(dtype));
  if (n) LB2_LAUNCH("normalize", normalize_kernel, cdiv(n, 128), 128, 0, x.get(), n, (int)d, o.get());
  o.commit();
  sync_stream();
  LB2_API_END
}

lb2_status lb2_kmeans_train(const void* data, uint64_t n, uint32_t d, lb2_dtype dtype, uint32_t k,
                            const lb2_kmeans_params* params, void* centroids_out, double* loss_out,
                            uint32_t* iters_out) {
  LB2_API_BEGIN
  LB2_REQUIRE(params && data && centroids_out, "null argument");
  check_redos(params->redos, params->balance_factor);
  const int m = metric_of(params->metric);
  if (m == METRIC_COSINE)
    fail(LB2_INVALID_ARG, "KMeans: cosine is trained as L2 on normalised vectors (normalise first)");
  LB2_REQUIRE(current_comm() || n >= k, "KMeans: can not train %u centroids with %llu vectors, choose a smaller K (< %llu) instead",
              k, (unsigned long long)n, (unsigned long long)n);
  // free fn train_kmeans (kmeans.rs:1328-1344); sharded: every rank contributes its share of the cap
  const uint64_t kr0 = current_comm() ? current_comm()->nranks : 1;
  const uint64_t cap = (params->sample_rate * k + kr0 - 1) / kr0;
  const uint64_t rows = n > cap ? cap : n;
  VecIn x(data, (size_t)rows * d, dtype);
  VecIn init(params->init_centroids, (size_t)k * d, model_dtype(dtype));
  DevBuf<float> cent((size_t)k * d);
  std::vector<double> loss;
  std::vector<uint32_t> iters;
  const uint64_t kr = current_comm() ? current_comm()->nranks : 1;  // sharded: every rank passes its rows
  if (k > 256 && params->hierarchical_k > 1 && !params->init_centroids) {  // kmeans.rs:1027
    hierarchical_train(x.get(), rows, d, k, m, params->balance_factor / (float)(rows * kr),
                       (int)params->max_iters, params->tolerance, (int)params->hierarchical_k, params->seed, cent.p);
    loss.assign(1, 0.0);
    iters.assign(1, 0);
  } else {
    lloyd_train(x.get(), rows, d, 1, d, k, m, params->balance_factor / (float)(rows * kr),
                (int)params->max_iters, params->tolerance, params->seed, init.get(), cent.p, &loss,
                &iters);
  }
  VecOut o(centroids_out, (size_t)k * d, model_dtype(dtype));
  d2d(o.get(), cent.p, (size_t)k * d);
  o.commit();
  sync_stream();
  if (loss_out) *loss_out = loss[0];
  if (iters_out) *iters_out = iters[0];
  LB2_API_END
}

lb2_status lb2_compute_partitions(const void* centroids, uint32_t k, uint32_t d, lb2_dtype dtype,
                                  lb2_metric metric, const void* vectors, uint64_t n,
                                  uint32_t* part_out, float* dist_out, uint8_t* valid_out) {
  LB2_API_BEGIN
  const int m = metric_of(metric);
  if (m == METRIC_COSINE) fail(LB2_INVALID_ARG, "compute_partitions: normalise and use L2 for cosine");
  VecIn c(centroids, (size_t)k * d, model_dtype(dtype));
  OutArg<uint32_t> p(part_out, n);
  OutArg<float> dd(dist_out, n);
  OutArg<uint8_t> v(valid_out, n);
  if (n) {
    Source src(vectors, n, (int)d, dtype);
    src.start_resident_copy();
    for_each_chunk(src, [&](const float* xf, const void* xnat, uint64_t r0, uint64_t rows) {
      assign_f32(xf, rows, d, c.get(), k, m, nullptr, p.get() + r0, dd.get() ? dd.get() + r0 : nullptr,
                 v.get() ? v.get() + r0 : nullptr, nullptr, xnat, (int)src.dtype());
    });
  }
  p.commit(); dd.commit(); v.commit();
  sync_stream();
  LB2_API_END
}

lb2_status lb2_find_partitions(const void* centroids, uint32_t k, uint32_t d, lb2_dtype dtype,
                               lb2_metric metric, const void* queries, uint64_t nq,
                               uint32_t nprobes, uint32_t* ids_out, float* dists_out) {
  LB2_API_BEGIN

  const int m = metric_of(metric);
  if (m == METRIC_COSINE) fail(LB2_INVALID_ARG, "find_partitions: normalise and use L2 for cosine");
  const uint32_t np = std::min(nprobes, k);
  LB2_REQUIRE(np == nprobes, "nprobes %u exceeds the number of partitions %u", nprobes, k);
  VecIn c(centroids, (size_t)k * d, model_dtype(dtype)), q(queries, (size_t)nq * d, dtype);
  OutArg<uint32_t> ids(ids_out, (size_t)nq * np);
  OutArg<float> dd(dists_out, (size_t)nq * np);
  find_partitions_f32(c.get(), k, d, m, q.get(), nq, np, ids.get(), dd.get());
  ids.commit(); dd.commit();
  sync_stream();
  LB2_API_END
}

lb2_status lb2_compute_residual(const void* centroids, uint32_t k, uint32_t d, lb2_dtype dtype,
                                const void* vectors, uint64_t n, const uint32_t* part_ids,
                                void* out) {
  LB2_API_BEGIN
  VecIn c(centroids, (size_t)k * d, model_dtype(dtype)), x(vectors, (size_t)n * d, dtype);
  InArg<uint32_t> p(part_ids, n);
  check_part_ids(p.get(), n, k, "compute_residual");
  VecOut o(out, (size_t)n * d, model_dtype(dtype));
  if (n)
    LB2_LAUNCH("residual", residual_kernel, cdiv(n * d, 256), 256, 0, x.get(), c.get(), p.get(), n,
               (int)d, o.get());
  o.commit();
  sync_stream();
  LB2_API_END
}

lb2_status lb2_pq_train(const void* data, uint64_t n, uint32_t d, lb2_dtype dtype,
                        lb2_metric metric, const lb2_pq_params* params, void* codebook_out,
                        uint32_t* iters_out) {
  LB2_API_BEGIN
  LB2_REQUIRE(params && data && codebook_out, "null argument");
  const int m = metric_of(metric);
  if (m == METRIC_COSINE) fail(LB2_INVALID_ARG, "PQ code does not support cosine");  // pq/builder.rs:98-102
  VecIn x(data, (size_t)n * d, dtype);
  const size_t cb = (size_t)(1u << params->num_bits) * d;
  DevBuf<float> codebook(cb);
  std::vector<uint32_t> iters;
  VecIn cb_init(params->codebook, cb, model_dtype(dtype));
  lb2_pq_params pp = *params;
  pp.codebook = cb_init.get();  // device f32 view of the user codebook (or NULL)
  pq_train_dev(x.get(), n, d, m, &pp, codebook.p, &iters);
  VecOut o(codebook_out, cb, model_dtype(dtype));
  d2d(o.get(), codebook.p, cb);
  o.commit();
  sync_stream();
  if (iters_out)
    for (uint32_t i = 0; i < params->num_sub_vectors; ++i) iters_out[i] = iters[i];
  LB2_API_END
}

lb2_status lb2_pq_encode(const void* codebook, uint32_t num_sub_vectors, uint32_t num_bits,
                         uint32_t d, lb2_dtype dtype, lb2_metric metric, const void* centroids,
                         uint32_t num_centroids, const uint32_t* part_ids, const void* vectors, uint64_t n,
                         uint8_t* codes_out) {
  LB2_API_BEGIN
  if (num_bits != 8 && num_bits != 4) fail(LB2_INVALID_ARG, "PQ: num_bits must be 4 or 8, got %u", num_bits);
  const int M = num_sub_vectors, ds = d / M;
  LB2_REQUIRE(M > 0 && d % M == 0, "num_sub_vectors must divide vector dimension %u, but got %d", d, M);
  LB2_REQUIRE(num_bits == 8 || M % 2 == 0, "PQ: num_sub_vectors must be divisible by 2 for num_bits=4, but got %d", M);
  LB2_REQUIRE((centroids == nullptr) == (part_ids == nullptr),
              "centroids and part_ids must be given together");
  LB2_REQUIRE(centroids == nullptr || num_centroids > 0, "num_centroids must be given with centroids");
  const int ncode = 1 << num_bits;
  const int m = metric_of(metric) == METRIC_DOT ? METRIC_DOT : METRIC_L2;
  if (!small_d_supported(ds)) fail(LB2_UNSUPPORTED, "PQ sub-vector width %d not supported yet", ds);
  VecIn cb(codebook, (size_t)ncode * d, model_dtype(dtype)), x(vectors, (size_t)n * d, dtype);
  VecIn c(centroids, (size_t)num_centroids * d, model_dtype(dtype));
  InArg<uint32_t> p(part_ids, n);
  if (centroids) check_part_ids(p.get(), n, num_centroids, "pq_encode");
  OutArg<uint8_t> o(codes_out, (size_t)n * (num_bits == 4 ? M / 2 : M));
  pq_encode_any(x.get(), n, d, M, ds, cb.get(), m, c.get(), p.get(), nullptr, (int)num_bits, o.get());
  o.commit();
  sync_stream();
  LB2_API_END
}

lb2_status lb2_pq_scan_4bit(const float* lut, uint32_t num_sub_vectors, lb2_metric metric,
                            const uint8_t* codes_transposed, uint64_t n, uint64_t k_hint, float* dists_out) {
  LB2_API_BEGIN
  LB2_REQUIRE(num_sub_vectors > 0 && num_sub_vectors % 2 == 0,
              "PQ: num_sub_vectors must be divisible by 2 for num_bits=4, but got %u", num_sub_vectors);
  InArg<float> l(lut, (size_t)num_sub_vectors * 16);
  InArg<uint8_t> c(codes_transposed, (size_t)n * (num_sub_vectors / 2));
  OutArg<float> o(dists_out, n);
  pq_scan_4bit_f32(l.get(), num_sub_vectors, metric_of(metric), c.get(), n, k_hint, o.get());
  o.commit();
  sync_stream();
  LB2_API_END
}

lb2_status lb2_pq_build_lut(const void* codebook, uint32_t num_sub_vectors, uint32_t num_bits,
                            uint32_t d, lb2_metric metric, const float* query, float* lut_out) {
  LB2_API_BEGIN
  const int ncode = 1 << num_bits;
  LB2_REQUIRE(num_sub_vectors > 0 && d % num_sub_vectors == 0, "num_sub_vectors must divide d");
  InArg<float> cb(codebook, (size_t)ncode * d), q(query, d);
  OutArg<float> o(lut_out, (size_t)num_sub_vectors * ncode);
  build_lut_f32(cb.get(), num_sub_vectors, num_bits, d,
                metric_of(metric) == METRIC_DOT ? METRIC_DOT : METRIC_L2, q.get(), o.get());
  o.commit();
  sync_stream();
  LB2_API_END
}

lb2_status lb2_pq_scan(const float* lut, uint32_t num_sub_vectors, uint32_t num_bits,
                       lb2_metric metric, const uint8_t* codes_transposed, uint64_t n,
                       float* dists_out) {
  LB2_API_BEGIN
  if (num_bits != 8) fail(LB2_UNSUPPORTED, "num_bits %u is not implemented on the device", num_bits);
  InArg<float> l(lut, (size_t)num_sub_vectors * 256);
  InArg<uint8_t> c(codes_transposed, (size_t)n * num_sub_vectors);
  OutArg<float> o(dists_out, n);
  pq_scan_transposed_f32(l.get(), num_sub_vectors, metric_of(metric), c.get(), n, o.get());
  o.commit();
  sync_stream();
  LB2_API_END
}

static ScanFilter make_filter(const uint64_t* allow, int has_lower, float lower, int has_upper, float upper) {
  ScanFilter f;
  f.allow = allow;
  f.range = (has_lower || has_upper) ? 1 : 0;
  // flat/index.rs:101-102: lower_bound.unwrap_or(f32::MIN), upper_bound.unwrap_or(f32::MAX)
  f.lo_key = host_total_key(has_lower ? lower : -3.40282347e+38f);
  f.hi_key = host_total_key(has_upper ? upper : 3.40282347e+38f);
  return f;
}

lb2_status lb2_flat_topk_range(const float* dists, const uint64_t* row_ids, uint64_t n, uint32_t k,
                               int has_lower, float lower, int has_upper, float upper,
                               uint64_t* ids_out, float* dists_out, uint32_t* count_out) {
  LB2_API_BEGIN
  LB2_REQUIRE(k > 0, "k must be positive");
  LB2_REQUIRE(n < 0xffffffffull, "too many rows");
  InArg<float> dd(dists, n);
  InArg<uint64_t> r(row_ids, n);
  OutArg<uint64_t> oi(ids_out, k);
  OutArg<float> od(dists_out, k);
  OutArg<uint32_t> oc(count_out, 1);
  DevBuf<uint32_t> cnt_tmp;
  uint32_t* cp = oc.get();
  if (!cp) { cnt_tmp.alloc(1); cp = cnt_tmp.p; }
  flat_topk_f32(dd.get(), r.get(), n, k, make_filter(nullptr, has_lower, lower, has_upper, upper), oi.get(),
                od.get(), cp);
  oi.commit(); od.commit(); oc.commit();
  sync_stream();
  LB2_API_END
}

lb2_status lb2_flat_topk(const float* dists, const uint64_t* row_ids, uint64_t n, uint32_t k,
                         uint64_t* ids_out, float* dists_out, uint32_t* count_out) {
  return lb2_flat_topk_range(dists, row_ids, n, k, 0, 0.0f, 0, 0.0f, ids_out, dists_out, count_out);
}

lb2_status lb2_ivfpq_transform(const void* centroids, uint32_t k, const void* codebook,
                               uint32_t num_sub_vectors, uint32_t num_bits, uint32_t d,
                               lb2_dtype dtype, lb2_metric metric, const void* vectors, uint64_t n,
                               uint32_t* part_out, uint8_t* codes_out, uint8_t* valid_out) {
  LB2_API_BEGIN

  if (num_bits != 8 && num_bits != 4) fail(LB2_INVALID_ARG, "PQ: num_bits must be 4 or 8, got %u", num_bits);
  const int M = num_sub_vectors, ds = d / M;
  LB2_REQUIRE(M > 0 && d % M == 0, "num_sub_vectors must divide vector dimension %u, but got %d", d, M);
  LB2_REQUIRE(num_bits == 8 || M % 2 == 0, "PQ: num_sub_vectors must be divisible by 2 for num_bits=4, but got %d", M);
  if (!small_d_supported(ds)) fail(LB2_UNSUPPORTED, "PQ sub-vector width %d not supported yet", ds);
  const int m = metric_of(metric);
  VecIn c(centroids, (size_t)k * d, model_dtype(dtype)), cb(codebook, ((size_t)1 << num_bits) * d, model_dtype(dtype));
  const size_t cw = num_bits == 4 ? M / 2 : M;
  OutArg<uint32_t> p(part_out, n);
  OutArg<uint8_t> co(codes_out, (size_t)n * cw), v(valid_out, n);
  DevBuf<uint8_t> vtmp;
  uint8_t* vp = v.get();
  if (!vp) { vtmp.alloc(std::max<uint64_t>(n, 1)); vp = vtmp.p; }
  if (n) {
    Source src(vectors, n, (int)d, dtype);
    src.start_resident_copy();
    DevBuf<float> normbuf;
    for_each_chunk(src, [&](const float* xf, const void* xnat, uint64_t r0, uint64_t rows) {
      transform_chunk(xf, xnat, (int)src.dtype(), rows, (int)d, m, c.get(), (int)k, cb.get(), M, (int)num_bits, normbuf,
                      p.get() + r0, co.get() + r0 * cw, vp + r0);
    });
  }
  p.commit(); co.commit(); v.commit();
  sync_stream();
  LB2_API_END
}

lb2_status lb2_index_create(const void* centroids, uint32_t k, uint32_t d, lb2_dtype dtype,
                            lb2_metric metric, const void* codebook, uint32_t num_sub_vectors,
                            uint32_t num_bits, lb2_index** out) {
  LB2_API_BEGIN
  LB2_REQUIRE(out && centroids && codebook, "null argument");
  LB2_REQUIRE(num_sub_vectors > 0 && d % num_sub_vectors == 0, "num_sub_vectors must divide d");
  if (num_bits != 8 && num_bits != 4) fail(LB2_INVALID_ARG, "PQ: num_bits must be 4 or 8, got %u", num_bits);
  LB2_REQUIRE(num_bits == 8 || num_sub_vectors % 2 == 0,
              "PQ: num_sub_vectors must be divisible by 2 for num_bits=4, but got %u", num_sub_vectors);
  ctx();
  lb2_index* ix = new lb2_index();
  ix->K = k; ix->d = d; ix->M = num_sub_vectors; ix->nbits = num_bits; ix->metric = metric_of(metric);
  ix->dtype = dtype;
  ix->centroids.alloc((size_t)k * d);
  ix->codebook.alloc(ix->codebook_len());
  {
    VecIn c(centroids, (size_t)k * d, model_dtype(dtype)), cb(codebook, ix->codebook_len(), model_dtype(dtype));
    d2d(ix->centroids.p, c.get(), (size_t)k * d);
    d2d(ix->codebook.p, cb.get(), ix->codebook_len());
    sync_stream();
  }
  ix->part_offsets.alloc(k + 1);
  ix->part_offsets.zero();
  sync_stream();
  *out = ix;
  LB2_API_END
}

lb2_status lb2_index_load(lb2_index* index, const uint32_t* part_ids, const uint8_t* codes,
                          const uint64_t* row_ids, uint64_t n) {
  LB2_API_BEGIN
  LB2_REQUIRE(index && index->kind == 0, "not an IVF_PQ index");
  InArg<uint32_t> p(part_ids, n);
  InArg<uint8_t> c(codes, (size_t)n * index->code_bytes());
  InArg<uint64_t> r(row_ids, n);
  check_part_ids(p.get(), n, (uint32_t)index->K, "index_load");
  index_load_dev(index, p.get(), c.get(), r.get(), n);
  LB2_API_END
}

// one implementation behind lb2_index_search / _search_refine / _search_ex
static void index_search_impl(lb2_index* index, const void* queries, uint64_t nq, uint32_t k, uint32_t nprobes,
                              uint32_t refine_factor, const void* vectors, uint64_t num_vectors,
                              const uint64_t* allow_bitmap, uint64_t* row_ids_out, float* dists_out,
                              uint32_t* counts_out, int has_lower = 0, float lower = 0.0f, int has_upper = 0,
                              float upper = 0.0f, ProbeRule* pr = nullptr) {
  LB2_REQUIRE(index && k > 0 && (nprobes > 0 || pr), "bad argument");
  const bool refine = refine_factor > 0 && vectors != nullptr;
  const uint64_t kc = refine ? (uint64_t)k * refine_factor : k;
  if (kc > 1024) fail(LB2_UNSUPPORTED, "k * refine_factor = %llu > 1024 is not implemented", (unsigned long long)kc);
  const int d = index->d;
  VecIn q(queries, (size_t)nq * d, index->dtype);
  const float* qp = q.get();
  DevBuf<float> qn;
  if (index->metric == METRIC_COSINE) {  // knn.rs:497-499
    qn.alloc((size_t)nq * d);
    if (nq) LB2_LAUNCH("normalize", normalize_kernel, cdiv(nq, 128), 128, 0, qp, nq, d, qn.p);
    qp = qn.p;
  }
  InArg<uint64_t> allow(allow_bitmap, allow_bitmap ? (size_t)((index->n + 63) / 64) : 0);
  OutArg<uint64_t> oi(row_ids_out, (size_t)nq * k);
  OutArg<float> od(dists_out, (size_t)nq * k);
  OutArg<uint32_t> oc(counts_out, nq);
  DevBuf<uint64_t> cid;
  DevBuf<float> cdist;
  DevBuf<uint32_t> ccnt;
  if (refine) {
    cid.alloc((size_t)nq * kc);
    cdist.alloc((size_t)nq * kc);
    ccnt.alloc(nq);
  }
  uint64_t* si = refine ? cid.p : oi.get();
  float* sd = refine ? cdist.p : od.get();
  uint32_t* sc = refine ? ccnt.p : oc.get();
  TagScope tg("search");
  const ScanFilter flt = make_filter(allow_bitmap ? allow.get() : nullptr, has_lower, lower, has_upper, upper);
  DevBuf<uint8_t> qcodes;
  if (index->kind == 1) {
    ivfflat_search_f32(index->centroids.p, index->K, d, index->metric, index->part_offsets.p, index->vectors.p,
                       (int)index->vdtype(), index->row_ids.p, qp, nq, (int)kc, nprobes, si, sd, sc, flt, pr);
  } else if (index->kind == 3) {
    // the (normalised) query's residual to each probed centroid is rotated (v2.rs:316-332, bq/storage.rs:407-445)
    ivfrq_search_f32(index->centroids.p, index->K, d, index->metric, index->rq_rot.p, index->code_dim(),
                     index->part_offsets.p, index->codes.p, index->rq_add.p, index->rq_scale.p, index->row_ids.p, qp,
                     nq, (int)kc, nprobes, si, sd, sc, flt, pr);
  } else if (index->kind == 2) {
    // the (normalised) query is encoded with the index's bounds, not turned into a residual (sq/storage.rs:404-430)
    qcodes.alloc(std::max<uint64_t>(1, nq * d));
    sq_encode_f32(qp, nq * d, index->sq_lower, index->sq_upper, qcodes.p);
    const float rf = (float)(index->sq_upper - index->sq_lower);  // inverse_scalar_dist (sq.rs:279-287)
    ivfsq_search_f32(index->centroids.p, index->K, d, index->metric, index->part_offsets.p, index->codes.p,
                     index->row_ids.p, rf * rf, qp, qcodes.p, nq, (int)kc, nprobes, si, sd, sc, flt, pr);
  } else {
    ivfpq_search_f32(index->centroids.p, index->K, d, index->metric, index->codebook.p, index->M, index->nbits,
                     index->part_offsets.p, index->codes.p, index->row_ids.p, qp, nq, (int)kc, nprobes, si, sd,
                     sc, flt, index->slab_off.p, index->codes_skew.p, pr);
  }
  if (refine) {
    // exact re-rank with the true metric on the ORIGINAL (un-normalised) query, as flat_knn does; the
    // plan then filters `_distance >= lower AND _distance < upper` on the exact distances (scanner.rs:3342-3377)
    InArg<uint8_t> v(vectors, (size_t)num_vectors * d * dtype_size(index->dtype));  // raw column, native type
    refine_f32(q.get(), nq, d, index->metric, v.get(), (int)index->dtype, num_vectors, cid.p, ccnt.p, (int)kc, (int)k,
               oi.get(), od.get(), oc.get(), has_lower, lower, has_upper, upper);
    oi.commit(); od.commit(); oc.commit();
    if (!ctx().async_call) sync_stream();
    return;
  }
  oi.commit(); od.commit(); oc.commit();
  if (!ctx().async_call) sync_stream();
}

lb2_status lb2_index_search(lb2_index* index, const void* queries, uint64_t nq, uint32_t k,
                            uint32_t nprobes, uint64_t* row_ids_out, float* dists_out,
                            uint32_t* counts_out) {
  LB2_API_BEGIN
  index_search_impl(index, queries, nq, k, nprobes, 0, nullptr, 0, nullptr, row_ids_out, dists_out, counts_out);
  LB2_API_END
}

lb2_status lb2_index_search_refine(lb2_index* index, const void* vectors, uint64_t num_vectors,
                                   const void* queries, uint64_t nq, uint32_t k, uint32_t nprobes,
                                   uint32_t refine_factor, uint64_t* row_ids_out, float* dists_out,
                                   uint32_t* counts_out) {
  LB2_API_BEGIN
  LB2_REQUIRE(vectors && refine_factor > 0, "bad argument");
  index_search_impl(index, queries, nq, k, nprobes, refine_factor, vectors, num_vectors, nullptr, row_ids_out,
                    dists_out, counts_out);
  LB2_API_END
}

lb2_status lb2_index_search_ex(lb2_index* index, const void* queries, uint64_t nq,
                               const lb2_search_params* sp, uint64_t* row_ids_out, float* dists_out,
                               uint32_t* counts_out) {
  LB2_API_BEGIN
  LB2_REQUIRE(sp, "null search params");
  LB2_REQUIRE(sp->refine_factor == 0 || sp->refine_vectors, "refine_factor > 0 needs refine_vectors");
  index_search_impl(index, queries, nq, sp->k, sp->nprobes, sp->refine_factor, sp->refine_vectors,
                    sp->num_vectors, sp->allow_bitmap, row_ids_out, dists_out, counts_out, sp->has_lower_bound != 0,
                    sp->lower_bound, sp->has_upper_bound != 0, sp->upper_bound);
  LB2_API_END
}

lb2_status lb2_index_search_probed(lb2_index* index, const void* queries, uint64_t nq, const lb2_search_params* sp,
                                   const lb2_probe_params* pp, uint64_t* row_ids_out, float* dists_out,
                                   uint32_t* counts_out, uint32_t* nprobes_out) {
  LB2_API_BEGIN
  LB2_REQUIRE(sp && pp && index, "null argument");
  LB2_REQUIRE(sp->nprobes == 0, "nprobes must be 0: the probe parameters decide the probes");
  LB2_REQUIRE(sp->refine_factor == 0 || sp->refine_vectors, "refine_factor > 0 needs refine_vectors");
  LB2_REQUIRE(pp->minimum_nprobes >= 1, "minimum_nprobes must be at least 1");
  LB2_REQUIRE(pp->maximum_nprobes == 0 || pp->maximum_nprobes >= pp->minimum_nprobes,
              "maximum_nprobes %u is below minimum_nprobes %u", pp->maximum_nprobes, pp->minimum_nprobes);
  LB2_REQUIRE(pp->late_width >= 1, "late_width must be at least 1");
  LB2_REQUIRE(sp->allow_bitmap || (!pp->has_max_len && !pp->mask_ids), "max_len and mask_ids need an allow bitmap");
  if (current_comm() && current_comm()->nranks > 1)
    fail(LB2_UNSUPPORTED, "a search with minimum / maximum nprobes on a row-sharded index is not implemented");
  InArg<uint64_t> mask(pp->mask_ids, pp->mask_ids ? pp->num_mask_ids : 0);
  DevBuf<uint64_t> no_ids(pp->mask_ids && pp->num_mask_ids == 0 ? 1 : 0);  // an iterable, empty allow list
  OutArg<uint32_t> np_out(nprobes_out, nq);
  ProbeRule pr;
  pr.min_np = pp->minimum_nprobes;
  pr.max_np = pp->maximum_nprobes;
  pr.late_width = pp->late_width;
  pr.k = sp->k;
  pr.has_max_len = pp->has_max_len != 0;
  pr.max_len = pp->max_len;
  pr.mask_ids = pp->mask_ids ? (mask.get() ? mask.get() : no_ids.p) : nullptr;
  pr.num_mask_ids = pp->mask_ids ? pp->num_mask_ids : 0;
  pr.nprobes_out = np_out.get();
  index_search_impl(index, queries, nq, sp->k, 0, sp->refine_factor, sp->refine_vectors, sp->num_vectors,
                    sp->allow_bitmap, row_ids_out, dists_out, counts_out, sp->has_lower_bound != 0, sp->lower_bound,
                    sp->has_upper_bound != 0, sp->upper_bound, &pr);
  np_out.commit();
  sync_stream();
  LB2_API_END
}

// RAII: route the thread's work to the caller's stream for one asynchronous call
namespace {
struct AsyncScope {
  Ctx& c;
  cudaStream_t saved;
  explicit AsyncScope(void* stream) : c(ctx()), saved(c.stream) {
    if (stream) c.stream = static_cast<cudaStream_t>(stream);
    c.async_call = true;
  }
  ~AsyncScope() {
    c.async_call = false;
    c.stream = saved;
  }
};
}  // namespace

lb2_status lb2_index_search_async(lb2_index* index, const void* queries, uint64_t nq,
                                  const lb2_search_params* sp, uint64_t* row_ids_out, float* dists_out,
                                  uint32_t* counts_out, void* cuda_stream, void* done_event) {
  LB2_API_BEGIN
  LB2_REQUIRE(sp, "null search params");
  LB2_REQUIRE(sp->refine_factor == 0 || sp->refine_vectors, "refine_factor > 0 needs refine_vectors");
  AsyncScope scope(cuda_stream);
  index_search_impl(index, queries, nq, sp->k, sp->nprobes, sp->refine_factor, sp->refine_vectors,
                    sp->num_vectors, sp->allow_bitmap, row_ids_out, dists_out, counts_out, sp->has_lower_bound != 0,
                    sp->lower_bound, sp->has_upper_bound != 0, sp->upper_bound);
  if (done_event) LB2_CUDA(cudaEventRecord(static_cast<cudaEvent_t>(done_event), ctx().stream));
  LB2_API_END
}

lb2_status lb2_index_search_sharded(lb2_index* index, const void* queries, uint64_t nq,
                                    const lb2_search_params* sp, uint64_t* row_ids_out, float* dists_out,
                                    uint32_t* counts_out) {
  LB2_API_BEGIN
  LB2_REQUIRE(sp && index, "null argument");
  LB2_REQUIRE(sp->refine_factor == 0 || sp->refine_vectors, "refine_factor > 0 needs refine_vectors");
  const uint32_t k = sp->k;
  DevBuf<uint64_t> li((size_t)std::max<uint64_t>(1, nq * k));
  DevBuf<float> ld((size_t)std::max<uint64_t>(1, nq * k));
  DevBuf<uint32_t> lc(std::max<uint64_t>(1, nq));
  index_search_impl(index, queries, nq, k, sp->nprobes, sp->refine_factor, sp->refine_vectors, sp->num_vectors,
                    sp->allow_bitmap, li.p, ld.p, lc.p, sp->has_lower_bound != 0, sp->lower_bound,
                    sp->has_upper_bound != 0, sp->upper_bound);
  OutArg<uint64_t> oi(row_ids_out, (size_t)nq * k);
  OutArg<float> od(dists_out, (size_t)nq * k);
  OutArg<uint32_t> oc(counts_out, nq);
  DevBuf<uint32_t> ctmp;
  uint32_t* cp = oc.get();
  if (!cp) { ctmp.alloc(std::max<uint64_t>(1, nq)); cp = ctmp.p; }
  if (nq) merge_sharded_topk(li.p, ld.p, lc.p, nq, (int)k, oi.get(), od.get(), cp);
  oi.commit(); od.commit(); oc.commit();
  sync_stream();
  LB2_API_END
}

// ---- partition ownership: device all-to-all (SURVEY 8e "partition build", 8f-4) ---------------------------------
// The reference groups the transformed rows by partition with a disk shuffler on the host
// (rust/lance-index/src/vector/v3/shuffler.rs:105).  For a build sharded by rows over G GPUs the same grouping
// is one exchange over NVLink: rank g becomes the owner of every partition p with p % G == g.
namespace lb2 {
// row i of the shard (storage order) -> slot in the send buffer: rows are grouped by destination rank, inside a
// destination by partition, inside a partition in storage order
__global__ void repart_pack_kernel(const uint64_t* __restrict__ part_offsets, int K, uint64_t n, int row_bytes,
                                   const uint64_t* __restrict__ send_base /*[K]*/, const uint8_t* __restrict__ payload,
                                   const uint64_t* __restrict__ row_ids, uint8_t* __restrict__ payload_out,
                                   uint64_t* __restrict__ row_ids_out) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int lo = 0, hi = K;  // last p with part_offsets[p] <= i
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (part_offsets[mid] <= i) lo = mid; else hi = mid;
  }
  const uint64_t dst = send_base[lo] + (i - part_offsets[lo]);
  row_ids_out[dst] = row_ids[i];
  const uint8_t* src = payload + i * (uint64_t)row_bytes;
  uint8_t* o = payload_out + dst * (uint64_t)row_bytes;
  if ((row_bytes & 15) == 0) {
    for (int b = 0; b < row_bytes; b += 16) *reinterpret_cast<uint4*>(o + b) = *reinterpret_cast<const uint4*>(src + b);
  } else {
    for (int b = 0; b < row_bytes; ++b) o[b] = src[b];
  }
}
// received row j of source rank r (rows of my partitions in ascending partition order) -> final storage position
__global__ void repart_unpack_kernel(const uint64_t* __restrict__ seg_prefix /*[nown + 1] rows of r before owned part i*/,
                                     const uint64_t* __restrict__ seg_dst /*[nown] final position of r's first row*/,
                                     int nown, uint64_t nrows, int row_bytes, const uint8_t* __restrict__ payload,
                                     const uint64_t* __restrict__ row_ids, uint8_t* __restrict__ payload_out,
                                     uint64_t* __restrict__ row_ids_out) {
  const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= nrows) return;
  int lo = 0, hi = nown;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (seg_prefix[mid] <= j) lo = mid; else hi = mid;
  }
  const uint64_t dst = seg_dst[lo] + (j - seg_prefix[lo]);
  row_ids_out[dst] = row_ids[j];
  const uint8_t* src = payload + j * (uint64_t)row_bytes;
  uint8_t* o = payload_out + dst * (uint64_t)row_bytes;
  if ((row_bytes & 15) == 0) {
    for (int b = 0; b < row_bytes; b += 16) *reinterpret_cast<uint4*>(o + b) = *reinterpret_cast<const uint4*>(src + b);
  } else {
    for (int b = 0; b < row_bytes; ++b) o[b] = src[b];
  }
}
}  // namespace lb2

lb2_status lb2_index_repartition(const lb2_index* shard, lb2_index** owned_out) {
  LB2_API_BEGIN
  LB2_REQUIRE(shard && owned_out, "null argument");
  if (shard->kind == 3) fail(LB2_UNSUPPORTED, "lb2_index_repartition: IVF_RQ indexes are not implemented");
  Comm* cm = current_comm();
  const int G = cm ? cm->nranks : 1, me = cm ? cm->rank : 0;
  const int K = shard->K;
  // the row payload: IVF_FLAT's vectors, or the codes of IVF_PQ / IVF_SQ (code_bytes() = d for IVF_SQ)
  const int rb = shard->kind == 1 ? (int)shard->vrow_bytes() : shard->code_bytes();
  const uint8_t* payload = shard->kind == 1 ? shard->vectors.p : shard->codes.p;
  // every rank's partition sizes (one all-gather of K counters), then the layouts on the host
  std::vector<uint64_t> offs(K + 1);
  d2h(offs.data(), shard->part_offsets.p, (size_t)K + 1);
  sync_stream();
  std::vector<uint64_t> mine(K), all((size_t)G * K);
  for (int p = 0; p < K; ++p) mine[p] = offs[p + 1] - offs[p];
  {
    DevBuf<uint64_t> dm(K), da((size_t)G * K);
    h2d(dm.p, mine.data(), K);
    comm_allgather_bytes(dm.p, da.p, (size_t)K * 8);
    d2h(all.data(), da.p, (size_t)G * K);
    sync_stream();
  }
  // send side: rows for destination g = partitions p % G == g, ascending p
  std::vector<size_t> s_off(G), s_bytes(G), r_off(G), r_bytes(G);
  std::vector<uint64_t> s_rows(G, 0), r_rows(G, 0), send_base(K);
  for (int p = 0; p < K; ++p) s_rows[p % G] += mine[p];
  {
    std::vector<uint64_t> run(G, 0);
    uint64_t acc = 0;
    std::vector<uint64_t> gbase(G);
    for (int g = 0; g < G; ++g) { gbase[g] = acc; acc += s_rows[g]; }
    for (int p = 0; p < K; ++p) { send_base[p] = gbase[p % G] + run[p % G]; run[p % G] += mine[p]; }
    for (int g = 0; g < G; ++g) { s_off[g] = gbase[g]; s_bytes[g] = s_rows[g]; }
  }
  // receive side: from source r the rows of my partitions; final order inside a partition = source rank order
  const int nown = (K - me + G - 1) / G;  // partitions me, me + G, ...
  uint64_t n_new = 0;
  std::vector<uint64_t> new_off(K + 1, 0);
  for (int p = 0; p < K; ++p) {
    new_off[p] = n_new;
    if (p % G == me) for (int r = 0; r < G; ++r) n_new += all[(size_t)r * K + p];
  }
  new_off[K] = n_new;
  LB2_REQUIRE(n_new < 0xffffffffull, "more than 2^32-1 rows per index shard");
  {
    uint64_t acc = 0;
    for (int r = 0; r < G; ++r) {
      for (int i = 0; i < nown; ++i) r_rows[r] += all[(size_t)r * K + (me + (size_t)i * G)];
      r_off[r] = acc; r_bytes[r] = r_rows[r]; acc += r_rows[r];
    }
  }
  const uint64_t n = shard->n;
  DevBuf<uint8_t> sp(std::max<uint64_t>(1, n * rb)), rp(std::max<uint64_t>(1, n_new * rb));
  DevBuf<uint64_t> si(std::max<uint64_t>(1, n)), ri(std::max<uint64_t>(1, n_new)), dbase(K);
  h2d(dbase.p, send_base.data(), K);
  if (n)
    LB2_LAUNCH("repartition_pack", repart_pack_kernel, cdiv(n, 256), 256, 0, shard->part_offsets.p, K, n, rb,
               (const uint64_t*)dbase.p, payload, (const uint64_t*)shard->row_ids.p, sp.p, si.p);
  {
    std::vector<size_t> so(G), sb(G), ro(G), rbv(G);
    for (int g = 0; g < G; ++g) { so[g] = s_off[g] * rb; sb[g] = s_bytes[g] * rb; ro[g] = r_off[g] * rb; rbv[g] = r_bytes[g] * rb; }
    comm_alltoallv_bytes(sp.p, so.data(), sb.data(), rp.p, ro.data(), rbv.data());
    for (int g = 0; g < G; ++g) { so[g] = s_off[g] * 8; sb[g] = s_bytes[g] * 8; ro[g] = r_off[g] * 8; rbv[g] = r_bytes[g] * 8; }
    comm_alltoallv_bytes(si.p, so.data(), sb.data(), ri.p, ro.data(), rbv.data());
  }
  std::unique_ptr<lb2_index> ix(new lb2_index());
  ix->kind = shard->kind; ix->dtype = shard->dtype; ix->K = K; ix->d = shard->d; ix->M = shard->M;
  ix->nbits = shard->nbits; ix->metric = shard->metric; ix->n = n_new;
  ix->sq_lower = shard->sq_lower; ix->sq_upper = shard->sq_upper;
  ix->centroids.alloc((size_t)K * shard->d);
  d2d(ix->centroids.p, shard->centroids.p, (size_t)K * shard->d);
  if (shard->kind == 0) {
    ix->codebook.alloc(shard->codebook_len());
    d2d(ix->codebook.p, shard->codebook.p, shard->codebook_len());
  }
  ix->part_offsets.alloc(K + 1);
  h2d(ix->part_offsets.p, new_off.data(), (size_t)K + 1);
  DevBuf<uint8_t>& dstp = shard->kind == 1 ? ix->vectors : ix->codes;
  dstp.alloc(std::max<uint64_t>(1, n_new * rb));
  ix->row_ids.alloc(std::max<uint64_t>(1, n_new));
  // place every (source rank, owned partition) segment: seg_prefix = rows of r before its i-th owned partition
  std::vector<uint64_t> pre((size_t)nown + 1), dst(std::max(1, nown));
  DevBuf<uint64_t> dpre((size_t)nown + 1), ddst(std::max(1, nown));
  std::vector<uint64_t> before(std::max(1, nown), 0);  // rows of lower ranks already placed in owned partition i
  for (int r = 0; r < G; ++r) {
    uint64_t acc = 0;
    for (int i = 0; i < nown; ++i) {
      const int p = me + i * G;
      pre[i] = acc;
      dst[i] = new_off[p] + before[i];
      acc += all[(size_t)r * K + p];
      before[i] += all[(size_t)r * K + p];
    }
    pre[nown] = acc;
    if (!acc) continue;
    h2d(dpre.p, pre.data(), (size_t)nown + 1);
    h2d(ddst.p, dst.data(), (size_t)nown);
    LB2_LAUNCH("repartition_unpack", repart_unpack_kernel, cdiv(acc, 256), 256, 0, (const uint64_t*)dpre.p,
               (const uint64_t*)ddst.p, nown, acc, rb, (const uint8_t*)(rp.p + r_off[r] * rb),
               (const uint64_t*)(ri.p + r_off[r]), dstp.p, ix->row_ids.p);
    sync_stream();  // pre / dst are reused by the next source rank
  }
  if (shard->kind == 0 && n_new && skew_layout_applies(ix->M, ix->d, ix->nbits)) {
    ix->slab_off.alloc(K + 1);
    ix->codes_skew.alloc(skew_bytes_bound(n_new, K));
    build_skew_codes(ix->part_offsets.p, K, ix->codes.p, n_new, ix->slab_off.p, ix->codes_skew.p);
  }
  sync_stream();
  *owned_out = ix.release();
  LB2_API_END
}

// ---- incremental update of an IVF_PQ index: the data path of optimize / split / join (SURVEY 8f-4) --------------
// The reference turns an optimize step into per-partition AssignOp::Add / AssignOp::Remove lists against a new
// centroid set (rust/lance/src/index/vector/builder.rs:1219-1333 split, :1476-1530 join, :1534-1650
// build_assign_batch) and merges them with the existing partitions when it writes the index.  The decisions --
// which partition to split or join, which rows to move -- stay on the host (they need the dataset); this entry
// point is the merge: old rows keep their codes, follow `part_map`, removed row ids are dropped, added rows join
// the end of their partitions.
namespace lb2 {
__device__ __forceinline__ bool in_sorted_u64(const uint64_t* __restrict__ a, uint64_t n, uint64_t v) {
  uint64_t lo = 0, hi = n;
  while (lo < hi) {
    const uint64_t mid = (lo + hi) >> 1;
    if (a[mid] < v) lo = mid + 1; else hi = mid;
  }
  return lo < n && a[lo] == v;
}
__global__ void update_old_rows_kernel(const uint64_t* __restrict__ part_offsets, int K, uint64_t n,
                                       const uint32_t* __restrict__ part_map /*nullable*/,
                                       const uint64_t* __restrict__ row_ids, const uint64_t* __restrict__ removed,
                                       uint64_t n_removed, uint32_t new_k, uint32_t* __restrict__ part_out,
                                       uint8_t* __restrict__ valid_out, uint32_t* __restrict__ bad) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int lo = 0, hi = K;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (part_offsets[mid] <= i) lo = mid; else hi = mid;
  }
  const uint32_t np_ = part_map ? part_map[lo] : (uint32_t)lo;
  bool keep = np_ != 0xffffffffu;
  if (keep && np_ >= new_k) { atomicMax(bad, np_); keep = false; }
  if (keep && n_removed) keep = !in_sorted_u64(removed, n_removed, row_ids[i]);
  part_out[i] = keep ? np_ : 0u;
  valid_out[i] = keep ? 1 : 0;
}
__global__ void fill_u8_kernel(uint8_t* __restrict__ p, uint64_t n, uint8_t v) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}
}  // namespace lb2

lb2_status lb2_index_update(const lb2_index* old, const void* new_centroids, uint32_t new_k, const uint32_t* part_map,
                            const uint32_t* add_part_ids, const uint8_t* add_codes, const uint64_t* add_row_ids,
                            uint64_t n_add, const uint64_t* remove_row_ids, uint64_t n_remove, lb2_index** out) {
  LB2_API_BEGIN
  LB2_REQUIRE(old && out && old->kind == 0, "lb2_index_update takes an IVF_PQ index");
  LB2_REQUIRE(new_k > 0 && (new_centroids || new_k == (uint32_t)old->K), "a changed partition count needs new centroids");
  LB2_REQUIRE(n_add == 0 || (add_part_ids && add_codes && add_row_ids), "added rows need partition ids, codes and row ids");
  LB2_REQUIRE(n_remove == 0 || remove_row_ids, "null remove list");
  const int d = old->d, cbw = old->code_bytes();
  const uint64_t n_old = old->n, n_all = n_old + n_add;
  LB2_REQUIRE(n_all < 0xffffffffull, "more than 2^32-1 rows per index shard");
  std::unique_ptr<lb2_index> ix(new lb2_index());
  ix->kind = 0; ix->dtype = old->dtype; ix->K = (int)new_k; ix->d = d; ix->M = old->M; ix->nbits = old->nbits;
  ix->metric = old->metric;
  ix->centroids.alloc((size_t)new_k * d);
  if (new_centroids) {
    VecIn c(new_centroids, (size_t)new_k * d, model_dtype(old->dtype));
    d2d(ix->centroids.p, c.get(), (size_t)new_k * d);
    sync_stream();
  } else {
    d2d(ix->centroids.p, old->centroids.p, (size_t)new_k * d);
  }
  ix->codebook.alloc(old->codebook_len());
  d2d(ix->codebook.p, old->codebook.p, old->codebook_len());
  InArg<uint32_t> pm(part_map, part_map ? (size_t)old->K : 0), ap(add_part_ids, n_add);
  InArg<uint8_t> ac(add_codes, (size_t)n_add * cbw);
  InArg<uint64_t> ar(add_row_ids, n_add), rm(remove_row_ids, n_remove);
  if (n_add) check_part_ids(ap.get(), n_add, new_k, "index_update");
  // one row list: old rows in storage order, then the added rows (so a partition keeps its old rows first)
  DevBuf<uint32_t> part(std::max<uint64_t>(1, n_all)), bad(1);
  DevBuf<uint8_t> valid(std::max<uint64_t>(1, n_all)), codes(std::max<uint64_t>(1, n_all * cbw));
  DevBuf<uint64_t> rid(std::max<uint64_t>(1, n_all));
  bad.zero();
  if (n_old) {
    LB2_LAUNCH("update_old_rows", update_old_rows_kernel, cdiv(n_old, 256), 256, 0, old->part_offsets.p, old->K, n_old,
               pm.get(), (const uint64_t*)old->row_ids.p, rm.get(), n_remove, new_k, part.p, valid.p, bad.p);
    d2d(codes.p, old->codes.p, (size_t)n_old * cbw);
    d2d(rid.p, old->row_ids.p, (size_t)n_old);
  }
  if (n_add) {
    d2d(part.p + n_old, ap.get(), (size_t)n_add);
    d2d(codes.p + n_old * cbw, ac.get(), (size_t)n_add * cbw);
    d2d(rid.p + n_old, ar.get(), (size_t)n_add);
    LB2_LAUNCH("fill_valid", fill_u8_kernel, cdiv(n_add, 256), 256, 0, valid.p + n_old, n_add, (uint8_t)1);
  }
  uint32_t hbad = 0;
  d2h(&hbad, bad.p, 1);
  sync_stream();
  if (hbad) fail(LB2_INVALID_ARG, "index_update: part_map sends a partition to %u, the new index has %u partitions", hbad, new_k);
  index_load_dev(ix.get(), part.p, codes.p, rid.p, n_all, valid.p);
  *out = ix.release();
  LB2_API_END
}

lb2_status lb2_comm_info(int* rank, int* nranks) {
  LB2_API_BEGIN
  Comm* c = current_comm();
  if (rank) *rank = c ? c->rank : 0;
  if (nranks) *nranks = c ? c->nranks : 1;
  LB2_API_END
}

lb2_status lb2_index_row_mask(const lb2_index* index, const uint64_t* allow_ids, uint64_t n_allow,
                              int has_allow, const uint64_t* block_ids, uint64_t n_block, int has_block,
                              uint64_t* bitmap_out) {
  LB2_API_BEGIN
  LB2_REQUIRE(index && bitmap_out, "bad argument");
  LB2_REQUIRE((!has_allow || n_allow == 0 || allow_ids) && (!has_block || n_block == 0 || block_ids), "null id list");
  InArg<uint64_t> a(allow_ids, has_allow ? (size_t)n_allow : 0), b(block_ids, has_block ? (size_t)n_block : 0);
  OutArg<uint64_t> bm(bitmap_out, (size_t)((index->n + 63) / 64));
  row_mask_f32(index->row_ids.p, index->n, a.get(), n_allow, has_allow != 0, b.get(), n_block, has_block != 0,
               bm.get());
  bm.commit();
  sync_stream();
  LB2_API_END
}

lb2_status lb2_index_info(const lb2_index* index, uint32_t* k, uint32_t* d, uint32_t* num_sub_vectors,
                          uint32_t* num_bits, uint64_t* num_rows) {
  LB2_API_BEGIN
  LB2_REQUIRE(index, "null index");
  if (k) *k = index->K;
  if (d) *d = index->d;
  if (num_sub_vectors) *num_sub_vectors = index->M;
  if (num_bits) *num_bits = index->nbits;
  if (num_rows) *num_rows = index->n;
  LB2_API_END
}

lb2_status lb2_index_export(const lb2_index* index, void* centroids_out, void* codebook_out,
                            uint64_t* part_offsets_out, uint8_t* codes_out, uint64_t* row_ids_out) {
  LB2_API_BEGIN
  LB2_REQUIRE(index && index->kind == 0, "not an IVF_PQ index");
  cudaStream_t s = ctx().stream;
  if (centroids_out)
    LB2_CUDA(cudaMemcpyAsync(centroids_out, index->centroids.p, sizeof(float) * index->K * index->d, cudaMemcpyDefault, s));
  if (codebook_out)
    LB2_CUDA(cudaMemcpyAsync(codebook_out, index->codebook.p, sizeof(float) * index->codebook_len(), cudaMemcpyDefault, s));
  if (part_offsets_out)
    LB2_CUDA(cudaMemcpyAsync(part_offsets_out, index->part_offsets.p, sizeof(uint64_t) * (index->K + 1), cudaMemcpyDefault, s));
  if (codes_out && index->n)
    LB2_CUDA(cudaMemcpyAsync(codes_out, index->codes.p, index->n * index->code_bytes(), cudaMemcpyDefault, s));
  if (row_ids_out && index->n)
    LB2_CUDA(cudaMemcpyAsync(row_ids_out, index->row_ids.p, sizeof(uint64_t) * index->n, cudaMemcpyDefault, s));
  sync_stream();
  LB2_API_END
}

void lb2_ivfflat_build_params_default(lb2_ivfflat_build_params* p) {
  p->num_partitions = 256;
  lb2_kmeans_params_default(&p->ivf);
  p->ivf.balance_factor = 1.0f;
  p->seed = 0;
}

// an empty IVF_FLAT / IVF_SQ index with the caller's centroids (in the model type of `dtype`)
static lb2_index* index_with_centroids(int kind, const void* centroids, uint32_t k, uint32_t d, lb2_dtype dtype,
                                       lb2_metric metric) {
  ctx();
  std::unique_ptr<lb2_index> ix(new lb2_index());
  ix->kind = kind; ix->K = k; ix->d = d; ix->M = 0; ix->nbits = 0; ix->metric = metric_of(metric);
  ix->dtype = dtype;
  ix->centroids.alloc((size_t)k * d);
  {
    VecIn c(centroids, (size_t)k * d, model_dtype(dtype));
    d2d(ix->centroids.p, c.get(), (size_t)k * d);
    sync_stream();
  }
  ix->part_offsets.alloc(k + 1);
  ix->part_offsets.zero();
  sync_stream();
  return ix.release();
}

lb2_status lb2_index_create_flat(const void* centroids, uint32_t k, uint32_t d, lb2_dtype dtype,
                                 lb2_metric metric, lb2_index** out) {
  LB2_API_BEGIN
  LB2_REQUIRE(out && centroids, "null argument");
  *out = index_with_centroids(1, centroids, k, d, dtype, metric);
  LB2_API_END
}

lb2_status lb2_index_load_flat(lb2_index* index, const uint32_t* part_ids, const void* vectors,
                               const uint64_t* row_ids, uint64_t n) {
  LB2_API_BEGIN
  LB2_REQUIRE(index && index->kind == 1, "not an IVF_FLAT index");
  LB2_REQUIRE(index->d % 4 == 0, "IVF_FLAT needs a dimension that is a multiple of 4");
  InArg<uint32_t> p(part_ids, n);
  InArg<uint64_t> r(row_ids, n);
  check_part_ids(p.get(), n, (uint32_t)index->K, "index_load_flat");
  Source src(vectors, n, index->d, index->dtype);
  src.start_resident_copy();
  index_load_flat_src(index, p.get(), src, r.get(), nullptr, /*normalize=*/false);
  LB2_API_END
}

lb2_status lb2_index_export_flat(const lb2_index* index, void* centroids_out,
                                 uint64_t* part_offsets_out, void* vectors_out,
                                 uint64_t* row_ids_out) {
  LB2_API_BEGIN
  LB2_REQUIRE(index && index->kind == 1, "not an IVF_FLAT index");
  cudaStream_t s = ctx().stream;
  if (centroids_out)
    LB2_CUDA(cudaMemcpyAsync(centroids_out, index->centroids.p, sizeof(float) * index->K * index->d, cudaMemcpyDefault, s));
  if (part_offsets_out)
    LB2_CUDA(cudaMemcpyAsync(part_offsets_out, index->part_offsets.p, sizeof(uint64_t) * (index->K + 1), cudaMemcpyDefault, s));
  if (vectors_out && index->n)
    LB2_CUDA(cudaMemcpyAsync(vectors_out, index->vectors.p, index->n * index->vrow_bytes(), cudaMemcpyDefault, s));
  if (row_ids_out && index->n)
    LB2_CUDA(cudaMemcpyAsync(row_ids_out, index->row_ids.p, sizeof(uint64_t) * index->n, cudaMemcpyDefault, s));
  sync_stream();
  LB2_API_END
}

namespace {
// CUDA events of a build, destroyed on every path
struct EventSet {
  std::vector<cudaEvent_t> ev;
  explicit EventSet(int n) : ev(n, nullptr) {
    for (auto& e : ev) LB2_CUDA(cudaEventCreate(&e));
  }
  ~EventSet() {
    for (auto& e : ev)
      if (e) cudaEventDestroy(e);
  }
  void record(int i) { LB2_CUDA(cudaEventRecord(ev[i], ctx().stream)); }
  float ms(int i, int j) const {
    float t = 0.f;
    cudaEventElapsedTime(&t, ev[i], ev[j]);
    return t;
  }
};
// KMeans::new_with_params (kmeans.rs:1008-1030): hierarchical for k > 256, flat Lloyd otherwise
void train_ivf(const float* xs, uint64_t s, int d, int K, int am, const lb2_kmeans_params& kp, uint64_t nranks,
               const float* init, float* centroids, std::vector<double>* loss, std::vector<uint32_t>* iters) {
  check_redos(kp.redos, kp.balance_factor);
  if (K > 256 && kp.hierarchical_k > 1 && !init) {
    loss->assign(1, 0.0);
    iters->assign(1, 0);
    if (nranks > 1) {
      // Sharded build: the hierarchical tree is thousands of small dependent Lloyd runs -- with a collective in
      // every iteration it is latency-bound on the exchange.  The sample (K * sample_rate rows) is small next to
      // the data, so when it fits every rank gathers ALL sample shards (rank order) and trains the same tree on
      // them without a communicator: identical arithmetic on identical input gives bit-identical models on all
      // ranks, and the splits train concurrently (kmeans.cu: SplitWorkers).  Otherwise: the sharded tree.
      DevBuf<uint64_t> cnt_in(1), cnt_all(nranks);
      h2d(cnt_in.p, &s, 1);
      comm_allgather_bytes(cnt_in.p, cnt_all.p, sizeof(uint64_t));
      std::vector<uint64_t> cnt(nranks);
      d2h(cnt.data(), cnt_all.p, nranks);
      sync_stream();
      uint64_t total = 0, mx = 0;
      for (uint64_t c : cnt) { total += c; mx = std::max(mx, c); }
      size_t free_b = 0, total_b = 0;
      cudaMemGetInfo(&free_b, &total_b);
      const bool off = getenv("LB2_SHARDED_TREE") && *getenv("LB2_SHARDED_TREE");
      if (!off && total < 0xffffffffull && (size_t)nranks * mx * d * 4 * 3 <= free_b) {
        DevBuf<float> pad, all((size_t)nranks * mx * d);
        const float* in = xs;
        if (s < mx) {
          pad.alloc((size_t)mx * d);
          pad.zero();
          if (s) d2d(pad.p, xs, (size_t)s * d);
          in = pad.p;
        }
        comm_allgather_bytes(in, all.p, (size_t)mx * d * sizeof(float));
        pad.release();
        if (total != nranks * mx) {  // unequal shards: close the gaps (rank order is kept)
          DevBuf<float> full(std::max<uint64_t>(total, 1) * d);
          uint64_t o = 0;
          for (uint64_t r = 0; r < nranks; ++r) {
            if (cnt[r]) d2d(full.p + o * d, all.p + r * mx * d, cnt[r] * d);
            o += cnt[r];
          }
          all = std::move(full);
        }
        Comm* saved = comm_swap(nullptr);
        try {
          hierarchical_train(all.p, total, d, K, am, kp.balance_factor / (float)total, (int)kp.max_iters, kp.tolerance,
                             (int)kp.hierarchical_k, kp.seed, centroids);
        } catch (...) {
          comm_swap(saved);
          throw;
        }
        comm_swap(saved);
        return;
      }
    }
    hierarchical_train(xs, s, d, K, am, kp.balance_factor / (float)(s * nranks), (int)kp.max_iters, kp.tolerance,
                       (int)kp.hierarchical_k, kp.seed, centroids);
  } else {
    lloyd_train(xs, s, d, 1, d, K, am, kp.balance_factor / (float)(s * nranks), (int)kp.max_iters, kp.tolerance,
                kp.seed, init, centroids, loss, iters);
  }
}
}  // namespace

// The IVF stage shared by the IVF_FLAT and IVF_SQ builds: sample (ivf.rs:1237-1241) -> drop rows that are not
// finite -> train (normalised first under cosine) -> centroids rounded to the column's type.  Starts the bulk copy.
static void train_ivf_stage(Source& src, lb2_index* ix, const lb2_kmeans_params& kp, uint64_t seed, uint64_t nranks,
                            std::vector<double>* loss, std::vector<uint32_t>* iters) {
  TagScope tg("ivf_train");
  const uint64_t n = src.n();
  const int d = src.d(), K = ix->K, m = ix->metric;
  const int am = m == METRIC_DOT ? METRIC_DOT : METRIC_L2;
  const uint64_t s0 = std::min<uint64_t>(n, ((uint64_t)K * kp.sample_rate + nranks - 1) / nranks);
  std::vector<uint64_t> rows = sample_rows(n, s0, seed);
  DevBuf<float> sample;
  const uint64_t s = gather_finite_sample(src, rows, m == METRIC_COSINE, sample);
  src.start_resident_copy();  // host rows: the bulk copy runs on its own stream while the centroids train
  LB2_REQUIRE(nranks > 1 || s >= (uint64_t)K, "KMeans: can not train %d centroids with %llu finite vectors", K,
              (unsigned long long)s);
  VecIn init(kp.init_centroids, (size_t)K * d, model_dtype(ix->dtype));
  train_ivf(sample.p, s, d, K, am, kp, nranks, init.get(), ix->centroids.p, loss, iters);
  round_model(ix->centroids.p, (size_t)K * d, ix->dtype);
}

// partition assignment of one chunk of rows (IVF_FLAT / IVF_SQ / IVF_RQ transform); returns the chunk as f32 as the
// index sees it: normalised under cosine (NormalizeTransformer first, ivf.rs:158-166).  Rows with a non-finite
// element are dropped in every metric (KeepFiniteVectors precedes the partition transform, ivf.rs:166, 256,
// 299).  Under L2 and cosine such a row has no finite distance and the assignment already drops it;
// under dot a +-inf element can still give a -inf best distance, so the elements are checked.
static const float* assign_flat_chunk(const float* xf, const void* xnat, int dtype, uint64_t rows, int d, int m,
                                      const float* cent, int K, DevBuf<float>& normbuf, uint32_t* part,
                                      uint8_t* valid, float* dist = nullptr) {
  const int am = m == METRIC_DOT ? METRIC_DOT : METRIC_L2;
  const float* xp = xf;
  if (m == METRIC_COSINE) {
    if (normbuf.n < (size_t)rows * d) normbuf.alloc((size_t)rows * d);
    LB2_LAUNCH("normalize", normalize_kernel, cdiv(rows, 128), 128, 0, xf, rows, d, normbuf.p);
    xp = normbuf.p;
    xnat = nullptr;
  }
  assign_f32(xp, rows, d, cent, K, am, nullptr, part, dist, valid, nullptr, xnat, dtype);
  if (am == METRIC_DOT && rows)
    LB2_LAUNCH("drop_nonfinite_rows", drop_nonfinite_rows_kernel, cdiv(rows * 32, 256), 256, 0, xp, rows, d, valid);
  return xp;
}

lb2_status lb2_ivfflat_build(const void* data, uint64_t n, uint32_t d, lb2_dtype dtype,
                             lb2_metric metric, const lb2_ivfflat_build_params* params,
                             const uint64_t* row_ids, lb2_index** out, lb2_build_stats* stats) {
  LB2_API_BEGIN
  LB2_REQUIRE(data && params && out, "null argument");
  LB2_REQUIRE(d % 4 == 0, "IVF_FLAT needs a dimension that is a multiple of 4");
  const int m = metric_of(metric);
  const int K = params->num_partitions;
  const uint64_t nranks = current_comm() ? current_comm()->nranks : 1;
  LB2_REQUIRE(K > 0 && (nranks > 1 || n >= (uint64_t)K), "KMeans: can not train %d centroids with %llu vectors", K,
              (unsigned long long)n);
  EventSet ev(4);
  ev.record(0);
  Source src(data, n, (int)d, dtype);
  std::unique_ptr<lb2_index> ix(new lb2_index());
  ix->kind = 1; ix->K = K; ix->d = d; ix->M = 0; ix->nbits = 0; ix->metric = m; ix->dtype = dtype;
  ix->centroids.alloc((size_t)K * d);
  std::vector<double> loss;
  std::vector<uint32_t> iters;
  train_ivf_stage(src, ix.get(), params->ivf, params->seed, nranks, &loss, &iters);
  ev.record(1);
  DevBuf<uint32_t> part(std::max<uint64_t>(n, 1));
  DevBuf<uint8_t> valid(std::max<uint64_t>(n, 1));
  {
    TagScope tg("transform");
    DevBuf<float> normbuf;
    for_each_chunk(src, [&](const float* xf, const void* xnat, uint64_t r0, uint64_t rows) {
      assign_flat_chunk(xf, xnat, (int)src.dtype(), rows, (int)d, m, ix->centroids.p, K, normbuf, part.p + r0,
                        valid.p + r0);
    });
  }
  ev.record(2);
  InArg<uint64_t> rid(row_ids, n);
  {
    TagScope tg("group");  // the stored vectors are the normalised ones when the metric is cosine
    index_load_flat_src(ix.get(), part.p, src, rid.get(), valid.p, m == METRIC_COSINE);
  }
  ev.record(3);
  sync_stream();
  if (stats) {
    memset(stats, 0, sizeof(*stats));
    stats->ms_ivf_train = ev.ms(0, 1);
    stats->ms_transform = ev.ms(1, 2);
    stats->ms_group = ev.ms(2, 3);
    stats->ms_total = ev.ms(0, 3);
    stats->ivf_iters = iters.empty() ? 0 : iters[0];
    stats->ivf_loss = loss.empty() ? 0.0 : loss[0];
  }
  *out = ix.release();
  LB2_API_END
}

// ---- IVF_SQ: IVFIndex<FlatIndex, ScalarQuantizer> (lance-index/src/vector/sq*.rs) --------------------------------
static void sq_check_dim(uint32_t d) {
  LB2_REQUIRE(d > 0 && d % 4 == 0, "IVF_SQ needs a dimension that is a multiple of 4");
  // the scan sums d terms of up to 255^2 in u32 (sq/storage.rs:432-468)
  LB2_REQUIRE((uint64_t)d * 255 * 255 < (1ull << 32), "IVF_SQ: d * 255^2 must be below 2^32, d = %u", d);
}

lb2_status lb2_sq_train(const void* data, uint64_t n, uint32_t d, lb2_dtype dtype, double* lower_out,
                        double* upper_out) {
  LB2_API_BEGIN
  LB2_REQUIRE((data || n == 0) && lower_out && upper_out, "null argument");
  ctx();
  VecIn x(data, (size_t)n * d, dtype);
  sq_bounds_f32(x.get(), (uint64_t)n * d, lower_out, upper_out);
  LB2_API_END
}

lb2_status lb2_sq_encode(const void* vectors, uint64_t n, uint32_t d, lb2_dtype dtype, double lower, double upper,
                         uint8_t* codes_out) {
  LB2_API_BEGIN
  LB2_REQUIRE((vectors && codes_out) || n == 0, "null argument");
  ctx();
  VecIn x(vectors, (size_t)n * d, dtype);
  OutArg<uint8_t> o(codes_out, (size_t)n * d);
  sq_encode_f32(x.get(), (uint64_t)n * d, lower, upper, o.get());
  o.commit();
  sync_stream();
  LB2_API_END
}

lb2_status lb2_index_create_sq(const void* centroids, uint32_t k, uint32_t d, lb2_dtype dtype, lb2_metric metric,
                               double lower, double upper, lb2_index** out) {
  LB2_API_BEGIN
  LB2_REQUIRE(out && centroids, "null argument");
  sq_check_dim(d);
  LB2_REQUIRE(std::isfinite(lower) && std::isfinite(upper) && lower <= upper,
              "IVF_SQ: the bounds must be finite with lower <= upper, got [%g, %g]", lower, upper);
  std::unique_ptr<lb2_index> ix(index_with_centroids(2, centroids, k, d, dtype, metric));
  ix->nbits = 8;
  ix->sq_lower = lower;
  ix->sq_upper = upper;
  *out = ix.release();
  LB2_API_END
}

lb2_status lb2_index_load_sq(lb2_index* index, const uint32_t* part_ids, const uint8_t* codes,
                             const uint64_t* row_ids, uint64_t n) {
  LB2_API_BEGIN
  LB2_REQUIRE(index && index->kind == 2, "not an IVF_SQ index");
  InArg<uint32_t> p(part_ids, n);
  InArg<uint8_t> c(codes, (size_t)n * index->d);
  InArg<uint64_t> r(row_ids, n);
  check_part_ids(p.get(), n, (uint32_t)index->K, "index_load_sq");
  index_load_dev(index, p.get(), c.get(), r.get(), n);
  LB2_API_END
}

lb2_status lb2_index_export_sq(const lb2_index* index, void* centroids_out, double* bounds_out,
                               uint64_t* part_offsets_out, uint8_t* codes_out, uint64_t* row_ids_out) {
  LB2_API_BEGIN
  LB2_REQUIRE(index && index->kind == 2, "not an IVF_SQ index");
  cudaStream_t s = ctx().stream;
  if (bounds_out) {
    bounds_out[0] = index->sq_lower;
    bounds_out[1] = index->sq_upper;
  }
  if (centroids_out)
    LB2_CUDA(cudaMemcpyAsync(centroids_out, index->centroids.p, sizeof(float) * index->K * index->d, cudaMemcpyDefault, s));
  if (part_offsets_out)
    LB2_CUDA(cudaMemcpyAsync(part_offsets_out, index->part_offsets.p, sizeof(uint64_t) * (index->K + 1), cudaMemcpyDefault, s));
  if (codes_out && index->n)
    LB2_CUDA(cudaMemcpyAsync(codes_out, index->codes.p, index->n * index->code_bytes(), cudaMemcpyDefault, s));
  if (row_ids_out && index->n)
    LB2_CUDA(cudaMemcpyAsync(row_ids_out, index->row_ids.p, sizeof(uint64_t) * index->n, cudaMemcpyDefault, s));
  sync_stream();
  LB2_API_END
}

void lb2_ivfsq_build_params_default(lb2_ivfsq_build_params* p) {
  p->num_partitions = 256;
  lb2_kmeans_params_default(&p->ivf);
  p->ivf.balance_factor = 1.0f;
  p->num_bits = 8;
  p->sample_rate = 256;
  p->seed = 0;
}

lb2_status lb2_ivfsq_build(const void* data, uint64_t n, uint32_t d, lb2_dtype dtype, lb2_metric metric,
                           const lb2_ivfsq_build_params* params, const uint64_t* row_ids, lb2_index** out,
                           lb2_build_stats* stats) {
  LB2_API_BEGIN
  LB2_REQUIRE(data && params && out, "null argument");
  sq_check_dim(d);
  if (params->num_bits != 8) fail(LB2_UNSUPPORTED, "IVF_SQ: num_bits = %u is not implemented (8 only)", params->num_bits);
  if (current_comm() && current_comm()->nranks > 1)
    fail(LB2_UNSUPPORTED, "IVF_SQ: builds sharded over ranks are not implemented (the bounds would need an exchange)");
  const int m = metric_of(metric);
  const int K = params->num_partitions;
  LB2_REQUIRE(K > 0 && n >= (uint64_t)K, "KMeans: can not train %d centroids with %llu vectors", K, (unsigned long long)n);
  EventSet ev(5);
  ev.record(0);
  Source src(data, n, (int)d, dtype);
  std::unique_ptr<lb2_index> ix(new lb2_index());
  ix->kind = 2; ix->K = K; ix->d = d; ix->M = 0; ix->nbits = 8; ix->metric = m; ix->dtype = dtype;
  ix->centroids.alloc((size_t)K * d);
  std::vector<double> loss;
  std::vector<uint32_t> iters;
  // 1. IVF: the same stage as lb2_ivfflat_build (same sample, seed, training)
  train_ivf_stage(src, ix.get(), params->ivf, params->seed, 1, &loss, &iters);
  ev.record(1);
  // 2. ScalarQuantizer::build (sq.rs:152-182) on sample_rate * 2^num_bits rows (builder.rs:410-421), normalised
  //    under cosine, rows that are not finite dropped (builder.rs:436), no residuals (quantizer.rs:52).  The bounds
  //    are taken over the values the index stores: normalised, in the column's element type.
  {
    TagScope tg("sq_train");
    std::vector<uint64_t> rows = sample_rows(n, std::min<uint64_t>(n, params->sample_rate * 256), params->seed + 1);
    DevBuf<float> sample;
    const uint64_t s = gather_finite_sample(src, rows, m == METRIC_COSINE, sample);
    round_model(sample.p, (size_t)s * d, dtype);
    sq_bounds_f32(sample.p, (uint64_t)s * d, &ix->sq_lower, &ix->sq_upper);
  }
  ev.record(2);
  // 3. transform (ivf.rs:238-279): partition, then the SQ codes of the stored vectors themselves
  DevBuf<uint32_t> part(std::max<uint64_t>(n, 1));
  DevBuf<uint8_t> valid(std::max<uint64_t>(n, 1)), codes(std::max<uint64_t>(1, (uint64_t)n * d));
  {
    TagScope tg("transform");
    DevBuf<float> normbuf;
    for_each_chunk(src, [&](const float* xf, const void* xnat, uint64_t r0, uint64_t rows) {
      const float* xs = assign_flat_chunk(xf, xnat, (int)src.dtype(), rows, (int)d, m, ix->centroids.p, K, normbuf,
                                          part.p + r0, valid.p + r0);
      if (m == METRIC_COSINE) round_model(normbuf.p, (size_t)rows * d, dtype);  // as IVF_FLAT stores them
      sq_encode_f32(xs, (uint64_t)rows * d, ix->sq_lower, ix->sq_upper, codes.p + r0 * d);
    });
  }
  ev.record(3);
  {
    TagScope tg("group");
    InArg<uint64_t> rid(row_ids, n);
    index_load_dev(ix.get(), part.p, codes.p, rid.get(), n, valid.p);
  }
  ev.record(4);
  sync_stream();
  if (stats) {
    memset(stats, 0, sizeof(*stats));
    stats->ms_ivf_train = ev.ms(0, 1);
    stats->ms_pq_train = ev.ms(1, 2);
    stats->ms_transform = ev.ms(2, 3);
    stats->ms_group = ev.ms(3, 4);
    stats->ms_total = ev.ms(0, 4);
    stats->ivf_iters = iters.empty() ? 0 : iters[0];
    stats->ivf_loss = loss.empty() ? 0.0 : loss[0];
  }
  *out = ix.release();
  LB2_API_END
}

// ---- IVF_RQ: IVFIndex<FlatIndex, RabitQuantizer> (lance-index/src/vector/bq/*.rs) ---------------------------------
static void rq_check(uint32_t d, lb2_dtype dtype, uint32_t num_bits) {
  // RabitQuantizer::build takes f16 / f32 / f64 columns only (bq/builder.rs:194-210)
  if (dtype == LB2_BF16 || dtype == LB2_U8) fail(LB2_INVALID_ARG, "IVF_RQ: unsupported data type %d", (int)dtype);
  if (dtype != LB2_F32)
    fail(LB2_UNSUPPORTED, "IVF_RQ: f16 columns are not implemented (the reference rotates them in f16)");
  LB2_REQUIRE(d > 0 && num_bits > 0, "IVF_RQ: the dimension and num_bits must be positive");
  const uint64_t cd = (uint64_t)d * num_bits;
  LB2_REQUIRE(cd % 8 == 0, "IVF_RQ: code_dim = d * num_bits = %llu is not a multiple of 8", (unsigned long long)cd);
  if (cd > 65536 || !rq_scan_fits((int)cd, 1))
    fail(LB2_UNSUPPORTED, "IVF_RQ: the tables of code_dim %llu do not fit the scan's shared memory",
         (unsigned long long)cd);
}

// IVF_RQ transform of one chunk (IvfTransformer::with_rq, ivf.rs:281-328): [normalise] -> partition and dist_v_c ->
// residual -> rotation -> sign codes and factors.  Cosine is L2 on the normalised rows from there on.
// The row chunk is bounded by d (Source::rows_per_chunk), the rotated rows by code_dim = d * num_bits: they are
// rotated and encoded in sub-chunks of at most 2^28 / code_dim rows (1 GB of f32).
struct RqWork {
  DevBuf<float> normbuf, dist, res, rot;
};
static void rq_transform_chunk(const float* xf, const void* xnat, int dtype, uint64_t rows, int d, int m,
                               const float* cent, int K, const float* rotation, int num_bits, const float* cnorm,
                               RqWork& w, uint32_t* part, uint8_t* valid, uint8_t* codes, float* add, float* scale) {
  const int cd = d * num_bits;
  const uint64_t sub = std::min<uint64_t>(rows, std::max<uint64_t>(1, (1ull << 28) / (uint64_t)cd));
  if (w.dist.n < rows) w.dist.alloc(rows);
  if (w.res.n < rows * d) w.res.alloc(rows * d);
  if (w.rot.n < sub * cd) w.rot.alloc(sub * cd);
  const float* xs = assign_flat_chunk(xf, xnat, dtype, rows, d, m, cent, K, w.normbuf, part, valid, w.dist.p);
  rq_residual_f32(xs, rows, d, cent, part, valid, w.res.p);
  for (uint64_t r0 = 0; r0 < rows; r0 += sub) {
    const uint64_t rs = std::min(sub, rows - r0);
    rq_rotate_f32(rotation, cd, d, w.res.p + r0 * d, rs, w.rot.p);
    rq_encode_f32(w.rot.p, w.res.p + r0 * d, w.dist.p + r0, part + r0, cnorm, valid + r0, rs, d, num_bits,
                  m == METRIC_DOT ? METRIC_DOT : METRIC_L2, codes + r0 * (cd / 8), add + r0, scale + r0);
  }
}

// |c|^2 per centroid (norm_squared_fsl, RQTransformer::new, bq/transform.rs:42-59): dot only
static void rq_centroid_norms(int metric, const float* cent, int K, int d, DevBuf<float>& out) {
  if (metric != METRIC_DOT) return;
  out.alloc(K);
  rq_norm_sq_f32(cent, K, d, out.p);
}

lb2_status lb2_rq_rotation(uint32_t code_dim, uint64_t seed, float* rotation_out) {
  LB2_API_BEGIN
  LB2_REQUIRE(rotation_out && code_dim > 0 && code_dim <= 65536, "bad argument");
  ctx();
  OutArg<float> o(rotation_out, (size_t)code_dim * code_dim);
  rq_rotation_f32((int)code_dim, seed, o.get());
  o.commit();
  sync_stream();
  LB2_API_END
}

lb2_status lb2_ivfrq_transform(const void* centroids, uint32_t k, const void* rotation, uint32_t d, uint32_t num_bits,
                               lb2_dtype dtype, lb2_metric metric, const void* vectors, uint64_t n, uint32_t* part_out,
                               uint8_t* codes_out, float* add_out, float* scale_out, uint8_t* valid_out) {
  LB2_API_BEGIN
  LB2_REQUIRE(centroids && rotation && (vectors || n == 0) && k > 0, "null argument");
  rq_check(d, dtype, num_bits);
  const int m = metric_of(metric);
  const uint64_t cd = (uint64_t)d * num_bits;
  VecIn c(centroids, (size_t)k * d, dtype), r(rotation, cd * cd, dtype);
  DevBuf<float> cnorm;
  rq_centroid_norms(m, c.get(), (int)k, (int)d, cnorm);
  OutArg<uint32_t> p(part_out, n);
  OutArg<uint8_t> co(codes_out, (size_t)(n * cd / 8)), v(valid_out, n);
  OutArg<float> ao(add_out, n), so(scale_out, n);
  DevBuf<uint32_t> ptmp;
  DevBuf<uint8_t> vtmp, ctmp;
  DevBuf<float> atmp, stmp;
  uint32_t* pp = p.get();
  uint8_t *vp = v.get(), *cp = co.get();
  float *ap = ao.get(), *sp = so.get();
  if (!pp) { ptmp.alloc(std::max<uint64_t>(n, 1)); pp = ptmp.p; }
  if (!vp) { vtmp.alloc(std::max<uint64_t>(n, 1)); vp = vtmp.p; }
  if (!cp) { ctmp.alloc(std::max<uint64_t>(n * cd / 8, 1)); cp = ctmp.p; }
  if (!ap) { atmp.alloc(std::max<uint64_t>(n, 1)); ap = atmp.p; }
  if (!sp) { stmp.alloc(std::max<uint64_t>(n, 1)); sp = stmp.p; }
  if (n) {
    Source src(vectors, n, (int)d, dtype);
    src.start_resident_copy();
    RqWork w;
    for_each_chunk(src, [&](const float* xf, const void* xnat, uint64_t r0, uint64_t rows) {
      rq_transform_chunk(xf, xnat, (int)src.dtype(), rows, (int)d, m, c.get(), (int)k, r.get(),
                         (int)num_bits, cnorm.p, w, pp + r0, vp + r0, cp + r0 * (cd / 8), ap + r0, sp + r0);
    });
  }
  p.commit(); co.commit(); v.commit(); ao.commit(); so.commit();
  sync_stream();
  LB2_API_END
}

void lb2_ivfrq_build_params_default(lb2_ivfrq_build_params* p) {
  p->num_partitions = 256;
  lb2_kmeans_params_default(&p->ivf);
  p->ivf.balance_factor = 1.0f;
  p->num_bits = 1;
  p->seed = 0;
}

lb2_status lb2_ivfrq_build(const void* data, uint64_t n, uint32_t d, lb2_dtype dtype, lb2_metric metric,
                           const lb2_ivfrq_build_params* params, const uint64_t* row_ids, lb2_index** out,
                           lb2_build_stats* stats) {
  LB2_API_BEGIN
  LB2_REQUIRE(data && params && out, "null argument");
  rq_check(d, dtype, params->num_bits);
  if (current_comm() && current_comm()->nranks > 1)
    fail(LB2_UNSUPPORTED, "IVF_RQ: builds sharded over ranks are not implemented");
  const int m = metric_of(metric);
  const int K = params->num_partitions;
  LB2_REQUIRE(K > 0 && n >= (uint64_t)K, "KMeans: can not train %d centroids with %llu vectors", K, (unsigned long long)n);
  EventSet ev(5);
  ev.record(0);
  Source src(data, n, (int)d, dtype);
  std::unique_ptr<lb2_index> ix(new lb2_index());
  ix->kind = 3; ix->K = K; ix->d = d; ix->M = 0; ix->nbits = (int)params->num_bits; ix->metric = m; ix->dtype = dtype;
  ix->centroids.alloc((size_t)K * d);
  const int cd = ix->code_dim();
  std::vector<double> loss;
  std::vector<uint32_t> iters;
  // 1. IVF: the same stage as lb2_ivfflat_build (same sample, seed, training)
  train_ivf_stage(src, ix.get(), params->ivf, params->seed, 1, &loss, &iters);
  ev.record(1);
  // 2. RabitQuantizer::new (bq/builder.rs:52-70): the rotation, from seed + 1
  {
    TagScope tg("rq_train");
    ix->rq_rot.alloc((size_t)cd * cd);
    rq_rotation_f32(cd, params->seed + 1, ix->rq_rot.p);
  }
  ev.record(2);
  // 3. transform (ivf.rs:281-328) of every row
  DevBuf<uint32_t> part(std::max<uint64_t>(n, 1));
  DevBuf<uint8_t> valid(std::max<uint64_t>(n, 1)), codes(std::max<uint64_t>(1, n * (cd / 8)));
  DevBuf<float> add(std::max<uint64_t>(n, 1)), scale(std::max<uint64_t>(n, 1)), cnorm;
  {
    TagScope tg("transform");
    rq_centroid_norms(m, ix->centroids.p, K, (int)d, cnorm);
    RqWork w;
    for_each_chunk(src, [&](const float* xf, const void* xnat, uint64_t r0, uint64_t rows) {
      rq_transform_chunk(xf, xnat, (int)src.dtype(), rows, (int)d, m, ix->centroids.p, K, ix->rq_rot.p, ix->nbits,
                         cnorm.p, w, part.p + r0, valid.p + r0, codes.p + r0 * (cd / 8), add.p + r0, scale.p + r0);
    });
  }
  ev.record(3);
  {
    TagScope tg("group");
    InArg<uint64_t> rid(row_ids, n);
    index_load_dev(ix.get(), part.p, codes.p, rid.get(), n, valid.p, add.p, scale.p);
  }
  ev.record(4);
  sync_stream();
  if (stats) {
    memset(stats, 0, sizeof(*stats));
    stats->ms_ivf_train = ev.ms(0, 1);
    stats->ms_pq_train = ev.ms(1, 2);
    stats->ms_transform = ev.ms(2, 3);
    stats->ms_group = ev.ms(3, 4);
    stats->ms_total = ev.ms(0, 4);
    stats->ivf_iters = iters.empty() ? 0 : iters[0];
    stats->ivf_loss = loss.empty() ? 0.0 : loss[0];
  }
  *out = ix.release();
  LB2_API_END
}

lb2_status lb2_index_create_rq(const void* centroids, uint32_t k, uint32_t d, lb2_dtype dtype, lb2_metric metric,
                               const void* rotation, uint32_t num_bits, lb2_index** out) {
  LB2_API_BEGIN
  LB2_REQUIRE(out && centroids && rotation, "null argument");
  rq_check(d, dtype, num_bits);
  std::unique_ptr<lb2_index> ix(index_with_centroids(3, centroids, k, d, dtype, metric));
  ix->nbits = (int)num_bits;
  const size_t cd = ix->code_dim();
  ix->rq_rot.alloc(cd * cd);
  VecIn r(rotation, cd * cd, dtype);
  d2d(ix->rq_rot.p, r.get(), cd * cd);
  ix->rq_add.alloc(1);
  ix->rq_scale.alloc(1);
  sync_stream();
  *out = ix.release();
  LB2_API_END
}

lb2_status lb2_index_load_rq(lb2_index* index, const uint32_t* part_ids, const uint8_t* codes, const float* add_factors,
                             const float* scale_factors, const uint64_t* row_ids, uint64_t n) {
  LB2_API_BEGIN
  LB2_REQUIRE(index && index->kind == 3, "not an IVF_RQ index");
  LB2_REQUIRE(n == 0 || (part_ids && codes && add_factors && scale_factors), "null argument");
  InArg<uint32_t> p(part_ids, n);
  InArg<uint8_t> c(codes, (size_t)n * index->code_bytes());
  InArg<float> a(add_factors, n), s(scale_factors, n);
  InArg<uint64_t> r(row_ids, n);
  check_part_ids(p.get(), n, (uint32_t)index->K, "index_load_rq");
  index_load_dev(index, p.get(), c.get(), r.get(), n, nullptr, a.get(), s.get());
  LB2_API_END
}

lb2_status lb2_index_export_rq(const lb2_index* index, void* centroids_out, void* rotation_out,
                               uint64_t* part_offsets_out, uint8_t* codes_out, float* add_out, float* scale_out,
                               uint64_t* row_ids_out) {
  LB2_API_BEGIN
  LB2_REQUIRE(index && index->kind == 3, "not an IVF_RQ index");
  cudaStream_t s = ctx().stream;
  const size_t cd = index->code_dim(), n = index->n;
  if (centroids_out)
    LB2_CUDA(cudaMemcpyAsync(centroids_out, index->centroids.p, sizeof(float) * index->K * index->d, cudaMemcpyDefault, s));
  if (rotation_out)
    LB2_CUDA(cudaMemcpyAsync(rotation_out, index->rq_rot.p, sizeof(float) * cd * cd, cudaMemcpyDefault, s));
  if (part_offsets_out)
    LB2_CUDA(cudaMemcpyAsync(part_offsets_out, index->part_offsets.p, sizeof(uint64_t) * (index->K + 1), cudaMemcpyDefault, s));
  if (codes_out && n)
    LB2_CUDA(cudaMemcpyAsync(codes_out, index->codes.p, n * index->code_bytes(), cudaMemcpyDefault, s));
  if (add_out && n) LB2_CUDA(cudaMemcpyAsync(add_out, index->rq_add.p, sizeof(float) * n, cudaMemcpyDefault, s));
  if (scale_out && n) LB2_CUDA(cudaMemcpyAsync(scale_out, index->rq_scale.p, sizeof(float) * n, cudaMemcpyDefault, s));
  if (row_ids_out && n)
    LB2_CUDA(cudaMemcpyAsync(row_ids_out, index->row_ids.p, sizeof(uint64_t) * n, cudaMemcpyDefault, s));
  sync_stream();
  LB2_API_END
}

lb2_status lb2_index_export_partition(const lb2_index* index, uint32_t partition, uint8_t* codes_transposed_out,
                                      uint64_t* row_ids_out, uint64_t* num_rows_out) {
  LB2_API_BEGIN
  LB2_REQUIRE(index && index->kind == 0, "not an IVF_PQ index");
  LB2_REQUIRE(partition < (uint32_t)index->K, "partition %u out of range (the index has %d)", partition, index->K);
  uint64_t off[2];
  d2h(off, index->part_offsets.p + partition, 2);
  sync_stream();
  const uint64_t np = off[1] - off[0];
  const int cw = index->code_bytes();
  if (num_rows_out) *num_rows_out = np;
  if (np && codes_transposed_out) {
    OutArg<uint8_t> o(codes_transposed_out, (size_t)np * cw);
    LB2_LAUNCH("transpose_codes", transpose_codes_kernel, cdiv(np * cw, 256), 256, 0, index->codes.p + off[0] * cw, np, cw, o.get());
    o.commit();
  }
  if (np && row_ids_out)
    LB2_CUDA(cudaMemcpyAsync(row_ids_out, index->row_ids.p + off[0], sizeof(uint64_t) * np, cudaMemcpyDefault, ctx().stream));
  sync_stream();
  LB2_API_END
}

lb2_status lb2_index_destroy(lb2_index* index) {
  LB2_API_BEGIN
  if (index) {
    ctx();
    delete index;
    sync_stream();
  }
  LB2_API_END
}

lb2_status lb2_ivfpq_build(const void* data, uint64_t n, uint32_t d, lb2_dtype dtype,
                           lb2_metric metric, const lb2_ivfpq_build_params* params,
                           const uint64_t* row_ids, lb2_index** out, lb2_build_stats* stats) {
  LB2_API_BEGIN
  LB2_REQUIRE(data && params && out, "null argument");
  const int m = metric_of(metric);
  const int K = params->num_partitions, M = params->pq.num_sub_vectors;
  const uint64_t nranks = current_comm() ? current_comm()->nranks : 1;  // sharded build: this rank's rows
  LB2_REQUIRE(K > 0 && (nranks > 1 || n >= (uint64_t)K), "KMeans: can not train %d centroids with %llu vectors", K,
              (unsigned long long)n);
  LB2_REQUIRE(M > 0 && d % M == 0, "num_sub_vectors must divide vector dimension %u, but got %d", d, M);
  const int nbits = (int)params->pq.num_bits;
  if (nbits != 8 && nbits != 4) fail(LB2_INVALID_ARG, "PQ: num_bits must be 4 or 8, got %d", nbits);
  LB2_REQUIRE(nbits == 8 || M % 2 == 0, "PQ: num_sub_vectors must be divisible by 2 for num_bits=4, but got %d", M);
  const int ds = d / M;
  if (!small_d_supported(ds)) fail(LB2_UNSUPPORTED, "PQ sub-vector width %d not supported yet", ds);
  EventSet ev(5);
  ev.record(0);

  // Staging (class Source).  Device rows: used in place.  Host rows: both training samples (<= K * 256 and
  // 65 536 rows) are gathered straight out of the caller's memory (zero-copy reads over PCIe when it is pinned),
  // then the matrix is copied ONCE, in its own element type, on a second stream while both trainings run; the
  // per-row pass waits for it and converts one chunk of rows at a time.  A matrix too large for that is streamed
  // chunk by chunk during the per-row pass instead (double buffered).  No whole-matrix f32 copy exists.
  // (declared before `src`: on an error path ~Source waits for the copy stream, which may still be writing the PQ
  // sample, before these buffers go back to the pool)
  DevBuf<float> sample_ivf, sample_pq;
  Source src(data, n, (int)d, dtype);
  const int am = m == METRIC_DOT ? METRIC_DOT : METRIC_L2;

  std::unique_ptr<lb2_index> ix(new lb2_index());
  ix->K = K; ix->d = d; ix->M = M; ix->nbits = nbits; ix->metric = m; ix->dtype = dtype;
  ix->centroids.alloc((size_t)K * d);
  ix->codebook.alloc(ix->codebook_len());
  std::vector<double> ivf_loss;
  std::vector<uint32_t> ivf_iters, pq_iters;
  // 0. both training samples are gathered first (IVF: K*sample_rate rows, rust/lance/src/index/
  //    vector/ivf.rs:1237-1241; PQ: 256*2^nbits rows, builder.rs:410-421), normalised for cosine; rows that are
  //    not finite are dropped from them (builder.rs:436); then the bulk copy starts
  const uint64_t s_ivf0 = std::min<uint64_t>(n, ((uint64_t)K * params->ivf.sample_rate + nranks - 1) / nranks);
  const uint64_t s_pq0 = std::min<uint64_t>(n, (params->pq.sample_rate * ((uint64_t)1 << nbits) + nranks - 1) / nranks);
  uint64_t s_ivf = 0, s_pq = 0;
  std::vector<uint64_t> rows_pq;
  bool pq_deferred = false;
  // LB2_TRACE_BUILD=1: host wall-clock stamps of the staging steps on stderr (diagnostics; adds synchronisations)
  static const bool trace = getenv("LB2_TRACE_BUILD") && *getenv("LB2_TRACE_BUILD");
  const auto tr0 = std::chrono::steady_clock::now();
  auto stamp = [&](const char* what) {
    if (!trace) return;
    sync_stream();
    fprintf(stderr, "[lb2 build] %-22s +%.3f ms\n", what,
            std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - tr0).count());
  };
  {
    std::vector<uint64_t> rows = sample_rows(n, s_ivf0, params->seed);
    stamp("sample_rows(ivf)");
    s_ivf = gather_finite_sample(src, rows, m == METRIC_COSINE, sample_ivf);
    stamp("gather(ivf sample)");
    rows_pq = sample_rows(n, s_pq0, params->seed + 1);
    // the PQ sample is not needed before the IVF model exists: from pinned f32 rows it is gathered on the copy
    // stream (in front of the bulk copy) while the IVF training runs; otherwise here
    if (m != METRIC_COSINE && !trace && !rows_pq.empty()) {
      sample_pq.alloc(rows_pq.size() * (uint64_t)d);
      pq_deferred = src.gather_f32_async(rows_pq, sample_pq.p);
    }
    if (!pq_deferred) {
      s_pq = gather_finite_sample(src, rows_pq, m == METRIC_COSINE, sample_pq);
      stamp("gather(pq sample)");
    }
  }
  LB2_REQUIRE(nranks > 1 || s_ivf >= (uint64_t)K, "KMeans: can not train %d centroids with %llu finite vectors", K,
              (unsigned long long)s_ivf);
  src.start_resident_copy();
  if (trace) fprintf(stderr, "[lb2 build] %-22s +%.3f ms (host, no sync)\n", "bulk copy issued",
                     std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - tr0).count());
  // 1. IVF
  {
    TagScope tg("ivf_train");
    VecIn init(params->ivf.init_centroids, (size_t)K * d, model_dtype(dtype));
    train_ivf(sample_ivf.p, s_ivf, d, K, am, params->ivf, nranks, init.get(), ix->centroids.p, &ivf_loss, &ivf_iters);
    round_model(ix->centroids.p, (size_t)K * d, dtype);
  }
  stamp("ivf trained");
  if (pq_deferred) {
    if (src.finish_async_sample()) {
      s_pq = rows_pq.size();
    } else {  // rare: some sampled rows are not finite -> the synchronous path drops them and gathers again
      s_pq = gather_finite_sample(src, rows_pq, false, sample_pq);
    }
  }
  sample_ivf.release();
  ev.record(1);
  // 2. PQ: residuals of its sample w.r.t. the IVF centroids (builder.rs:439-450)
  {
    TagScope tg("pq_train");
    if (am == METRIC_L2 && s_pq) {
      DevBuf<uint32_t> part(s_pq);
      assign_f32(sample_pq.p, s_pq, d, ix->centroids.p, K, METRIC_L2, nullptr, part.p, nullptr, nullptr, nullptr);
      LB2_LAUNCH("residual", residual_kernel, cdiv(s_pq * d, 256), 256, 0, sample_pq.p, ix->centroids.p,
                 part.p, s_pq, (int)d, sample_pq.p);
    }
    VecIn cb_init(params->pq.codebook, ix->codebook_len(), model_dtype(dtype));
    lb2_pq_params pqp = params->pq;
    pqp.codebook = cb_init.get();
    // always L2 k-means (builder.rs:460: Q::build(&training_data, DistanceType::L2, ..)); for a dot index
    // the sample is the raw vectors (no residual), for L2 / cosine the residuals computed above
    pq_train_dev(sample_pq.p, s_pq, d, METRIC_L2, &pqp, ix->codebook.p, &pq_iters);
    round_model(ix->codebook.p, ix->codebook_len(), dtype);
  }
  sample_pq.release();
  ev.record(2);
  // 3. transform every row (lance-index/src/vector/ivf.rs:357: partition -> residual -> PQ), chunk by chunk
  DevBuf<uint32_t> part(std::max<uint64_t>(n, 1));
  DevBuf<uint8_t> codes(std::max<uint64_t>(1, (size_t)n * ix->code_bytes())), valid(std::max<uint64_t>(n, 1));
  {
    TagScope tg("transform");
    DevBuf<float> normbuf;
    const size_t cw = ix->code_bytes();
    for_each_chunk(src, [&](const float* xf, const void* xnat, uint64_t r0, uint64_t rows) {
      transform_chunk(xf, xnat, (int)src.dtype(), rows, (int)d, m, ix->centroids.p, K, ix->codebook.p, M, nbits, normbuf,
                      part.p + r0, codes.p + r0 * cw, valid.p + r0);
    });
  }
  ev.record(3);
  {
    // 4. group the kept rows by partition (shuffle + build_partitions, builder.rs:501-937); rows the
    //    transform marked invalid are dropped, as KeepFiniteVectors does (transform.rs:112-159)
    TagScope tg("group");
    InArg<uint64_t> rid(row_ids, n);
    index_load_dev(ix.get(), part.p, codes.p, rid.get(), n, valid.p);
  }
  ev.record(4);
  sync_stream();
  if (stats) {
    stats->ms_ivf_train = ev.ms(0, 1);
    stats->ms_pq_train = ev.ms(1, 2);
    stats->ms_transform = ev.ms(2, 3);
    stats->ms_group = ev.ms(3, 4);
    stats->ms_total = ev.ms(0, 4);
    stats->ivf_iters = ivf_iters.empty() ? 0 : ivf_iters[0];
    stats->pq_iters_max = 0;
    for (auto v : pq_iters) stats->pq_iters_max = std::max(stats->pq_iters_max, v);
    stats->ivf_loss = ivf_loss.empty() ? 0.0 : ivf_loss[0];
  }
  *out = ix.release();
  LB2_API_END
}

}  // extern "C"
