// common.cuh -- runtime plumbing shared by every translation unit of liblance_b200.so:
// status/error reporting, per-thread device context (stream, launch counter, per-kernel event
// profiling), RAII device buffers and host<->device staging of caller pointers.
#pragma once
#include <cuda_runtime.h>

#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <map>
#include <mutex>
#include <new>
#include <string>
#include <vector>

#include "../../include/lance_b200.h"

namespace lb2 {

// ------------------------------------------------------------------------------------------
// errors: never throw across the C boundary.  Internally we throw Err and catch in LB2_API_*.
// ------------------------------------------------------------------------------------------
struct Err {
  lb2_status st;
  std::string msg;
};
void set_last_error(const std::string& m);

[[noreturn]] inline void fail(lb2_status st, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  throw Err{st, buf};
}

#define LB2_CUDA(expr)                                                                          \
  do {                                                                                          \
    cudaError_t _e = (expr);                                                                    \
    if (_e != cudaSuccess) {                                                                    \
      cudaGetLastError();                                                                       \
      ::lb2::fail(_e == cudaErrorMemoryAllocation ? LB2_OOM : LB2_CUDA_ERROR, "%s:%d: %s -> %s", \
                  __FILE__, __LINE__, #expr, cudaGetErrorString(_e));                           \
    }                                                                                           \
  } while (0)

#define LB2_REQUIRE(cond, ...)                                \
  do {                                                        \
    if (!(cond)) ::lb2::fail(LB2_INVALID_ARG, __VA_ARGS__);   \
  } while (0)

#define LB2_API_BEGIN try {
#define LB2_API_END                                   \
  return LB2_OK;                                      \
  }                                                   \
  catch (const ::lb2::Err& e) {                       \
    ::lb2::set_last_error(e.msg);                     \
    return e.st;                                      \
  }                                                   \
  catch (const std::bad_alloc&) {                     \
    ::lb2::set_last_error("host out of memory");      \
    return LB2_OOM;                                   \
  }                                                   \
  catch (...) {                                       \
    ::lb2::set_last_error("unknown internal error");  \
    return LB2_CUDA_ERROR;                            \
  }

// ------------------------------------------------------------------------------------------
// per-thread context
// ------------------------------------------------------------------------------------------
struct ProfEntry {
  uint64_t launches = 0;
  double total_ms = 0.0;
};

struct Ctx {
  int device = -1;
  cudaStream_t stream = nullptr;      // where work is enqueued: own_stream, or the caller's (lb2_set_stream / _async)
  cudaStream_t own_stream = nullptr;  // the thread's private non-blocking stream
  bool async_call = false;            // inside an _async entry point: the trailing synchronise is skipped
  uint64_t launches = 0;
  bool profiling = false;
  std::string tag;  // phase prefix of the profile key: "ivf_train", "pq_train", "transform", "search" ...
  std::map<std::string, ProfEntry> prof;
  std::vector<std::pair<std::string, std::pair<cudaEvent_t, cudaEvent_t>>> pending;
  cudaEvent_t t0 = nullptr, t1 = nullptr;
  int num_sms = 132;
  size_t smem_optin = 0;
  void flush_profile();
};
Ctx& ctx();  // initialises the device/stream lazily; throws LB2_NO_DEVICE without a GPU

// kernel launch wrapper: counts launches, optional per-kernel-family CUDA-event timing.
struct LaunchScope {
  Ctx& c;
  const char* name;
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  LaunchScope(const char* n) : c(ctx()), name(n) {
    c.launches++;
    if (c.profiling) {
      cudaEventCreate(&e0);
      cudaEventCreate(&e1);
      cudaEventRecord(e0, c.stream);
    }
  }
  ~LaunchScope() {
    if (c.profiling) {
      cudaEventRecord(e1, c.stream);
      c.pending.push_back({c.tag.empty() ? std::string(name) : c.tag + ":" + name, {e0, e1}});
    }
  }
};
#define LB2_LAUNCH(name, kernel, grid, block, smem, ...)                              \
  do {                                                                                \
    ::lb2::LaunchScope _ls(name);                                                     \
    kernel<<<(grid), (block), (smem), ::lb2::ctx().stream>>>(__VA_ARGS__);            \
    cudaError_t _le = cudaGetLastError();                                             \
    if (_le != cudaSuccess)                                                           \
      ::lb2::fail(LB2_CUDA_ERROR, "launch %s failed: %s", name, cudaGetErrorString(_le)); \
  } while (0)

// The limit is an attribute of the kernel, shared by every host thread: hierarchical training's split workers
// launch the same kernel with different sizes at once, so the limit only ever rises (under a lock, set before
// any launch that relies on it) -- lowering it could make another thread's launch fail with "invalid argument".
template <class K>
inline void set_smem(K kernel, size_t bytes) {
  if (bytes <= 32 * 1024) return;  // static shared memory counts against the 48 KB default as well
  static std::mutex mu;
  static std::map<std::pair<int, const void*>, size_t> limit;  // (device, kernel) -> limit set so far
  std::lock_guard<std::mutex> lk(mu);
  size_t& cur = limit[{ctx().device, reinterpret_cast<const void*>(kernel)}];
  if (bytes <= cur) return;
  LB2_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
  cur = bytes;
}
// the shared memory a launch of `kernel` with `dyn` dynamic bytes takes: its static shared memory counts against the
// same per-block opt-in limit, and cudaFuncSetAttribute refuses a dynamic size that leaves no room for it
template <class Kern>
size_t smem_with_static(Kern kernel, size_t dyn) {
  cudaFuncAttributes fa;
  LB2_CUDA(cudaFuncGetAttributes(&fa, kernel));
  return dyn + fa.sharedSizeBytes;
}

// ------------------------------------------------------------------------------------------
// memory
// ------------------------------------------------------------------------------------------
template <class T>
struct DevBuf {
  T* p = nullptr;
  size_t n = 0;
  DevBuf() = default;
  explicit DevBuf(size_t count) { alloc(count); }
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  DevBuf(DevBuf&& o) noexcept : p(o.p), n(o.n) { o.p = nullptr; o.n = 0; }
  DevBuf& operator=(DevBuf&& o) noexcept {
    if (this != &o) {
      release();
      p = o.p; n = o.n; o.p = nullptr; o.n = 0;
    }
    return *this;
  }
  ~DevBuf() { release(); }
  void alloc(size_t count) {
    release();
    n = count;
    if (count) LB2_CUDA(cudaMallocAsync((void**)&p, count * sizeof(T), ctx().stream));
  }
  void release() {
    if (p) cudaFreeAsync(p, ctx().stream);
    p = nullptr;
    n = 0;
  }
  void zero() { if (n) LB2_CUDA(cudaMemsetAsync(p, 0, n * sizeof(T), ctx().stream)); }
  T* get() const { return p; }
};

bool is_device_ptr(const void* p);

// Input staging: device pointers pass through; host pointers are copied to a temp device buffer.
template <class T>
struct InArg {
  const T* dev = nullptr;
  DevBuf<T> tmp;
  InArg() = default;
  InArg(const void* p, size_t count) { set(p, count); }
  void set(const void* p, size_t count) {
    if (p == nullptr || count == 0) { dev = nullptr; return; }
    if (is_device_ptr(p)) { dev = (const T*)p; return; }
    tmp.alloc(count);
    LB2_CUDA(cudaMemcpyAsync(tmp.p, p, count * sizeof(T), cudaMemcpyHostToDevice, ctx().stream));
    dev = tmp.p;
  }
  const T* get() const { return dev; }
};
// Output staging: device pointers are written in place; host pointers get a temp that is copied
// back by commit() (which also synchronises the stream -> blocking call semantics).
template <class T>
struct OutArg {
  T* dev = nullptr;
  void* host = nullptr;
  size_t count = 0;
  DevBuf<T> tmp;
  OutArg() = default;
  OutArg(void* p, size_t c) { set(p, c); }
  void set(void* p, size_t c) {
    count = c;
    if (p == nullptr || c == 0) { dev = nullptr; return; }
    if (is_device_ptr(p)) { dev = (T*)p; return; }
    host = p;
    tmp.alloc(c);
    dev = tmp.p;
  }
  T* get() const { return dev; }
  void commit() {
    if (host && count)
      LB2_CUDA(cudaMemcpyAsync(host, tmp.p, count * sizeof(T), cudaMemcpyDeviceToHost, ctx().stream));
  }
};
inline void sync_stream() { LB2_CUDA(cudaStreamSynchronize(ctx().stream)); }

template <class T>
inline void d2h(T* host, const T* dev, size_t count) {
  LB2_CUDA(cudaMemcpyAsync(host, dev, count * sizeof(T), cudaMemcpyDeviceToHost, ctx().stream));
}
template <class T>
inline void h2d(T* dev, const T* host, size_t count) {
  LB2_CUDA(cudaMemcpyAsync(dev, host, count * sizeof(T), cudaMemcpyHostToDevice, ctx().stream));
}
template <class T>
inline void d2d(T* dst, const T* src, size_t count) {
  LB2_CUDA(cudaMemcpyAsync(dst, src, count * sizeof(T), cudaMemcpyDeviceToDevice, ctx().stream));
}

struct TagScope {
  std::string prev;
  explicit TagScope(const char* t) : prev(ctx().tag) { ctx().tag = t; }
  ~TagScope() { ctx().tag = prev; }
};

inline unsigned cdiv(uint64_t a, uint64_t b) { return (unsigned)((a + b - 1) / b); }

// v is one of the n ascending values of a
__device__ __forceinline__ bool sorted_contains(const uint64_t* __restrict__ a, uint64_t n, uint64_t v) {
  uint64_t lo = 0, hi = n;
  while (lo < hi) {
    const uint64_t mid = (lo + hi) >> 1;
    if (a[mid] < v) lo = mid + 1; else hi = mid;
  }
  return lo < n && a[lo] == v;
}

// the last p < n with offsets[p] <= i (offsets ascending from offsets[0] <= i): the segment holding i, empty
// segments skipped
__device__ __forceinline__ int segment_of(const uint64_t* __restrict__ offsets, int n, uint64_t i) {
  int lo = 0, hi = n;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (offsets[mid] <= i) lo = mid; else hi = mid;
  }
  return lo;
}

// our reproducible rng (the reference's is unseeded: kmeans.rs:181,645)
struct SplitMix64 {
  uint64_t s;
  explicit SplitMix64(uint64_t seed) : s(seed) {}
  uint64_t next() {
    uint64_t z = (s += 0x9E3779B97F4A7C15ull);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
  }
  float next_f32() { return float(next() >> 40) * (1.0f / 16777216.0f); }
};

}  // namespace lb2
