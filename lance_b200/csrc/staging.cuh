// staging.cuh -- a caller's vectors on the device: element-type conversion (VecIn / VecOut), the host staging of a
// whole matrix (class Source), training samples and the chunked per-row pass.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <algorithm>
#include <cstdlib>

#include "common.cuh"
#include "exact.cuh"

namespace lb2 {

// ---- element types ---------------------------------------------------------------------------------
// f16 / bf16 / u8 buffers are converted to f32 on the device at the boundary and every loop runs
// with the reference's f32 semantics (what the reference itself does for Int8 vectors,
// rust/lance/src/index/vector/ivf.rs:1917-1929; its f16 paths accumulate in f16 / use a -ffast-math
// C kernel, so for f16 inputs parity with the reference is by tolerance, see DESIGN.md).
// Model outputs (centroids, codebook, residuals, normalised vectors) use the input's element type,
// except for u8 inputs, whose model is f32.
inline size_t dtype_size(lb2_dtype dt) { return dt == LB2_F32 ? 4 : (dt == LB2_U8 ? 1 : 2); }
inline lb2_dtype model_dtype(lb2_dtype dt) { return dt == LB2_U8 ? LB2_F32 : dt; }
inline int metric_of(lb2_metric m) {
  switch (m) {
    case LB2_L2: return METRIC_L2;
    case LB2_COSINE: return METRIC_COSINE;
    case LB2_DOT: return METRIC_DOT;
  }
  fail(LB2_INVALID_ARG, "unknown metric %d", (int)m);
}

__global__ void to_f32_kernel(const void* __restrict__ in, int dt, size_t count, float* __restrict__ out);
__global__ void from_f32_kernel(const float* __restrict__ in, int dt, size_t count, void* __restrict__ out);
__global__ void gather_rows_typed_kernel(const void* __restrict__ x, int dt, const uint64_t* __restrict__ rows,
                                         uint64_t s, int d, float* __restrict__ out);
__global__ void gather_rows_f32x4_kernel(const float4* __restrict__ x, const uint64_t* __restrict__ rows, uint64_t s,
                                         int d4, float4* __restrict__ out);
__global__ void finite_rows_kernel(const float* __restrict__ x, uint64_t n, int d, uint8_t* __restrict__ flag,
                                   int clear_only);

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

void round_model(float* v, size_t count, lb2_dtype dt);
// the rows of x [n][d] divided by their norms (x and out may be the same buffer); nothing for n == 0
void normalize_rows(const float* x, uint64_t n, int d, float* out);

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
extern thread_local std::map<int, StagingCache> g_staging;
inline size_t staging_cache_cap() {
  static const size_t cap = [] {
    const char* e = getenv("LB2_STAGING_CACHE_MB");
    return (size_t)(e && *e ? strtoull(e, nullptr, 10) : 1024ull) << 20;
  }();
  return cap;
}
void staging_cache_release();  // the calling thread's cache on the current device

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
    finite_rows_kernel<<<(unsigned)cdiv(s * 32, 256), 256, 0, cs>>>(out, s, d_, async_flag_.p, 0);
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
  // Decided once: a later call does nothing.
  void start_resident_copy() {
    if (dev_native_ || n_ == 0 || copy_decided_) return;
    copy_decided_ = true;
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
  bool copy_decided_ = false;       // start_resident_copy() has run
  uint64_t calls_ = 0;
};

uint64_t gather_finite_sample(Source& src, std::vector<uint64_t>& rows, bool normalize, DevBuf<float>& out);
std::vector<uint64_t> sample_rows(uint64_t n, uint64_t s, uint64_t seed);

// the rows per call of for_each_chunk (a little more than one chunk is not split: SIFT-1M is one call)
inline uint64_t chunk_step(const Source& src) {
  const uint64_t n = src.n(), chunk = src.rows_per_chunk();
  return n <= chunk + chunk / 2 ? std::max<uint64_t>(n, 1) : chunk;
}

// one pass over a caller's matrix in chunks of rows: f(xf, xnat, r0, rows) with xf = the chunk as f32 on the device
// and xnat = the same rows in the column's own type (for assign_f32: tc_assign.cu, "native 16-bit rows")
template <class F>
void for_each_chunk(Source& src, F&& f) {
  const uint64_t n = src.n(), step = chunk_step(src);
  for (uint64_t r0 = 0; r0 < n; r0 += step) {
    const uint64_t rows = std::min(step, n - r0);
    const float* xf = src.rows_f32(r0, rows);
    if (r0 + rows < n) src.prefetch(r0 + rows, std::min(step, n - r0 - rows));
    f(xf, src.last_native(), r0, rows);
  }
}

}  // namespace lb2
