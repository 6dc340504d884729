// api.cu -- the per-thread runtime behind the extern "C" surface declared in include/lance_b200.h (context, device,
// stream, memory, profiling, timer) and the stand-alone primitives: distances, normalisation, k-means, partitions,
// residuals, PQ train / encode / tables / scans, flat top-k, SQ train / encode and the RQ rotation.  The index handle
// lives in index.cu, the whole-index builds in build.cu.
#include <algorithm>

#include "assign.cuh"
#include "build.cuh"
#include "comm.cuh"
#include "common.cuh"
#include "exact.cuh"
#include "flat_search.cuh"
#include "index.cuh"
#include "ivf_search.cuh"
#include "kmeans.cuh"
#include "row_distance.cuh"
#include "rq.cuh"
#include "scan.cuh"
#include "sq.cuh"
#include "staging.cuh"
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


// cosine_distance_batch (cosine.rs:143-174,266-290): 1 - xy / |x| / sqrt(yy) with f32 FMA lanes; the
// reference's own lane order is ISA specific, so parity is the reference's tolerance (cosine.rs:361-393)
__global__ void cosine_f32_kernel(const float* __restrict__ from, const float* __restrict__ to, uint64_t n, int d,
                                  float* __restrict__ out) {
  const uint64_t w = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= n) return;
  float xx, xy, yy;
  cos32_sums(from, to + w * d, d, lane, xx, xy, yy);
  if (lane == 0) out[w] = cos32_finish(xy, xx, yy);
}

}  // namespace lb2

using namespace lb2;

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
  p->partition_index = LB2_PARTITION_INDEX_EXACT;
  p->partition_index_batch = 1;
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

lb2_status lb2_distance_batch(const void* from, const void* to, uint64_t n, uint32_t d,
                              lb2_dtype dtype, lb2_metric metric, float* out) {
  LB2_API_BEGIN
  const int m = metric_of(metric);
  LB2_REQUIRE(d > 0, "dimension must be positive");
  LB2_REQUIRE(n < (1ull << 31), "too many rows");
  OutArg<float> o(out, n);
  VecIn f(from, d, dtype);
  // the reference picks the arithmetic by element type: u8 sums are exact integers, 16-bit dot products take 32
  // lanes; the rows are read in their own type
  if (distance_batch_typed_applies(dtype, m)) {
    InArg<uint8_t> t(to, (size_t)n * d * dtype_size(dtype));
    distance_batch_typed(f.get(), t.get(), dtype, n, (int)d, m, o.get());
    o.commit();
    sync_stream();
    return LB2_OK;
  }
  VecIn t(to, (size_t)n * d, dtype);
  if (m == METRIC_COSINE) {
    if (n) LB2_LAUNCH("cosine_batch", cosine_f32_kernel, cdiv(n * 32, 256), 256, 0, f.get(), t.get(), n, (int)d, o.get());
    o.commit();
    sync_stream();
    return LB2_OK;
  }
  // f32 L2 / dot and 16-bit L2 (each element converted, l2.rs:100-106): the 16-lane f32 loop of the assignment
  // kernels, `from` as the one row and `to` as n centroids (none for n == 0: the tile kernel cannot lay out an empty
  // centroid matrix)
  if (n) centroid_distances(f.get(), 1, d, t.get(), (int)n, m, o.get());
  o.commit();
  sync_stream();
  LB2_API_END
}

lb2_status lb2_normalize(const void* vectors, uint64_t n, uint32_t d, lb2_dtype dtype, void* out) {
  LB2_API_BEGIN
  VecIn x(vectors, (size_t)n * d, dtype);
  VecOut o(out, (size_t)n * d, model_dtype(dtype));
  normalize_rows(x.get(), n, (int)d, o.get());
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
  if (params->partition_index != LB2_PARTITION_INDEX_EXACT)
    fail(LB2_INVALID_ARG, "KMeans: training never assigns through a partition index (partition_index must be EXACT)");
  const int m = metric_of(params->metric);
  if (m == METRIC_COSINE)
    fail(LB2_INVALID_ARG, "KMeans: cosine is trained as L2 on normalised vectors (normalise first)");
  LB2_REQUIRE(current_comm() || n >= k, "KMeans: can not train %u centroids with %llu vectors, choose a smaller K (< %llu) instead",
              k, (unsigned long long)n, (unsigned long long)n);
  // free fn train_kmeans (kmeans.rs:1328-1344); sharded: every rank contributes its share of the cap
  const uint64_t nranks = comm_nranks();
  const uint64_t cap = (params->sample_rate * k + nranks - 1) / nranks;
  const uint64_t rows = n > cap ? cap : n;
  VecIn x(data, (size_t)rows * d, dtype);
  VecIn init(params->init_centroids, (size_t)k * d, model_dtype(dtype));
  DevBuf<float> cent((size_t)k * d);
  std::vector<double> loss;
  std::vector<uint32_t> iters;
  train_kmeans(x.get(), rows, d, k, m, *params, init.get(), cent.p, &loss, &iters);
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
                 v.get() ? v.get() + r0 : nullptr, xnat, (int)src.dtype());
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
  LB2_REQUIRE((centroids == nullptr) == (part_ids == nullptr),
              "centroids and part_ids must be given together");
  LB2_REQUIRE(centroids == nullptr || num_centroids > 0, "num_centroids must be given with centroids");
  const int m = metric_of(metric) == METRIC_DOT ? METRIC_DOT : METRIC_L2;
  check_pq_shape(d, num_sub_vectors, num_bits, PqUse::ENCODE);
  const int M = num_sub_vectors, ds = d / M;
  const int ncode = 1 << num_bits;
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

lb2_status lb2_flat_search(const void* vectors, uint64_t n, uint32_t d, lb2_dtype dtype, lb2_metric metric,
                           const uint64_t* row_ids, const void* queries, uint64_t nq, const lb2_flat_search_params* p,
                           uint64_t* row_ids_out, float* dists_out, uint32_t* counts_out) {
  LB2_API_BEGIN
  LB2_REQUIRE(p, "null flat search params");
  LB2_REQUIRE(p->k > 0, "k must be positive");
  LB2_REQUIRE(d > 0, "dimension must be positive");
  LB2_REQUIRE(dtype >= LB2_F32 && dtype <= LB2_U8, "unknown element type %d", (int)dtype);
  LB2_REQUIRE((n == 0 || vectors) && (nq == 0 || queries) && (nq == 0 || (row_ids_out && dists_out)), "null argument");
  const int m = metric_of(metric);
  flat_search_check((int)d, dtype, m, (int)std::min<uint32_t>(p->k, 1025));
  VecIn q(queries, (size_t)nq * d, dtype);
  InArg<uint64_t> rid(row_ids, n), allow(p->allow_bitmap, p->allow_bitmap ? (size_t)((n + 63) / 64) : 0);
  OutArg<uint64_t> oi(row_ids_out, (size_t)nq * p->k);
  OutArg<float> od(dists_out, (size_t)nq * p->k);
  OutArg<uint32_t> oc(counts_out, nq);
  FlatFilter flt;
  flt.allow = allow.get();
  flt.has_lower = p->has_lower_bound != 0;
  flt.has_upper = p->has_upper_bound != 0;
  flt.lower = p->lower_bound;
  flt.upper = p->upper_bound;
  flat_search(q.get(), nq, (int)d, m, vectors, n, dtype, rid.get(), flt, (int)p->k, oi.get(), od.get(), oc.get());
  oi.commit(); od.commit(); oc.commit();
  sync_stream();
  LB2_API_END
}

// Every query is checked first, so a refusal writes nothing; each bitmap is staged once.
lb2_status lb2_flat_search_batch(const void* vectors, uint64_t n, uint32_t d, lb2_dtype dtype, lb2_metric metric,
                                 const uint64_t* row_ids, const void* queries, uint64_t nq,
                                 const lb2_flat_query_params* params, const uint64_t* const* filter_bitmaps,
                                 uint32_t num_filters, uint32_t k_stride, uint64_t* row_ids_out, float* dists_out,
                                 uint32_t* counts_out) {
  LB2_API_BEGIN
  LB2_REQUIRE(d > 0, "dimension must be positive");
  LB2_REQUIRE(dtype >= LB2_F32 && dtype <= LB2_U8, "unknown element type %d", (int)dtype);
  LB2_REQUIRE((n == 0 || vectors) && (nq == 0 || (queries && params && row_ids_out && dists_out)), "null argument");
  LB2_REQUIRE(num_filters == 0 || filter_bitmaps, "null filter_bitmaps");
  const int m = metric_of(metric);
  uint32_t kmax = 0;
  for (uint64_t q = 0; q < nq; ++q) {
    const lb2_flat_query_params& p = params[q];
    const unsigned long long qi = (unsigned long long)q;
    LB2_REQUIRE(p.k > 0, "query %llu: k must be positive", qi);
    if (p.k > 1024) fail(LB2_UNSUPPORTED, "query %llu: k = %u > 1024 is not implemented", qi, p.k);
    LB2_REQUIRE(p.filter < num_filters || p.filter == UINT32_MAX, "query %llu: filter %u is not below num_filters %u",
                qi, p.filter, num_filters);
    kmax = std::max(kmax, p.k);
  }
  LB2_REQUIRE(k_stride >= kmax, "k_stride %u is below the largest k %u", k_stride, kmax);
  flat_search_batch_check((int)d, dtype, m, (int)std::max<uint32_t>(kmax, 1));
  if (nq == 0) {
    sync_stream();
    return LB2_OK;
  }
  VecIn q(queries, (size_t)nq * d, dtype);
  InArg<uint64_t> rid(row_ids, n);
  std::vector<InArg<uint64_t>> bm(num_filters);
  std::vector<const uint64_t*> bm_dev(num_filters);
  for (uint32_t f = 0; f < num_filters; ++f) {
    bm[f].set(filter_bitmaps[f], filter_bitmaps[f] ? (size_t)((n + 63) / 64) : 0);
    bm_dev[f] = bm[f].get();
  }
  const std::vector<FlatQuery> fq = flat_queries(params, nq, bm_dev, nullptr);
  OutArg<uint64_t> oi(row_ids_out, (size_t)nq * k_stride);
  OutArg<float> od(dists_out, (size_t)nq * k_stride);
  OutArg<uint32_t> oc(counts_out, nq);
  flat_search_batch(q.get(), nq, (int)d, m, vectors, n, dtype, rid.get(), fq.data(), (int)k_stride, oi.get(), od.get(),
                    oc.get());
  oi.commit(); od.commit(); oc.commit();
  sync_stream();
  LB2_API_END
}

lb2_status lb2_comm_info(int* rank, int* nranks) {
  LB2_API_BEGIN
  Comm* c = current_comm();
  if (rank) *rank = c ? c->rank : 0;
  if (nranks) *nranks = c ? c->nranks : 1;
  LB2_API_END
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

}  // extern "C"
