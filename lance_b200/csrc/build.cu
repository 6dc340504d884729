// build.cu -- the whole-index builds (IVF_PQ, IVF_FLAT, IVF_SQ, IVF_RQ), their training stages and the per-row
// transforms they share with lb2_ivfpq_transform / lb2_ivfrq_transform.
#include <chrono>
#include <memory>

#include "assign.cuh"
#include "build.cuh"
#include "comm.cuh"
#include "hnsw.cuh"
#include "index.cuh"
#include "kmeans.cuh"
#include "rq.cuh"
#include "scan.cuh"
#include "sq.cuh"
#include "tc_assign.cuh"
#include "tc_pq.cuh"

namespace lb2 {

__global__ void residual_kernel(const float* x, const float* __restrict__ cent,
                                const uint32_t* __restrict__ part, uint64_t n, int d, float* out) {
  const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n * d) return;
  const uint64_t r = g / d;
  const int t = g % d;
  out[g] = __fsub_rn(x[g], cent[(size_t)part[r] * d + t]);  // residual.rs:93
}

void check_pq_shape(uint32_t d, uint32_t M, uint32_t nbits, PqUse use) {
  LB2_REQUIRE(M > 0 && d % M == 0, "num_sub_vectors must divide vector dimension %u, but got %u", d, M);
  if (nbits != 8 && nbits != 4)  // pq/builder.rs: only 4 and 8 exist in the reference
    fail(LB2_INVALID_ARG, "PQ: num_bits must be 4 or 8, got %u", nbits);
  if (use == PqUse::TRAIN) return;
  LB2_REQUIRE(nbits == 8 || M % 2 == 0, "PQ: num_sub_vectors must be divisible by 2 for num_bits=4, but got %u", M);
}

// ProductQuantizer::transform_impl for either code width (pq.rs:116-191): 8-bit -> [n][M] through the
// tensor path where it applies; 4-bit -> 16 codewords per sub-space, exact kernel, two codes per byte
void pq_encode_any(const float* x, uint64_t n, int d, int M, int ds, const float* codebook, int metric,
                   const float* cent, const uint32_t* part, const uint8_t* row_valid, int nbits, uint8_t* codes) {
  if (nbits == 8) {
    pq_encode_dev(x, n, d, M, ds, codebook, metric, cent, part, row_valid, codes);
    return;
  }
  if (n == 0) return;
  DevBuf<uint8_t> wide((size_t)n * M);
  pq_assign_f32(x, n, d, M, ds, codebook, 16, metric, cent, part, row_valid, wide.p, nullptr, nullptr, nullptr,
                nullptr);
  pack_nibbles(wide.p, n, M, codes);
  sync_stream();  // `wide` is freed on return
}

// KMeansParams::redos (kmeans.rs:643-716).  Every redo starts from `rng.clone()` of the same generator
// (kmeans.rs:645-653), i.e. from the SAME initial centroids; the only state carried from one redo to the
// next is cluster_sizes / adjusted_balance_factor, which only enter through the balance bias.  With
// balance_factor == 0 (every PQ codebook, pq/builder.rs:100) all redos are therefore identical and
// "best of redos" is the single run; with a balance bias the redo loop is not implemented -> UNSUPPORTED.
void check_redos(uint32_t redos, float balance_factor) {
  if (redos == 0) fail(LB2_INVALID_ARG, "KMeans: redos must be at least 1");
  if (redos > 1 && balance_factor != 0.0f)
    fail(LB2_UNSUPPORTED, "KMeans: redos = %u with a balance factor is not implemented (redos = 1 only)", redos);
}

void pq_train_dev(const float* data, uint64_t n, int d, int metric, const lb2_pq_params* p, float* codebook,
                  std::vector<uint32_t>* iters) {
  const int M = p->num_sub_vectors, K = 1 << p->num_bits;
  check_pq_shape(d, M, p->num_bits, PqUse::TRAIN);
  check_redos(p->kmeans_redos, 0.0f);
  LB2_REQUIRE(current_comm() || n >= (uint64_t)K, "Not enough rows to train PQ. Requires %d rows but only %llu available",
              K, (unsigned long long)n);
  // free fn train_kmeans (kmeans.rs:1328-1340): first sample_rate*k rows (per-rank share when sharded)
  const uint64_t nranks = comm_nranks();
  const uint64_t cap = (p->sample_rate * K + nranks - 1) / nranks;
  const uint64_t rows = n > cap ? cap : n;
  InArg<float> init(p->codebook, (size_t)M * K * (d / M));
  const LloydParams lp{metric == METRIC_DOT ? METRIC_DOT : METRIC_L2, 0.0f, (int)p->max_iters, 1e-4, p->seed};
  lloyd_train(data, rows, d, M, d / M, K, lp, init.get(), codebook, nullptr, iters);
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
// KMeans::new_with_params on the IVF training sample (train_kmeans).  Sharded build: the hierarchical tree is
// thousands of small dependent Lloyd runs -- with a collective in every iteration it is latency-bound on the exchange.
// The sample (K * sample_rate rows) is small next to the data, so when it fits every rank gathers ALL sample shards
// (rank order) and trains the same tree on them without a communicator: identical arithmetic on identical input gives
// bit-identical models on all ranks, and the splits train concurrently (kmeans.cu: SplitWorkers).  Otherwise: the
// sharded tree.
void train_ivf(const float* xs, uint64_t s, int d, int K, int am, const lb2_kmeans_params& kp, const float* init,
               float* centroids, std::vector<double>* loss, std::vector<uint32_t>* iters) {
  check_redos(kp.redos, kp.balance_factor);
  const uint64_t nranks = comm_nranks();
  if (nranks > 1 && kmeans_uses_tree(K, kp, init)) {
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
        train_kmeans(all.p, total, d, K, am, kp, init, centroids, loss, iters);
      } catch (...) {
        comm_swap(saved);
        throw;
      }
      comm_swap(saved);
      return;
    }
  }
  train_kmeans(xs, s, d, K, am, kp, init, centroids, loss, iters);
}
}  // namespace

// The IVF stage of every build, in two halves so that IVF_PQ can gather its own sample in between (build_index):
// (a) the IVF training sample's rows (ivf.rs:1237-1241), to be gathered with gather_finite_sample (rows that are not
// finite dropped, normalised first under cosine);
static std::vector<uint64_t> ivf_sample_rows(uint64_t n, int K, const lb2_kmeans_params& kp, uint64_t seed) {
  const uint64_t nranks = comm_nranks();  // sharded build: this rank's share
  return sample_rows(n, std::min<uint64_t>(n, ((uint64_t)K * kp.sample_rate + nranks - 1) / nranks), seed);
}
// (b) after the caller started the bulk copy: train on the s gathered rows, centroids rounded to the column's type
static void train_ivf_model(const float* sample, uint64_t s, lb2_index* ix, const lb2_kmeans_params& kp,
                            std::vector<double>* loss, std::vector<uint32_t>* iters) {
  const int K = ix->K, d = ix->d;
  LB2_REQUIRE(comm_nranks() > 1 || s >= (uint64_t)K, "KMeans: can not train %d centroids with %llu finite vectors", K,
              (unsigned long long)s);
  TagScope tg("ivf_train");
  VecIn init(kp.init_centroids, (size_t)K * d, model_dtype(ix->dtype));
  train_ivf(sample, s, d, K, ix->metric == METRIC_DOT ? METRIC_DOT : METRIC_L2, kp, init.get(), ix->centroids.p, loss,
            iters);
  round_model(ix->centroids.p, (size_t)K * d, ix->dtype);
}
// IvfTransformer's partition step over one chunk of rows (ivf.rs:158-166): normalised first under cosine, then
// assigned through the index's partition rule -- its partition index when it has one (PartitionTransformer's graph
// arm, ivf/transform.rs:112-124), else the exact scan (by dot or L2) from f32, or from the rows' own type (xnat /
// dtype, for_each_chunk) when not normalised.  Returns the chunk as the index sees it.
static const float* normalize_assign(const lb2_index& ix, const float* xf, const void* xnat, int dtype, uint64_t rows,
                                     DevBuf<float>& normbuf, uint32_t* part, uint8_t* valid, float* dist) {
  const int d = ix.d, m = ix.metric;
  const float* xp = xf;
  if (m == METRIC_COSINE) {
    if (normbuf.n < (size_t)rows * d) normbuf.alloc((size_t)rows * d);
    normalize_rows(xf, rows, d, normbuf.p);
    xp = normbuf.p;
    xnat = nullptr;
  }
  if (ix.pidx)
    partition_index_assign(*ix.pidx, xp, rows, part, dist, valid);
  else
    assign_f32(xp, rows, d, ix.centroids.p, ix.K, m == METRIC_DOT ? METRIC_DOT : METRIC_L2, nullptr, part, dist, valid,
               xnat, dtype);
  return xp;
}

// IvfTransformer::transform over one chunk of rows already on the device as f32 (lance-index/src/vector/ivf.rs:
// 188-236,357): [normalise if cosine] -> partition id -> residual -> PQ code.  The quantizer of an index build is
// trained -- and therefore encodes -- with L2 whatever the index metric is: Q::build(&training_data,
// DistanceType::L2, ..) (rust/lance/src/index/vector/builder.rs:460); the index metric only decides the partition
// assignment, whether residuals are taken (not for dot, PQBuildParams::use_residual) and the query-time table.
// res_part (nullable): the partitions the residuals are taken to instead of the assigned ones.
static void transform_chunk(const lb2_index& ix, const float* xf, const void* xnat, int dtype, uint64_t rows,
                            DevBuf<float>& normbuf, uint32_t* part, uint8_t* codes, uint8_t* valid,
                            const uint32_t* res_part) {
  const float* xp = normalize_assign(ix, xf, xnat, dtype, rows, normbuf, part, valid, nullptr);
  const bool dot = ix.metric == METRIC_DOT;
  pq_encode_any(xp, rows, ix.d, ix.M, ix.d / ix.M, ix.codebook.p, METRIC_L2, dot ? nullptr : ix.centroids.p,
                dot ? nullptr : (res_part ? res_part : part), valid, ix.nbits, codes);
}

// partition assignment of one chunk of rows (IVF_FLAT / IVF_SQ / IVF_RQ transform); returns the chunk as f32 as the
// index sees it: normalised under cosine.  Rows with a non-finite element are dropped in every metric
// (KeepFiniteVectors precedes the partition transform, ivf.rs:166, 256, 299).  Under L2 and cosine such a row has
// no finite distance and the assignment already drops it; under dot a +-inf element can still give a -inf best
// distance, so the elements are checked.
static const float* assign_flat_chunk(const lb2_index& ix, const float* xf, const void* xnat, int dtype, uint64_t rows,
                                      DevBuf<float>& normbuf, uint32_t* part, uint8_t* valid, float* dist) {
  const float* xp = normalize_assign(ix, xf, xnat, dtype, rows, normbuf, part, valid, dist);
  if (ix.metric == METRIC_DOT && rows)
    LB2_LAUNCH("drop_nonfinite_rows", finite_rows_kernel, cdiv(rows * 32, 256), 256, 0, xp, rows, ix.d, valid, 1);
  return xp;
}

// ---- IVF_SQ: IVFIndex<FlatIndex, ScalarQuantizer> (lance-index/src/vector/sq*.rs) --------------------------------
void sq_check_dim(uint32_t d) {
  LB2_REQUIRE(d > 0 && d % 4 == 0, "IVF_SQ needs a dimension that is a multiple of 4");
  // the scan sums d terms of up to 255^2 in u32 (sq/storage.rs:432-468)
  LB2_REQUIRE((uint64_t)d * 255 * 255 < (1ull << 32), "IVF_SQ: d * 255^2 must be below 2^32, d = %u", d);
}

// ---- IVF_RQ: IVFIndex<FlatIndex, RabitQuantizer> (lance-index/src/vector/bq/*.rs) ---------------------------------
void rq_check(uint32_t d, lb2_dtype dtype, uint32_t num_bits) {
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
// rotated and encoded in sub-chunks of at most 2^28 / code_dim rows (1 GB of f32).  cnorm: |c|^2 per centroid
// (norm_squared_fsl, RQTransformer::new, bq/transform.rs:42-59), dot only.
struct RqWork {
  DevBuf<float> normbuf, dist, res, rot, cnorm;
};
static void rq_transform_chunk(const lb2_index& ix, const float* xf, const void* xnat, int dtype, uint64_t rows,
                               RqWork& w, uint32_t* part, uint8_t* valid, uint8_t* codes, float* add, float* scale) {
  const int d = ix.d, cd = ix.code_dim();
  const uint64_t sub = std::min<uint64_t>(rows, std::max<uint64_t>(1, (1ull << 28) / (uint64_t)cd));
  if (w.dist.n < rows) w.dist.alloc(rows);
  if (w.res.n < rows * d) w.res.alloc(rows * d);
  if (w.rot.n < sub * cd) w.rot.alloc(sub * cd);
  const float* xs = assign_flat_chunk(ix, xf, xnat, dtype, rows, w.normbuf, part, valid, w.dist.p);
  rq_residual_f32(xs, rows, d, ix.centroids.p, part, valid, w.res.p);
  for (uint64_t r0 = 0; r0 < rows; r0 += sub) {
    const uint64_t rs = std::min(sub, rows - r0);
    rq_rotate_f32(ix.rq_rot.p, cd, d, w.res.p + r0 * d, rs, w.rot.p);
    rq_encode_f32(w.rot.p, w.res.p + r0 * d, w.dist.p + r0, part + r0, w.cnorm.p, valid + r0, rs, d, ix.nbits,
                  ix.metric == METRIC_DOT ? METRIC_DOT : METRIC_L2, codes + r0 * (cd / 8), add + r0, scale + r0);
  }
}

// The transform of every row of `src` with the model and partition rule of `index`, chunk by chunk: the builds' full
// pass, lb2_index_transform, the stand-alone IVF_PQ / IVF_RQ transforms and a split's moved rows.  Every output is
// nullable: a NULL part_out, valid_out, add_out / scale_out (IVF_RQ) or payload_out gets scratch, except IVF_FLAT's
// payload, whose stored rows are then not converted (a build groups them from `src` again, index_load_flat_src).
// Synchronises only when it allocated scratch.  given_part (nullable, device): the partition of every row is given
// (a split's decisions, build_assign_batch's PART_ID column, builder.rs:1534-1650): IVF_PQ takes its residuals to it;
// the other kinds store the same payload whatever the partition, and part_out still gets the assigned partition.
void index_transform_rows(const lb2_index* index, Source& src, const uint32_t* given_part, uint32_t* part_out,
                          uint8_t* payload_out, float* add_out, float* scale_out, uint8_t* valid_out) {
  const uint64_t n = src.n();
  const bool rq = index->kind == IndexKind::RQ;
  const int d = index->d;
  const size_t rb = index->row_bytes();
  DevBuf<uint32_t> ptmp;
  DevBuf<uint8_t> vtmp, ltmp;
  DevBuf<float> atmp, stmp;
  bool scratch = false;
  auto need = [&](auto& buf, auto*& p, uint64_t count) {
    if (p) return;
    buf.alloc(std::max<uint64_t>(count, 1));
    p = buf.p;
    scratch = true;
  };
  need(ptmp, part_out, n);
  need(vtmp, valid_out, n);
  if (index->kind != IndexKind::FLAT) need(ltmp, payload_out, n * rb);
  if (rq) {
    need(atmp, add_out, n);
    need(stmp, scale_out, n);
  }
  if (n) {
    src.start_resident_copy();
    const int sdt = (int)src.dtype();
    RqWork w;
    if (rq && index->metric == METRIC_DOT) {
      w.cnorm.alloc(index->K);
      rq_norm_sq_f32(index->centroids.p, index->K, d, w.cnorm.p);
    }
    for_each_chunk(src, [&](const float* xf, const void* xnat, uint64_t r0, uint64_t rows) {
      uint32_t* part = part_out + r0;
      uint8_t* valid = valid_out + r0;
      switch (index->kind) {
        case IndexKind::PQ:
          transform_chunk(*index, xf, xnat, sdt, rows, w.normbuf, part, payload_out + r0 * rb, valid,
                          given_part ? given_part + r0 : nullptr);
          break;
        case IndexKind::RQ:
          rq_transform_chunk(*index, xf, xnat, sdt, rows, w, part, valid, payload_out + r0 * rb, add_out + r0,
                             scale_out + r0);
          break;
        case IndexKind::SQ: {  // the SQ codes of the stored vectors themselves
          const float* xs = assign_flat_chunk(*index, xf, xnat, sdt, rows, w.normbuf, part, valid, nullptr);
          if (index->metric == METRIC_COSINE)  // as IVF_FLAT stores them
            round_model(w.normbuf.p, (size_t)rows * d, index->dtype);
          sq_encode_f32(xs, (uint64_t)rows * d, index->sq_lower, index->sq_upper, payload_out + r0 * rb);
          break;
        }
        case IndexKind::FLAT: {  // index_load_flat_src's stored rows: (normalised) f32 in the stored element type
          const float* xs = assign_flat_chunk(*index, xf, xnat, sdt, rows, w.normbuf, part, valid, nullptr);
          if (!payload_out) break;
          const lb2_dtype vdt = index->vdtype();
          if (vdt == LB2_F32)
            d2d(reinterpret_cast<float*>(payload_out + r0 * rb), xs, (size_t)rows * d);
          else
            LB2_LAUNCH("convert_from_f32", from_f32_kernel, cdiv(rows * d, 256), 256, 0, xs, (int)vdt, (size_t)rows * d,
                       (void*)(payload_out + r0 * rb));
          break;
        }
      }
    });
  }
  if (scratch) sync_stream();  // the scratch outputs are freed on return
}

// IVF_PQ's IVF stage, gathering its own sample before the bulk copy starts.  Staging (class Source): device rows are used in place.  Host rows:
// both training samples (<= K * 256 and 65 536 rows) are gathered straight out of the caller's memory (zero-copy
// reads over PCIe when it is pinned), then the matrix is copied ONCE, in its own element type, on a second stream
// while both trainings run; the per-row pass waits for it and converts one chunk of rows at a time.  A matrix too
// large for that is streamed chunk by chunk during the per-row pass instead (double buffered).  No whole-matrix f32
// copy exists.  Returns the PQ sample (256*2^nbits rows, builder.rs:410-421; normalised for cosine, rows that are
// not finite dropped, builder.rs:436) in sample_pq.
static uint64_t stage_ivf_pq(Source& src, lb2_index* ix, const lb2_kmeans_params& kp, const lb2_pq_params& pq,
                             uint64_t seed, DevBuf<float>& sample_pq, std::vector<double>* loss,
                             std::vector<uint32_t>* iters) {
  const uint64_t n = src.n();
  const int m = ix->metric, d = ix->d;
  const uint64_t nranks = comm_nranks();  // sharded build: this rank's rows
  const uint64_t s_pq0 = std::min<uint64_t>(n, (pq.sample_rate * ((uint64_t)1 << ix->nbits) + nranks - 1) / nranks);
  DevBuf<float> sample_ivf;
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
    std::vector<uint64_t> rows = ivf_sample_rows(n, ix->K, kp, seed);
    stamp("sample_rows(ivf)");
    s_ivf = gather_finite_sample(src, rows, m == METRIC_COSINE, sample_ivf);
    stamp("gather(ivf sample)");
    rows_pq = sample_rows(n, s_pq0, seed + 1);
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
  src.start_resident_copy();
  if (trace) fprintf(stderr, "[lb2 build] %-22s +%.3f ms (host, no sync)\n", "bulk copy issued",
                     std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - tr0).count());
  train_ivf_model(sample_ivf.p, s_ivf, ix, kp, loss, iters);
  stamp("ivf trained");
  if (pq_deferred) {
    if (src.finish_async_sample()) {
      s_pq = rows_pq.size();
    } else {  // rare: some sampled rows are not finite -> the synchronous path drops them and gathers again
      s_pq = gather_finite_sample(src, rows_pq, false, sample_pq);
    }
  }
  return s_pq;
}

// a build's quantizer parameters: nbits (IVF_SQ, IVF_RQ, IVF_PQ), the IVF_SQ bounds' sample_rate, IVF_PQ's parameters
struct QuantizerParams {
  uint32_t nbits = 0;
  uint64_t sample_rate = 0;
  const lb2_pq_params* pq = nullptr;
};

// IvfIndexBuilder::build (builder.rs:236) of every kind, its arguments checked: 1. the IVF stage; 2. the quantizer
// (none for IVF_FLAT); 3. every row transformed through the index's partition rule; 4. the kept rows grouped by
// partition.  stats: the time between the stages' events.
static void build_index(IndexKind kind, const void* data, uint64_t n, uint32_t d, lb2_dtype dtype, int m, uint32_t K,
                        const lb2_kmeans_params& kp, uint64_t seed, const QuantizerParams& q, const uint64_t* row_ids,
                        lb2_index** out, lb2_build_stats* stats) {
  const bool flat = kind == IndexKind::FLAT;
  const int q1 = flat ? 0 : 1;  // the quantizer stage's event
  EventSet ev(4 + q1);
  ev.record(0);
  // (declared before `src`: on an error path ~Source waits for the copy stream, which may still be writing IVF_PQ's
  // deferred sample, before the buffer goes back to the pool)
  DevBuf<float> sample_pq;
  Source src(data, n, (int)d, dtype);
  std::unique_ptr<lb2_index> ix = make_index(kind, K, d, m, dtype);
  ix->nbits = (int)q.nbits;
  std::vector<double> loss;
  std::vector<uint32_t> iters, pq_iters;
  // 1. IVF: the same sample, seed and training for every kind
  uint64_t s_pq = 0;
  if (kind == IndexKind::PQ) {
    ix->M = q.pq->num_sub_vectors;
    ix->codebook.alloc(ix->codebook_len());
    s_pq = stage_ivf_pq(src, ix.get(), kp, *q.pq, seed, sample_pq, &loss, &iters);
  } else {
    TagScope tg("ivf_train");
    std::vector<uint64_t> rows = ivf_sample_rows(n, K, kp, seed);
    DevBuf<float> sample;
    const uint64_t s = gather_finite_sample(src, rows, m == METRIC_COSINE, sample);
    src.start_resident_copy();  // host rows: the bulk copy runs on its own stream while the centroids train
    train_ivf_model(sample.p, s, ix.get(), kp, &loss, &iters);
  }
  ev.record(1);
  // 2. the quantizer
  switch (kind) {
    case IndexKind::FLAT:
      break;
    case IndexKind::SQ: {
      // ScalarQuantizer::build (sq.rs:152-182) on sample_rate * 2^num_bits rows (builder.rs:410-421), normalised under
      // cosine, rows that are not finite dropped (builder.rs:436), no residuals (quantizer.rs:52).  The bounds are
      // taken over the values the index stores: normalised, in the column's element type.
      TagScope tg("sq_train");
      std::vector<uint64_t> rows = sample_rows(n, std::min<uint64_t>(n, q.sample_rate * 256), seed + 1);
      DevBuf<float> sample;
      const uint64_t s = gather_finite_sample(src, rows, m == METRIC_COSINE, sample);
      round_model(sample.p, (size_t)s * d, dtype);
      sq_bounds_f32(sample.p, (uint64_t)s * d, &ix->sq_lower, &ix->sq_upper);
      break;
    }
    case IndexKind::RQ: {  // RabitQuantizer::new (bq/builder.rs:52-70): the rotation, from seed + 1
      TagScope tg("rq_train");
      const int cd = ix->code_dim();
      ix->rq_rot.alloc((size_t)cd * cd);
      rq_rotation_f32(cd, seed + 1, ix->rq_rot.p);
      break;
    }
    case IndexKind::PQ: {  // residuals of its sample w.r.t. the IVF centroids (builder.rs:439-450)
      TagScope tg("pq_train");
      if (m != METRIC_DOT && s_pq) {
        DevBuf<uint32_t> part(s_pq);
        assign_f32(sample_pq.p, s_pq, d, ix->centroids.p, K, METRIC_L2, nullptr, part.p, nullptr, nullptr);
        LB2_LAUNCH("residual", residual_kernel, cdiv(s_pq * d, 256), 256, 0, sample_pq.p, ix->centroids.p, part.p, s_pq,
                   (int)d, sample_pq.p);
      }
      VecIn cb_init(q.pq->codebook, ix->codebook_len(), model_dtype(dtype));
      lb2_pq_params pqp = *q.pq;
      pqp.codebook = cb_init.get();
      // always L2 k-means (builder.rs:460: Q::build(&training_data, DistanceType::L2, ..)); for a dot index the sample
      // is the raw vectors (no residual), for L2 / cosine the residuals computed above
      pq_train_dev(sample_pq.p, s_pq, d, METRIC_L2, &pqp, ix->codebook.p, &pq_iters);
      round_model(ix->codebook.p, ix->codebook_len(), dtype);
      sample_pq.release();
      break;
    }
  }
  if (q1) ev.record(2);
  // 3. transform (ivf.rs:188-328): IVF_FLAT keeps the partitions only, index_load_flat_src gathers its rows again
  DevBuf<uint32_t> part(std::max<uint64_t>(n, 1));
  DevBuf<uint8_t> valid(std::max<uint64_t>(n, 1)), payload;
  DevBuf<float> add, scale;
  if (!flat) payload.alloc(std::max<uint64_t>(1, n * ix->row_bytes()));
  if (kind == IndexKind::RQ) {
    add.alloc(std::max<uint64_t>(n, 1));
    scale.alloc(std::max<uint64_t>(n, 1));
  }
  {
    TagScope tg("transform");
    set_partition_index(ix.get(), kp.partition_index, partition_index_seed(seed), kp.partition_index_batch);
    index_transform_rows(ix.get(), src, nullptr, part.p, payload.p, add.p, scale.p, valid.p);
  }
  ev.record(2 + q1);
  {
    // 4. group the kept rows by partition (shuffle + build_partitions, builder.rs:501-937); rows the transform marked
    //    invalid are dropped, as KeepFiniteVectors does (transform.rs:112-159)
    TagScope tg("group");
    InArg<uint64_t> rid(row_ids, n);
    if (flat)  // the stored vectors are the normalised ones when the metric is cosine
      index_load_flat_src(ix.get(), part.p, src, rid.get(), valid.p, m == METRIC_COSINE);
    else
      index_load_dev(ix.get(), part.p, payload.p, rid.get(), n, valid.p, add.p, scale.p);
  }
  ev.record(3 + q1);
  sync_stream();
  if (stats) {
    memset(stats, 0, sizeof(*stats));
    stats->ms_ivf_train = ev.ms(0, 1);
    if (q1) stats->ms_pq_train = ev.ms(1, 2);
    stats->ms_transform = ev.ms(1 + q1, 2 + q1);
    stats->ms_group = ev.ms(2 + q1, 3 + q1);
    stats->ms_total = ev.ms(0, 3 + q1);
    stats->ivf_iters = iters.empty() ? 0 : iters[0];
    for (auto v : pq_iters) stats->pq_iters_max = std::max(stats->pq_iters_max, v);
    stats->ivf_loss = loss.empty() ? 0.0 : loss[0];
  }
  *out = ix.release();
}

// the defaults of every build's IVF fields (IvfBuildParams, ivf/builder.rs:62-78; balance factor 1,
// rust/lance/src/index/vector/ivf.rs:1858) and of an HNSW build's graph (HnswBuildParams::default,
// hnsw/builder.rs:63-72, inserted serially)
template <class P>
static void ivf_defaults(P* p) {
  p->num_partitions = 256;
  lb2_kmeans_params_default(&p->ivf);
  p->ivf.balance_factor = 1.0f;
  p->seed = 0;
}
template <class P>
static void hnsw_defaults(P* p) {
  p->max_level = 7;
  p->m = 20;
  p->ef_construction = 150;
  p->insert_batch = 1;
}

// lb2_index_transform's rows into the caller's buffers (host or device, each nullable)
static void transform_into(const lb2_index* ix, const void* vectors, uint64_t n, uint32_t* part_out,
                           uint8_t* payload_out, float* add_out, float* scale_out, uint8_t* valid_out) {
  OutArg<uint32_t> po(part_out, n);
  OutArg<uint8_t> pl(payload_out, (size_t)n * ix->row_bytes()), vo(valid_out, n);
  OutArg<float> ao(add_out, n), so(scale_out, n);
  if (n) {
    Source src(vectors, n, ix->d, ix->dtype);
    index_transform_rows(ix, src, nullptr, po.get(), pl.get(), ao.get(), so.get(), vo.get());
  }
  po.commit(); pl.commit(); vo.commit(); ao.commit(); so.commit();
  sync_stream();
}
// the stand-alone transforms run on a handle holding the caller's model as it is (never rounded to the column's type)
static void copy_in(float* to, const void* from, size_t count, lb2_dtype dt) {
  VecIn v(from, count, dt);
  d2d(to, v.get(), count);
}

}  // namespace lb2

using namespace lb2;

extern "C" {

void lb2_ivfpq_build_params_default(lb2_ivfpq_build_params* p) {
  ivf_defaults(p);
  lb2_pq_params_default(&p->pq);
}

void lb2_ivfflat_build_params_default(lb2_ivfflat_build_params* p) { ivf_defaults(p); }

void lb2_ivfsq_build_params_default(lb2_ivfsq_build_params* p) {
  ivf_defaults(p);
  p->num_bits = 8;
  p->sample_rate = 256;
}

void lb2_ivfhnswsq_build_params_default(lb2_ivfhnswsq_build_params* p) {
  lb2_ivfsq_build_params_default(&p->sq);
  hnsw_defaults(p);
}

void lb2_ivfhnswpq_build_params_default(lb2_ivfhnswpq_build_params* p) {
  lb2_ivfpq_build_params_default(&p->pq);
  hnsw_defaults(p);
}

void lb2_ivfhnswflat_build_params_default(lb2_ivfhnswflat_build_params* p) {
  lb2_ivfflat_build_params_default(&p->flat);
  hnsw_defaults(p);
}

void lb2_ivfrq_build_params_default(lb2_ivfrq_build_params* p) {
  ivf_defaults(p);
  p->num_bits = 1;
}

lb2_status lb2_ivfpq_transform(const void* centroids, uint32_t k, const void* codebook,
                               uint32_t num_sub_vectors, uint32_t num_bits, uint32_t d,
                               lb2_dtype dtype, lb2_metric metric, const void* vectors, uint64_t n,
                               uint32_t* part_out, uint8_t* codes_out, uint8_t* valid_out) {
  LB2_API_BEGIN
  check_pq_shape(d, num_sub_vectors, num_bits, PqUse::ENCODE);
  std::unique_ptr<lb2_index> ix = make_index(IndexKind::PQ, k, d, metric_of(metric), dtype);
  ix->M = (int)num_sub_vectors;
  ix->nbits = (int)num_bits;
  ix->codebook.alloc(ix->codebook_len());
  copy_in(ix->centroids.p, centroids, (size_t)k * d, model_dtype(dtype));
  copy_in(ix->codebook.p, codebook, ix->codebook_len(), model_dtype(dtype));
  transform_into(ix.get(), vectors, n, part_out, codes_out, nullptr, nullptr, valid_out);
  LB2_API_END
}

lb2_status lb2_ivfrq_transform(const void* centroids, uint32_t k, const void* rotation, uint32_t d, uint32_t num_bits,
                               lb2_dtype dtype, lb2_metric metric, const void* vectors, uint64_t n, uint32_t* part_out,
                               uint8_t* codes_out, float* add_out, float* scale_out, uint8_t* valid_out) {
  LB2_API_BEGIN
  LB2_REQUIRE(centroids && rotation && (vectors || n == 0) && k > 0, "null argument");
  rq_check(d, dtype, num_bits);
  std::unique_ptr<lb2_index> ix = make_index(IndexKind::RQ, k, d, metric_of(metric), dtype);
  ix->nbits = (int)num_bits;
  const uint64_t cd = ix->code_dim();
  ix->rq_rot.alloc(cd * cd);
  copy_in(ix->centroids.p, centroids, (size_t)k * d, dtype);
  copy_in(ix->rq_rot.p, rotation, cd * cd, dtype);
  transform_into(ix.get(), vectors, n, part_out, codes_out, add_out, scale_out, valid_out);
  LB2_API_END
}

lb2_status lb2_index_transform(const lb2_index* index, const void* vectors, uint64_t n, uint32_t* part_out,
                               uint8_t* payload_out, float* add_out, float* scale_out, uint8_t* valid_out) {
  LB2_API_BEGIN
  LB2_REQUIRE(index && (vectors || n == 0), "null argument");
  LB2_REQUIRE(index->kind == IndexKind::RQ || (!add_out && !scale_out), "lb2_index_transform: add and scale factors are for IVF_RQ indexes only");
  transform_into(index, vectors, n, part_out, payload_out, add_out, scale_out, valid_out);
  LB2_API_END
}

lb2_status lb2_ivfflat_build(const void* data, uint64_t n, uint32_t d, lb2_dtype dtype,
                             lb2_metric metric, const lb2_ivfflat_build_params* params,
                             const uint64_t* row_ids, lb2_index** out, lb2_build_stats* stats) {
  LB2_API_BEGIN
  LB2_REQUIRE(data && params && out, "null argument");
  LB2_REQUIRE(d % 4 == 0, "IVF_FLAT needs a dimension that is a multiple of 4");
  const int m = metric_of(metric);
  const int K = params->num_partitions;
  LB2_REQUIRE(K > 0 && (comm_nranks() > 1 || n >= (uint64_t)K), "KMeans: can not train %d centroids with %llu vectors", K,
              (unsigned long long)n);
  build_index(IndexKind::FLAT, data, n, d, dtype, m, K, params->ivf, params->seed, {}, row_ids, out, stats);
  LB2_API_END
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
  build_index(IndexKind::SQ, data, n, d, dtype, m, K, params->ivf, params->seed, {params->num_bits, params->sample_rate},
              row_ids, out, stats);
  LB2_API_END
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
  build_index(IndexKind::RQ, data, n, d, dtype, m, K, params->ivf, params->seed, {params->num_bits}, row_ids, out,
              stats);
  LB2_API_END
}

lb2_status lb2_ivfpq_build(const void* data, uint64_t n, uint32_t d, lb2_dtype dtype,
                           lb2_metric metric, const lb2_ivfpq_build_params* params,
                           const uint64_t* row_ids, lb2_index** out, lb2_build_stats* stats) {
  LB2_API_BEGIN
  LB2_REQUIRE(data && params && out, "null argument");
  const int m = metric_of(metric);
  const int K = params->num_partitions;
  LB2_REQUIRE(K > 0 && (comm_nranks() > 1 || n >= (uint64_t)K), "KMeans: can not train %d centroids with %llu vectors", K,
              (unsigned long long)n);
  check_pq_shape(d, params->pq.num_sub_vectors, params->pq.num_bits, PqUse::ENCODE);
  build_index(IndexKind::PQ, data, n, d, dtype, m, K, params->ivf, params->seed, {params->pq.num_bits, 0, &params->pq},
              row_ids, out, stats);
  LB2_API_END
}

}  // extern "C"

// the graph parameters of an HNSW build (hnsw/builder.rs:63-72) and the batched insertion's B
static void check_hnsw_params(IndexKind kind, uint32_t max_level, uint32_t m, uint32_t ef_construction,
                              uint32_t insert_batch) {
  const char* name = hnsw_kind_name(kind);
  LB2_REQUIRE(max_level >= 1 && max_level <= 64, "%s: max_level must be in 1 .. 64, got %u", name, max_level);
  LB2_REQUIRE(m >= 1 && m <= 1024, "%s: m must be in 1 .. 1024, got %u", name, m);
  LB2_REQUIRE(ef_construction >= 1, "%s: ef_construction must be at least 1", name);
  LB2_REQUIRE(insert_batch <= 65536, "%s: insert_batch must be at most 65536, got %u", name, insert_batch);
}

// an IVF_HNSW_* build: 1. build_base, the IVF_SQ, IVF_PQ or IVF_FLAT build with the same arguments (params->*base),
// gives the IVF stage, the model and the payload; 2. HNSW::index_vectors per partition over its storage (v3
// IvfIndexBuilder with an HNSW sub-index), counted in stats->ms_total only.  Only IVF_HNSW_SQ builds over more than
// one rank.
template <class P, class BP>
static lb2_status build_hnsw(IndexKind kind, BP P::*base,
                             lb2_status (*build_base)(const void*, uint64_t, uint32_t, lb2_dtype, lb2_metric, const BP*,
                                                      const uint64_t*, lb2_index**, lb2_build_stats*),
                             const void* data, uint64_t n, uint32_t d, lb2_dtype dtype, lb2_metric metric,
                             const P* params, const uint64_t* row_ids, lb2_index** out, lb2_build_stats* stats) {
  LB2_API_BEGIN
  LB2_REQUIRE(data && params && out, "null argument");
  check_hnsw_params(kind, params->max_level, params->m, params->ef_construction, params->insert_batch);
  if (kind != IndexKind::SQ && comm_nranks() > 1)
    fail(LB2_UNSUPPORTED, "%s: a build over more than one rank is not implemented", hnsw_kind_name(kind));
  lb2_index* built = nullptr;
  const lb2_status st = build_base(data, n, d, dtype, metric, &(params->*base), row_ids, &built, stats);
  if (st != LB2_OK) return st;  // its message is already the last error
  std::unique_ptr<lb2_index> ix(built);
  EventSet ev(2);
  ev.record(0);
  attach_graph(ix.get(), params->max_level, params->m, params->ef_construction, params->insert_batch,
               (params->*base).seed);
  ev.record(1);
  if (stats) stats->ms_total += ev.ms(0, 1);
  *out = ix.release();
  LB2_API_END
}

extern "C" {

lb2_status lb2_ivfhnswsq_build(const void* data, uint64_t n, uint32_t d, lb2_dtype dtype, lb2_metric metric,
                               const lb2_ivfhnswsq_build_params* params, const uint64_t* row_ids, lb2_index** out,
                               lb2_build_stats* stats) {
  return build_hnsw(IndexKind::SQ, &lb2_ivfhnswsq_build_params::sq, lb2_ivfsq_build, data, n, d, dtype, metric,
                    params, row_ids, out, stats);
}

lb2_status lb2_ivfhnswpq_build(const void* data, uint64_t n, uint32_t d, lb2_dtype dtype, lb2_metric metric,
                               const lb2_ivfhnswpq_build_params* params, const uint64_t* row_ids, lb2_index** out,
                               lb2_build_stats* stats) {
  return build_hnsw(IndexKind::PQ, &lb2_ivfhnswpq_build_params::pq, lb2_ivfpq_build, data, n, d, dtype, metric,
                    params, row_ids, out, stats);
}

lb2_status lb2_ivfhnswflat_build(const void* data, uint64_t n, uint32_t d, lb2_dtype dtype, lb2_metric metric,
                                 const lb2_ivfhnswflat_build_params* params, const uint64_t* row_ids, lb2_index** out,
                                 lb2_build_stats* stats) {
  return build_hnsw(IndexKind::FLAT, &lb2_ivfhnswflat_build_params::flat, lb2_ivfflat_build, data, n, d, dtype,
                    metric, params, row_ids, out, stats);
}

}  // extern "C"
