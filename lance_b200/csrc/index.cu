// index.cu -- the device-resident index: creation, loads and exports of every kind, the grouping of rows by
// partition, the attachment of HNSW graphs, search dispatch, incremental update and the partition exchange of a
// row-sharded index.
#include <algorithm>
#include <cstring>
#include <memory>

#include "build.cuh"
#include "comm.cuh"
#include "flat_search.cuh"
#include "index.cuh"
#include "ivf_search.cuh"
#include "member_sort.cuh"
#include "rq.cuh"
#include "scan.cuh"
#include "sq.cuh"

namespace lb2 {

std::unique_ptr<lb2_index> make_index(IndexKind kind, uint32_t K, uint32_t d, int metric, lb2_dtype dtype) {
  std::unique_ptr<lb2_index> ix(new lb2_index());
  ix->kind = kind; ix->K = K; ix->d = d; ix->metric = metric; ix->dtype = dtype;
  ix->centroids.alloc((size_t)K * d);
  return ix;
}

// an empty index with the caller's centroids (in the model type of `dtype`)
static std::unique_ptr<lb2_index> index_with_centroids(IndexKind kind, const void* centroids, uint32_t k, uint32_t d,
                                                       lb2_dtype dtype, lb2_metric metric) {
  ctx();
  std::unique_ptr<lb2_index> ix = make_index(kind, k, d, metric_of(metric), dtype);
  {
    VecIn c(centroids, (size_t)k * d, model_dtype(dtype));
    d2d(ix->centroids.p, c.get(), (size_t)k * d);
    sync_stream();
  }
  ix->part_offsets.alloc(k + 1);
  ix->part_offsets.zero();
  sync_stream();
  return ix;
}

// the model of `from` in `to`, an index of the same kind from make_index: the centroids (or `new_centroids`, in the
// model type of the index, when given), M, nbits, and the codebook, SQ bounds or RQ rotation as the kind has them
void copy_model(const lb2_index* from, lb2_index* to, const void* new_centroids) {
  const size_t kd = (size_t)to->K * to->d;
  if (new_centroids) {
    VecIn c(new_centroids, kd, model_dtype(to->dtype));
    d2d(to->centroids.p, c.get(), kd);
    sync_stream();
  } else {
    d2d(to->centroids.p, from->centroids.p, kd);
  }
  to->M = from->M;
  to->nbits = from->nbits;
  switch (from->kind) {
    case IndexKind::PQ:
      to->codebook.alloc(from->codebook_len());
      d2d(to->codebook.p, from->codebook.p, from->codebook_len());
      break;
    case IndexKind::SQ:
      to->sq_lower = from->sq_lower;
      to->sq_upper = from->sq_upper;
      break;
    case IndexKind::RQ:
      to->rq_rot.alloc((size_t)from->code_dim() * from->code_dim());
      d2d(to->rq_rot.p, from->rq_rot.p, (size_t)from->code_dim() * from->code_dim());
      break;
    case IndexKind::FLAT:
      break;
  }
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

void check_part_ids(const uint32_t* part_ids, uint64_t n, uint32_t K, const char* what) {
  if (n == 0) return;
  DevBuf<uint32_t> mx(1);
  mx.zero();
  LB2_LAUNCH("check_part_ids", max_u32_kernel, (unsigned)std::min<uint64_t>(cdiv(n, 1024), 1024), 256, 0, part_ids, n, mx.p);
  uint32_t h = 0;
  d2h(&h, mx.p, 1);
  sync_stream();
  if (h >= K) fail(LB2_INVALID_ARG, "%s: partition id %u out of range (the index has %u partitions)", what, h, K);
}

__global__ void widen_offsets_kernel(const uint32_t* __restrict__ off32, int K,
                                     uint64_t* __restrict__ off64) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i <= K) off64[i] = off32[i];
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

// the conflict-free scan's skewed copy of the codes, for the shapes that have one
static void build_skew(lb2_index* ix) {
  if (ix->n && skew_layout_applies(ix->M, ix->d, ix->nbits)) {
    ix->slab_off.alloc(ix->K + 1);
    ix->codes_skew.alloc(skew_bytes_bound(ix->n, ix->K));
    build_skew_codes(ix->part_offsets.p, ix->K, ix->codes.p, ix->n, ix->slab_off.p, ix->codes_skew.p);
  } else {
    ix->slab_off.release();
    ix->codes_skew.release();
  }
}

// vec16: M is a multiple of 16 and both payloads are 16-byte aligned (IVF_FLAT rows), copied 16 bytes at a time
__global__ void group_kernel(const uint32_t* __restrict__ members, uint64_t n, int M,
                             const uint8_t* __restrict__ codes, const uint64_t* __restrict__ row_ids,
                             uint8_t* __restrict__ codes_out, uint64_t* __restrict__ row_ids_out, int vec16) {
  const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n) return;
  const uint32_t src = members[g];
  row_ids_out[g] = row_ids ? row_ids[src] : (uint64_t)src;
  if (vec16) {
    for (int m = 0; m < M; m += 16)
      *reinterpret_cast<uint4*>(codes_out + g * M + m) = *reinterpret_cast<const uint4*>(codes + (size_t)src * M + m);
  } else {
    for (int m = 0; m < M; ++m) codes_out[g * M + m] = codes[(size_t)src * M + m];
  }
}

__global__ void gather_f32_kernel(const uint32_t* __restrict__ members, uint64_t n, const float* __restrict__ src,
                                  float* __restrict__ dst) {
  const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g < n) dst[g] = src[members[g]];
}

void index_load_dev(lb2_index* ix, const uint32_t* part_ids, const uint8_t* codes, const uint64_t* row_ids,
                    uint64_t n, const uint8_t* valid, const float* rq_add, const float* rq_scale) {
  MemberSort ms;
  const uint64_t kept = member_sort_index(ms, ix, part_ids, valid, n);
  const int cb = (int)ix->row_bytes();
  DevBuf<uint8_t>& out = ix->payload();
  out.alloc(std::max<uint64_t>(1, kept * cb));
  ix->row_ids.alloc(std::max<uint64_t>(1, kept));
  const int vec16 = cb % 16 == 0 && (reinterpret_cast<uintptr_t>(codes) & 15) == 0;
  if (kept)
    LB2_LAUNCH("group_by_partition", group_kernel, cdiv(kept, 256), 256, 0, ms.members.p, kept, cb, codes, row_ids,
               out.p, ix->row_ids.p, vec16);
  if (ix->kind == IndexKind::RQ) {
    ix->rq_add.alloc(std::max<uint64_t>(1, kept));
    ix->rq_scale.alloc(std::max<uint64_t>(1, kept));
    if (kept) {
      LB2_LAUNCH("group_by_partition", gather_f32_kernel, cdiv(kept, 256), 256, 0, ms.members.p, kept, rq_add, ix->rq_add.p);
      LB2_LAUNCH("group_by_partition", gather_f32_kernel, cdiv(kept, 256), 256, 0, ms.members.p, kept, rq_scale,
                 ix->rq_scale.p);
    }
  }
  ix->n = kept;
  if (ix->kind == IndexKind::PQ) build_skew(ix);
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

void index_load_flat_src(lb2_index* ix, const uint32_t* part_ids, Source& src, const uint64_t* row_ids,
                         const uint8_t* valid, bool normalize) {
  const uint64_t n = src.n();
  MemberSort ms;
  const uint64_t kept = member_sort_index(ms, ix, part_ids, valid, n);
  const lb2_dtype vdt = ix->vdtype();
  const size_t rb = ix->row_bytes();
  ix->vectors.alloc(std::max<size_t>(1, kept * rb));
  ix->row_ids.alloc(std::max<uint64_t>(1, kept));
  ix->n = kept;
  if (!kept) { sync_stream(); return; }
  LB2_LAUNCH("group_row_ids", copy_row_ids_kernel, cdiv(kept, 256), 256, 0, ms.members.p, kept, row_ids, ix->row_ids.p);
  const void* nat = src.native_device();
  if (!nat) fail(LB2_OOM, "IVF_FLAT keeps a copy of the vectors: the %llu x %d matrix must fit in device memory",
                 (unsigned long long)n, ix->d);
  const int d = ix->d;
  if (!normalize && vdt == src.dtype() && rb % 16 == 0 && (reinterpret_cast<uintptr_t>(nat) & 15) == 0) {
    // stored type == column type: one pass, no f32 round trip (a C4 shard: 2 x 19 GB of bf16 at HBM speed)
    const uint32_t vpr = (uint32_t)(rb / 16);
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
  if (normalize && vdt != LB2_F32) tmp2.alloc(std::min(chunk, kept) * d);
  for (uint64_t p0 = 0; p0 < kept; p0 += chunk) {
    const uint64_t rows = std::min(chunk, kept - p0);
    LB2_LAUNCH("group_vectors", members_to_u64_kernel, cdiv(rows, 256), 256, 0, ms.members.p + p0, rows, rows64.p);
    uint8_t* dst = ix->vectors.p + p0 * rb;
    float* g = direct ? reinterpret_cast<float*>(dst) : tmp.p;
    LB2_LAUNCH("group_vectors", gather_rows_typed_kernel, cdiv(rows * d, 256), 256, 0, nat, (int)src.dtype(), rows64.p, rows, d, g);
    if (normalize) {
      float* o = vdt == LB2_F32 ? reinterpret_cast<float*>(dst) : tmp2.p;
      normalize_rows(g, rows, d, o);
      g = o;
    }
    if (vdt != LB2_F32)
      LB2_LAUNCH("convert_from_f32", from_f32_kernel, cdiv(rows * d, 256), 256, 0, g, (int)vdt, (size_t)rows * d, (void*)dst);
  }
  sync_stream();
}

// the code loads of IVF_PQ, IVF_SQ and IVF_RQ (add / scale: IVF_RQ's factors)
static void load_codes(lb2_index* index, const uint32_t* part_ids, const uint8_t* codes, const uint64_t* row_ids,
                       uint64_t n, const char* what, const float* add = nullptr, const float* scale = nullptr) {
  InArg<uint32_t> p(part_ids, n);
  InArg<uint8_t> c(codes, (size_t)n * index->row_bytes());
  InArg<float> a(add, n), s(scale, n);
  InArg<uint64_t> r(row_ids, n);
  check_part_ids(p.get(), n, (uint32_t)index->K, what);
  index_load_dev(index, p.get(), c.get(), r.get(), n, nullptr, a.get(), s.get());
}

// what every kind exports: centroids, partition offsets, the row payload and the row ids (each output nullable, host
// or device memory); the caller adds its kind's model and synchronises
static void export_common(const lb2_index* index, void* centroids_out, uint64_t* part_offsets_out, void* payload_out,
                          uint64_t* row_ids_out) {
  cudaStream_t s = ctx().stream;
  if (centroids_out)
    LB2_CUDA(cudaMemcpyAsync(centroids_out, index->centroids.p, sizeof(float) * index->K * index->d, cudaMemcpyDefault, s));
  if (part_offsets_out)
    LB2_CUDA(cudaMemcpyAsync(part_offsets_out, index->part_offsets.p, sizeof(uint64_t) * (index->K + 1), cudaMemcpyDefault, s));
  if (payload_out && index->n)
    LB2_CUDA(cudaMemcpyAsync(payload_out, index->payload().p, index->n * index->row_bytes(), cudaMemcpyDefault, s));
  if (row_ids_out && index->n)
    LB2_CUDA(cudaMemcpyAsync(row_ids_out, index->row_ids.p, sizeof(uint64_t) * index->n, cudaMemcpyDefault, s));
}

static void search_kind(lb2_index* index, const IvfSearch& s, uint32_t ef);

// the queries of every lb2_index_search*: the index's element type -> f32 (q), normalised under cosine (knn.rs:497-499;
// get() is the search's view)
namespace {
struct SearchQueries {
  VecIn q;
  DevBuf<float> qn;
  const float* p;
  SearchQueries(const lb2_index* index, const void* queries, uint64_t nq)
      : q(queries, (size_t)nq * index->d, index->dtype), p(q.get()) {
    if (index->metric == METRIC_COSINE) {
      qn.alloc((size_t)nq * index->d);
      normalize_rows(p, nq, index->d, qn.p);
      p = qn.p;
    }
  }
  const float* get() const { return p; }
};
}  // namespace

// one implementation behind every lb2_index_search* (pr: the probe rule of lb2_index_search_probed; ef: the graph
// search's ef of lb2_index_search_hnsw, 0 for k' + k' / 2)
static void index_search_impl(lb2_index* index, const void* queries, uint64_t nq, const lb2_search_params& sp,
                              uint64_t* row_ids_out, float* dists_out, uint32_t* counts_out, ProbeRule* pr = nullptr,
                              uint32_t ef = 0) {
  const uint32_t k = sp.k, nprobes = sp.nprobes;
  LB2_REQUIRE(index && k > 0 && (nprobes > 0 || pr), "bad argument");
  const bool refine = sp.refine_factor > 0 && sp.refine_vectors != nullptr;
  const uint64_t kc = refine ? (uint64_t)k * sp.refine_factor : k;
  if (kc > 1024) fail(LB2_UNSUPPORTED, "k * refine_factor = %llu > 1024 is not implemented", (unsigned long long)kc);
  const int d = index->d;
  const SearchQueries q(index, queries, nq);
  const float* qp = q.get();
  InArg<uint64_t> allow(sp.allow_bitmap, sp.allow_bitmap ? (size_t)((index->n + 63) / 64) : 0);
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
  const ScanFilter flt = make_filter(sp.allow_bitmap ? allow.get() : nullptr, sp.has_lower_bound != 0, sp.lower_bound,
                                    sp.has_upper_bound != 0, sp.upper_bound);
  const IvfSearch s{index->centroids.p, index->K, d, index->metric, index->part_offsets.p, index->row_ids.p, qp, nq,
                    (int)kc, (int)nprobes, si, sd, sc, flt, pr};
  search_kind(index, s, ef);
  if (refine) {
    // exact re-rank with the true metric on the ORIGINAL (un-normalised) query, as flat_knn does; the
    // plan then filters `_distance >= lower AND _distance < upper` on the exact distances (scanner.rs:3342-3377)
    InArg<uint8_t> v(sp.refine_vectors, (size_t)sp.num_vectors * d * dtype_size(index->dtype));  // raw column, native type
    refine_f32(q.q.get(), nq, d, index->metric, v.get(), (int)index->dtype, sp.num_vectors, cid.p, ccnt.p, (int)kc, (int)k,
               oi.get(), od.get(), oc.get(), sp.has_lower_bound != 0, sp.lower_bound, sp.has_upper_bound != 0,
               sp.upper_bound);
  }
  oi.commit(); od.commit(); oc.commit();
  if (!ctx().async_call) sync_stream();
}

// the scan of the index's kind over the search s (ef: IVF_HNSW_*'s graph search ef, 0 for k' + k' / 2)
static void search_kind(lb2_index* index, const IvfSearch& s, uint32_t ef) {
  const uint64_t nq = s.nq;
  const int d = s.d;
  DevBuf<uint8_t> qcodes;
  if (index->kind == IndexKind::SQ) {
    // the (normalised) query is encoded with the index's bounds, not turned into a residual (sq/storage.rs:404-430)
    qcodes.alloc(std::max<uint64_t>(1, nq * d));
    sq_encode_f32(s.queries, nq * d, index->sq_lower, index->sq_upper, qcodes.p);
  }
  if (index->hnsw) {  // IVF_HNSW_*: the kind's scan distances, searched through each partition's graph
    hnsw_search(s, *index, qcodes.p, ef);
  } else {
    switch (index->kind) {
      case IndexKind::FLAT:
        ivfflat_search(s, index->vectors.p, (int)index->vdtype());
        break;
      case IndexKind::RQ:
        // the (normalised) query's residual to each probed centroid is rotated (v2.rs:316-332, bq/storage.rs:407-445)
        ivfrq_search(s, index->rq_rot.p, index->code_dim(), index->codes.p, index->rq_add.p, index->rq_scale.p);
        break;
      case IndexKind::SQ: {
        const float rf = (float)(index->sq_upper - index->sq_lower);  // inverse_scalar_dist (sq.rs:279-287)
        ivfsq_search(s, index->codes.p, rf * rf, qcodes.p);
        break;
      }
      case IndexKind::PQ:
        ivfpq_search(s, index->codebook.p, index->M, index->nbits, index->codes.p, index->slab_off.p,
                     index->codes_skew.p);
        break;
    }
  }
}

// ---- partition ownership: device all-to-all (SURVEY 8e "partition build", 8f-4) ---------------------------------
// The reference groups the transformed rows by partition with a disk shuffler on the host
// (rust/lance-index/src/vector/v3/shuffler.rs:105).  For a build sharded by rows over G GPUs the same grouping
// is one exchange over NVLink: rank g becomes the owner of every partition p with p % G == g.

// (these kernels have C linkage: their symbols are the bare names)
extern "C" {
// row i of the shard (storage order) -> slot in the send buffer: rows are grouped by destination rank, inside a
// destination by partition, inside a partition in storage order
__global__ void repart_pack_kernel(const uint64_t* __restrict__ part_offsets, int K, uint64_t n, int row_bytes,
                                   const uint64_t* __restrict__ send_base /*[K]*/, const uint8_t* __restrict__ payload,
                                   const uint64_t* __restrict__ row_ids, uint8_t* __restrict__ payload_out,
                                   uint64_t* __restrict__ row_ids_out) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int p = segment_of(part_offsets, K, i);
  const uint64_t dst = send_base[p] + (i - part_offsets[p]);
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
  const int s = segment_of(seg_prefix, nown, j);
  const uint64_t dst = seg_dst[s] + (j - seg_prefix[s]);
  row_ids_out[dst] = row_ids[j];
  const uint8_t* src = payload + j * (uint64_t)row_bytes;
  uint8_t* o = payload_out + dst * (uint64_t)row_bytes;
  if ((row_bytes & 15) == 0) {
    for (int b = 0; b < row_bytes; b += 16) *reinterpret_cast<uint4*>(o + b) = *reinterpret_cast<const uint4*>(src + b);
  } else {
    for (int b = 0; b < row_bytes; ++b) o[b] = src[b];
  }
}

// ---- the merge of optimize / split / join / remap, for every kind (SURVEY 8f-4) ------------------------------------
// The reference turns an optimize step into per-partition AssignOp::Add / AssignOp::Remove lists against a new
// centroid set (rust/lance/src/index/vector/builder.rs:1219-1333 split, :1476-1530 join, :1534-1650
// build_assign_batch) and merges them with the existing partitions when it writes the index.  The decisions of a
// split or join are split.cu's; index_merge is the merge: old rows keep their payload, follow `part_map`, removed row
// ids are dropped, added rows join the end of their partitions, and a compaction's row-id mapping is applied last.
// One pass over the old rows (storage order): the new partition and keep flag of each, and the rows each old
// partition loses (dropped[p], nullable: the graph kinds' change detection)
__global__ void update_old_rows_kernel(const uint64_t* __restrict__ part_offsets, int K, uint64_t n,
                                       const uint32_t* __restrict__ part_map /*nullable*/,
                                       const uint64_t* __restrict__ row_ids, const uint64_t* __restrict__ removed,
                                       uint64_t n_removed, uint32_t new_k, uint32_t* __restrict__ part_out,
                                       uint8_t* __restrict__ valid_out, uint32_t* __restrict__ bad,
                                       uint32_t* __restrict__ dropped) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int p = segment_of(part_offsets, K, i);
  const uint32_t np_ = part_map ? part_map[p] : (uint32_t)p;
  bool keep = np_ != 0xffffffffu;
  if (keep && np_ >= new_k) { atomicMax(bad, np_); keep = false; }
  if (keep && n_removed) keep = !sorted_contains(removed, n_removed, row_ids[i]);
  part_out[i] = keep ? np_ : 0u;
  valid_out[i] = keep ? 1 : 0;
  if (!keep && dropped) atomicAdd(&dropped[p], 1u);
}
// bad = 1 when the remap's old ids are not strictly ascending
__global__ void remap_order_kernel(const uint64_t* __restrict__ old_ids, uint64_t n, uint32_t* __restrict__ bad) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i + 1 < n && old_ids[i] >= old_ids[i + 1]) atomicOr(bad, 1u);
}
// storage.remap of every kept row (pq/storage.rs:499-540): one binary search into the sorted pairs; a row mapped to
// UINT64_MAX (None) loses its keep flag (an old row of partition p counts in dropped[p], nullable), a row mapped to
// a value takes it, a row not in the mapping is left as it is
__global__ void remap_rows_kernel(uint64_t* __restrict__ row_ids, uint8_t* __restrict__ valid, uint64_t n,
                                  const uint64_t* __restrict__ old_ids, const uint64_t* __restrict__ new_ids,
                                  uint64_t n_remap, const uint64_t* __restrict__ part_offsets, int K, uint64_t n_old,
                                  uint32_t* __restrict__ dropped) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || !valid[i]) return;
  const uint64_t id = row_ids[i];
  uint64_t lo = 0, hi = n_remap;
  while (lo < hi) {
    const uint64_t mid = (lo + hi) >> 1;
    if (old_ids[mid] < id) lo = mid + 1; else hi = mid;
  }
  if (lo == n_remap || old_ids[lo] != id) return;
  const uint64_t to = new_ids[lo];
  if (to != ~0ull) {
    row_ids[i] = to;
    return;
  }
  valid[i] = 0;
  if (dropped && i < n_old) atomicAdd(&dropped[segment_of(part_offsets, K, i)], 1u);
}
// rows per partition id
__global__ void count_parts_kernel(const uint32_t* __restrict__ part, uint64_t n, uint32_t* __restrict__ counts) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) atomicAdd(&counts[part[i]], 1u);
}
__global__ void fill_u8_kernel(uint8_t* __restrict__ p, uint64_t n, uint8_t v) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

}  // extern "C"

// bit i of bitmap = RowIdMask::selected(row_ids[i]) (lance-core/src/utils/mask.rs:84-93); lists sorted
__global__ void row_mask_kernel(const uint64_t* __restrict__ row_ids, uint64_t n,
                                const uint64_t* __restrict__ allow, uint64_t n_allow, int has_allow,
                                const uint64_t* __restrict__ block, uint64_t n_block, int has_block,
                                uint32_t* __restrict__ bitmap32) {
  const uint64_t pos = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;  // n padded to 64 by the grid
  bool sel = false;
  if (pos < n) {
    const uint64_t id = row_ids[pos];
    sel = (!has_allow || sorted_contains(allow, n_allow, id)) && !(has_block && sorted_contains(block, n_block, id));
  }
  const unsigned bal = __ballot_sync(0xffffffffu, sel);
  // the bitmap holds ceil(n / 64) u64 words; the last CTA may reach beyond it
  if ((threadIdx.x & 31) == 0 && (pos >> 5) < ((n + 63) / 64) * 2) bitmap32[pos >> 5] = bal;
}
static void row_mask_f32(const uint64_t* row_ids, uint64_t n, const uint64_t* allow, uint64_t n_allow, bool has_allow,
                  const uint64_t* block, uint64_t n_block, bool has_block, uint64_t* bitmap) {
  const uint64_t padded = (n + 63) / 64 * 64;
  if (padded == 0) return;
  LB2_LAUNCH("row_mask", row_mask_kernel, cdiv(padded, 256), 256, 0, row_ids, n, allow, n_allow,
             has_allow ? 1 : 0, block, n_block, has_block ? 1 : 0, reinterpret_cast<uint32_t*>(bitmap));
}

// the kept graphs of a merge (lb2_optimize_params' rule): new partition p keeps old partition q's graph when q lost no
// row, nothing was added to p, and p holds exactly q's rows (then no other old partition sent p a row)
static HnswKeep kept_partitions(const lb2_index* old, const lb2_index* ix, const uint32_t* part_map,
                                const uint32_t* dropped, const uint32_t* added) {
  HnswKeep keep;
  keep.old = old->hnsw.get();
  const int ok = old->K, nk = ix->K;
  keep.old_off.resize(ok + 1);
  std::vector<uint64_t> noff(nk + 1);
  std::vector<uint32_t> pm(part_map ? ok : 0), dr(ok), ad(nk);
  d2h(keep.old_off.data(), old->part_offsets.p, (size_t)ok + 1);
  d2h(noff.data(), ix->part_offsets.p, (size_t)nk + 1);
  if (part_map) d2h(pm.data(), part_map, (size_t)ok);
  d2h(dr.data(), dropped, (size_t)ok);
  d2h(ad.data(), added, (size_t)nk);
  sync_stream();
  keep.src.assign(nk, -1);
  for (int q = 0; q < ok; ++q) {
    const uint32_t p = part_map ? pm[q] : (uint32_t)q;
    const uint64_t rows = keep.old_off[q + 1] - keep.old_off[q];
    if (p == 0xffffffffu || rows == 0 || dr[q] || ad[p] || noff[p + 1] - noff[p] != rows) continue;
    keep.src[p] = q;
  }
  return keep;
}

// rows per partition id among the rows with valid[i] != 0
__global__ void count_valid_parts_kernel(const uint32_t* __restrict__ part, const uint8_t* __restrict__ valid,
                                         uint64_t n, uint32_t* __restrict__ counts) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && valid[i]) atomicAdd(&counts[part[i]], 1u);
}

// lb2_index_optimize's merge (and lb2_index_update's, lb2_index_split's and lb2_index_join's); `what` names the entry
// point in messages.  add_valid (nullable, device [n_add]): added rows with 0 are left out.
std::unique_ptr<lb2_index> index_merge(const lb2_index* old, const lb2_optimize_params& p, const char* what,
                                       const uint8_t* add_valid) {
  const bool rq = old->kind == IndexKind::RQ;
  const uint32_t new_k = p.new_k;
  LB2_REQUIRE(new_k > 0 && (p.new_centroids || new_k == (uint32_t)old->K), "a changed partition count needs new centroids");
  LB2_REQUIRE(p.n_add == 0 || (p.add_part_ids && p.add_payload && p.add_row_ids),
              "%s: added rows need partition ids, payload and row ids", what);
  if (rq)
    LB2_REQUIRE(p.n_add == 0 || (p.add_rq_add && p.add_rq_scale), "%s: IVF_RQ rows need their add and scale factors",
                what);
  else
    LB2_REQUIRE(!p.add_rq_add && !p.add_rq_scale, "%s: add and scale factors are for IVF_RQ indexes only", what);
  LB2_REQUIRE(p.n_remove == 0 || p.remove_row_ids, "null remove list");
  LB2_REQUIRE(p.n_remap == 0 || (p.remap_old_ids && p.remap_new_ids), "%s: null remap list", what);
  if (old->hnsw && comm_nranks() > 1)
    fail(LB2_UNSUPPORTED, "%s: %s indexes over more than one rank are not implemented", what, old->hnsw->kind);
  if (old->hnsw)
    LB2_REQUIRE(p.insert_batch <= 65536, "%s: insert_batch must be at most 65536, got %u", what, p.insert_batch);
  const int rb = (int)old->row_bytes();
  const uint64_t n_old = old->n, n_add = p.n_add, n_all = n_old + n_add;
  LB2_REQUIRE(n_all < 0xffffffffull, "more than 2^32-1 rows per index shard");
  std::unique_ptr<lb2_index> ix = make_index(old->kind, new_k, old->d, old->metric, old->dtype);
  copy_model(old, ix.get(), p.new_centroids);
  InArg<uint32_t> pm(p.part_map, p.part_map ? (size_t)old->K : 0), ap(p.add_part_ids, n_add);
  InArg<uint8_t> ac(p.add_payload, (size_t)n_add * rb);
  InArg<float> aa(p.add_rq_add, rq ? n_add : 0), as(p.add_rq_scale, rq ? n_add : 0);
  InArg<uint64_t> ar(p.add_row_ids, n_add), rm(p.remove_row_ids, p.n_remove), ro(p.remap_old_ids, p.n_remap),
      rn(p.remap_new_ids, p.n_remap);
  if (n_add) check_part_ids(ap.get(), n_add, new_k, what);
  // one row list: old rows in storage order, then the added rows (so a partition keeps its old rows first)
  DevBuf<uint32_t> part(std::max<uint64_t>(1, n_all)), bad(2), dropped, added;
  DevBuf<uint8_t> valid(std::max<uint64_t>(1, n_all)), payload(std::max<uint64_t>(1, n_all * rb));
  DevBuf<uint64_t> rid(std::max<uint64_t>(1, n_all));
  DevBuf<float> fa, fs;
  bad.zero();
  if (old->hnsw) {  // what the graph kinds need to find the unchanged partitions
    dropped.alloc(old->K);
    dropped.zero();
    added.alloc(new_k);
    added.zero();
    if (n_add && add_valid)
      LB2_LAUNCH("count_added", count_valid_parts_kernel, cdiv(n_add, 256), 256, 0, ap.get(), add_valid, n_add, added.p);
    else if (n_add)
      LB2_LAUNCH("count_added", count_parts_kernel, cdiv(n_add, 256), 256, 0, ap.get(), n_add, added.p);
  }
  if (rq) {
    fa.alloc(std::max<uint64_t>(1, n_all));
    fs.alloc(std::max<uint64_t>(1, n_all));
  }
  if (p.n_remap > 1)
    LB2_LAUNCH("remap_order", remap_order_kernel, cdiv(p.n_remap, 256), 256, 0, ro.get(), p.n_remap, bad.p + 1);
  if (n_old) {
    LB2_LAUNCH("update_old_rows", update_old_rows_kernel, cdiv(n_old, 256), 256, 0, old->part_offsets.p, old->K, n_old,
               pm.get(), (const uint64_t*)old->row_ids.p, rm.get(), p.n_remove, new_k, part.p, valid.p, bad.p,
               dropped.p);
    d2d(payload.p, old->payload().p, (size_t)n_old * rb);
    d2d(rid.p, old->row_ids.p, (size_t)n_old);
    if (rq) {
      d2d(fa.p, old->rq_add.p, (size_t)n_old);
      d2d(fs.p, old->rq_scale.p, (size_t)n_old);
    }
  }
  if (n_add) {
    d2d(part.p + n_old, ap.get(), (size_t)n_add);
    d2d(payload.p + n_old * rb, ac.get(), (size_t)n_add * rb);
    d2d(rid.p + n_old, ar.get(), (size_t)n_add);
    if (rq) {
      d2d(fa.p + n_old, aa.get(), (size_t)n_add);
      d2d(fs.p + n_old, as.get(), (size_t)n_add);
    }
    if (add_valid)
      d2d(valid.p + n_old, add_valid, (size_t)n_add);
    else
      LB2_LAUNCH("fill_valid", fill_u8_kernel, cdiv(n_add, 256), 256, 0, valid.p + n_old, n_add, (uint8_t)1);
  }
  uint32_t hbad[2] = {0, 0};
  d2h(hbad, bad.p, 2);
  sync_stream();
  if (hbad[0]) fail(LB2_INVALID_ARG, "%s: part_map sends a partition to %u, the new index has %u partitions", what, hbad[0], new_k);
  if (hbad[1]) fail(LB2_INVALID_ARG, "%s: the remap's old row ids are not strictly ascending", what);
  if (p.n_remap && n_all)
    LB2_LAUNCH("remap_rows", remap_rows_kernel, cdiv(n_all, 256), 256, 0, rid.p, valid.p, n_all, ro.get(), rn.get(),
               p.n_remap, old->part_offsets.p, old->K, n_old, dropped.p);
  index_load_dev(ix.get(), part.p, payload.p, rid.p, n_all, valid.p, fa.p, fs.p);
  set_partition_index(ix.get(), old->pi_mode, old->pi_seed, old->pi_batch);  // the rule, over the new centroids
  if (old->hnsw) {
    const HnswGraph& og = *old->hnsw;
    const HnswKeep keep = kept_partitions(old, ix.get(), pm.get(), dropped.p, added.p);
    attach_graph(ix.get(), og.max_level, og.m, og.ef_construction, p.insert_batch ? p.insert_batch : og.insert_batch,
                 p.seed, &keep);
  }
  sync_stream();
  return ix;
}

}  // namespace lb2

using namespace lb2;

extern "C" {

lb2_status lb2_index_create(const void* centroids, uint32_t k, uint32_t d, lb2_dtype dtype,
                            lb2_metric metric, const void* codebook, uint32_t num_sub_vectors,
                            uint32_t num_bits, lb2_index** out) {
  LB2_API_BEGIN
  LB2_REQUIRE(out && centroids && codebook, "null argument");
  check_pq_shape(d, num_sub_vectors, num_bits, PqUse::ENCODE);
  std::unique_ptr<lb2_index> ix = index_with_centroids(IndexKind::PQ, centroids, k, d, dtype, metric);
  ix->M = num_sub_vectors;
  ix->nbits = num_bits;
  ix->codebook.alloc(ix->codebook_len());
  {
    VecIn cb(codebook, ix->codebook_len(), model_dtype(dtype));
    d2d(ix->codebook.p, cb.get(), ix->codebook_len());
    sync_stream();
  }
  *out = ix.release();
  LB2_API_END
}

lb2_status lb2_index_create_flat(const void* centroids, uint32_t k, uint32_t d, lb2_dtype dtype,
                                 lb2_metric metric, lb2_index** out) {
  LB2_API_BEGIN
  LB2_REQUIRE(out && centroids, "null argument");
  *out = index_with_centroids(IndexKind::FLAT, centroids, k, d, dtype, metric).release();
  LB2_API_END
}

lb2_status lb2_index_create_sq(const void* centroids, uint32_t k, uint32_t d, lb2_dtype dtype, lb2_metric metric,
                               double lower, double upper, lb2_index** out) {
  LB2_API_BEGIN
  LB2_REQUIRE(out && centroids, "null argument");
  sq_check_dim(d);
  LB2_REQUIRE(std::isfinite(lower) && std::isfinite(upper) && lower <= upper,
              "IVF_SQ: the bounds must be finite with lower <= upper, got [%g, %g]", lower, upper);
  std::unique_ptr<lb2_index> ix = index_with_centroids(IndexKind::SQ, centroids, k, d, dtype, metric);
  ix->nbits = 8;
  ix->sq_lower = lower;
  ix->sq_upper = upper;
  *out = ix.release();
  LB2_API_END
}

lb2_status lb2_index_create_rq(const void* centroids, uint32_t k, uint32_t d, lb2_dtype dtype, lb2_metric metric,
                               const void* rotation, uint32_t num_bits, lb2_index** out) {
  LB2_API_BEGIN
  LB2_REQUIRE(out && centroids && rotation, "null argument");
  rq_check(d, dtype, num_bits);
  std::unique_ptr<lb2_index> ix = index_with_centroids(IndexKind::RQ, centroids, k, d, dtype, metric);
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

lb2_status lb2_index_load(lb2_index* index, const uint32_t* part_ids, const uint8_t* codes,
                          const uint64_t* row_ids, uint64_t n) {
  LB2_API_BEGIN
  LB2_REQUIRE(index && index->kind == IndexKind::PQ, "not an IVF_PQ index");
  LB2_REQUIRE(!index->hnsw, "lb2_index_load: the index already has an HNSW graph over its rows");
  load_codes(index, part_ids, codes, row_ids, n, "index_load");
  LB2_API_END
}

lb2_status lb2_index_load_flat(lb2_index* index, const uint32_t* part_ids, const void* vectors,
                               const uint64_t* row_ids, uint64_t n) {
  LB2_API_BEGIN
  LB2_REQUIRE(index && index->kind == IndexKind::FLAT, "not an IVF_FLAT index");
  LB2_REQUIRE(!index->hnsw, "lb2_index_load_flat: the IVF_HNSW_FLAT index already has an HNSW graph over its rows");
  LB2_REQUIRE(index->d % 4 == 0, "IVF_FLAT needs a dimension that is a multiple of 4");
  InArg<uint32_t> p(part_ids, n);
  InArg<uint64_t> r(row_ids, n);
  check_part_ids(p.get(), n, (uint32_t)index->K, "index_load_flat");
  Source src(vectors, n, index->d, index->dtype);
  src.start_resident_copy();
  index_load_flat_src(index, p.get(), src, r.get(), nullptr, /*normalize=*/false);
  LB2_API_END
}

lb2_status lb2_index_load_sq(lb2_index* index, const uint32_t* part_ids, const uint8_t* codes,
                             const uint64_t* row_ids, uint64_t n) {
  LB2_API_BEGIN
  LB2_REQUIRE(index && index->kind == IndexKind::SQ, "not an IVF_SQ index");
  LB2_REQUIRE(!index->hnsw, "lb2_index_load_sq: the index already has an HNSW graph over its rows");
  load_codes(index, part_ids, codes, row_ids, n, "index_load_sq");
  LB2_API_END
}

lb2_status lb2_index_load_rq(lb2_index* index, const uint32_t* part_ids, const uint8_t* codes, const float* add_factors,
                             const float* scale_factors, const uint64_t* row_ids, uint64_t n) {
  LB2_API_BEGIN
  LB2_REQUIRE(index && index->kind == IndexKind::RQ, "not an IVF_RQ index");
  LB2_REQUIRE(n == 0 || (part_ids && codes && add_factors && scale_factors), "null argument");
  load_codes(index, part_ids, codes, row_ids, n, "index_load_rq", add_factors, scale_factors);
  LB2_API_END
}

lb2_status lb2_index_export(const lb2_index* index, void* centroids_out, void* codebook_out,
                            uint64_t* part_offsets_out, uint8_t* codes_out, uint64_t* row_ids_out) {
  LB2_API_BEGIN
  LB2_REQUIRE(index && index->kind == IndexKind::PQ, "not an IVF_PQ index");
  export_common(index, centroids_out, part_offsets_out, codes_out, row_ids_out);
  if (codebook_out)
    LB2_CUDA(cudaMemcpyAsync(codebook_out, index->codebook.p, sizeof(float) * index->codebook_len(), cudaMemcpyDefault,
                             ctx().stream));
  sync_stream();
  LB2_API_END
}

lb2_status lb2_index_export_flat(const lb2_index* index, void* centroids_out,
                                 uint64_t* part_offsets_out, void* vectors_out,
                                 uint64_t* row_ids_out) {
  LB2_API_BEGIN
  LB2_REQUIRE(index && index->kind == IndexKind::FLAT, "not an IVF_FLAT index");
  export_common(index, centroids_out, part_offsets_out, vectors_out, row_ids_out);
  sync_stream();
  LB2_API_END
}

lb2_status lb2_index_export_sq(const lb2_index* index, void* centroids_out, double* bounds_out,
                               uint64_t* part_offsets_out, uint8_t* codes_out, uint64_t* row_ids_out) {
  LB2_API_BEGIN
  LB2_REQUIRE(index && index->kind == IndexKind::SQ, "not an IVF_SQ index");
  if (bounds_out) {
    bounds_out[0] = index->sq_lower;
    bounds_out[1] = index->sq_upper;
  }
  export_common(index, centroids_out, part_offsets_out, codes_out, row_ids_out);
  sync_stream();
  LB2_API_END
}

}  // extern "C"

namespace lb2 {

const char* hnsw_kind_name(IndexKind kind) {
  return kind == IndexKind::SQ ? "IVF_HNSW_SQ" : kind == IndexKind::PQ ? "IVF_HNSW_PQ" : "IVF_HNSW_FLAT";
}

std::unique_ptr<HnswGraph> new_graph(IndexKind kind, uint32_t max_level, uint32_t m, uint32_t ef_construction,
                                     uint32_t insert_batch) {
  LB2_REQUIRE(max_level >= 1 && max_level <= 64 && m >= 1 && m <= 1024, "%s: max_level %u or m %u out of range",
              hnsw_kind_name(kind), max_level, m);
  std::unique_ptr<HnswGraph> g(new HnswGraph());
  g->kind = hnsw_kind_name(kind);
  g->max_level = (int)max_level;
  g->m = (int)m;
  g->ef_construction = (int)ef_construction;
  g->insert_batch = std::max<uint32_t>(insert_batch, 1);
  return g;
}

void set_partition_index(lb2_index* ix, uint32_t mode, uint64_t seed, uint32_t insert_batch) {
  PartitionIndexPtr pi = partition_index_make(ix->centroids.p, (uint32_t)ix->K, (uint32_t)ix->d, ix->dtype,
                                              ix->metric == METRIC_DOT ? METRIC_DOT : METRIC_L2, mode, seed,
                                              insert_batch);
  ix->pi_mode = mode;
  ix->pi_seed = seed;
  ix->pi_batch = std::max<uint32_t>(insert_batch, 1);
  ix->pidx = std::move(pi);
}

void attach_graph(lb2_index* ix, uint32_t max_level, uint32_t m, uint32_t ef_construction, uint32_t insert_batch,
                  uint64_t seed, const HnswKeep* keep) {
  TagScope tg("hnsw_build");
  std::unique_ptr<HnswGraph> g = new_graph(ix->kind, max_level, m, ef_construction, insert_batch);
  ix->slab_off.release();  // the skewed code copy serves only the IVF_PQ scan
  ix->codes_skew.release();
  hnsw_build(*g, *ix, seed, keep);
  ix->hnsw = std::move(g);
}

}  // namespace lb2

// lb2_index_load_hnsw_sq / _pq / _flat: a graph over the rows of an index of `kind`
static void load_hnsw(lb2_index* index, IndexKind kind, uint32_t max_level, uint32_t m, uint32_t ef_construction,
                      const uint8_t* levels, const uint32_t* counts0, const uint32_t* neighbors0, const float* dists0,
                      const uint32_t* counts_up, const uint32_t* neighbors_up, const float* dists_up) {
  // the refusal names the index kind, IVF_SQ, IVF_PQ or IVF_FLAT: the graph kind's name past "IVF_HNSW_"
  LB2_REQUIRE(index && index->kind == kind, "not an IVF_%s index", hnsw_kind_name(kind) + strlen("IVF_HNSW_"));
  std::unique_ptr<HnswGraph> g = new_graph(kind, max_level, m, ef_construction);
  hnsw_load(*g, index->part_offsets.p, index->K, levels, counts0, neighbors0, dists0, counts_up, neighbors_up, dists_up);
  index->hnsw = std::move(g);
}

// lb2_index_hnsw_*_info / lb2_index_export_hnsw_*: the graph of an index of `kind`
static const HnswGraph& graph_of(const lb2_index* index, IndexKind kind) {
  LB2_REQUIRE(index && index->hnsw && index->kind == kind, "not an %s index", hnsw_kind_name(kind));
  return *index->hnsw;
}
static void hnsw_info(const HnswGraph& g, uint32_t* max_level, uint32_t* m, uint32_t* ef_construction,
                      uint64_t* num_upper_rows) {
  if (max_level) *max_level = (uint32_t)g.max_level;
  if (m) *m = (uint32_t)g.m;
  if (ef_construction) *ef_construction = (uint32_t)g.ef_construction;
  if (num_upper_rows) *num_upper_rows = g.n_up;
}
static void export_hnsw(const lb2_index* index, const HnswGraph& g, uint8_t* levels_out, uint32_t* counts0_out,
                        uint32_t* neighbors0_out, float* dists0_out, uint32_t* counts_up_out,
                        uint32_t* neighbors_up_out, float* dists_up_out) {
  const size_t n = index->n, nu = g.n_up, m = (size_t)g.m;
  cudaStream_t st = ctx().stream;
  auto out = [&](void* dst, const void* src, size_t bytes) {
    if (dst && bytes) LB2_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDefault, st));
  };
  out(levels_out, g.nlev.p, n);
  out(counts0_out, g.cnt0.p, 4 * n);
  out(neighbors0_out, g.nbr0.p, 4 * n * 2 * m);
  out(dists0_out, g.dst0.p, 4 * n * 2 * m);
  out(counts_up_out, g.cntu.p, 4 * nu);
  out(neighbors_up_out, g.nbru.p, 4 * nu * m);
  out(dists_up_out, g.dstu.p, 4 * nu * m);
  sync_stream();
}

extern "C" {

lb2_status lb2_index_load_hnsw_sq(lb2_index* index, uint32_t max_level, uint32_t m, uint32_t ef_construction,
                                  const uint8_t* levels, const uint32_t* counts0, const uint32_t* neighbors0,
                                  const float* dists0, const uint32_t* counts_up, const uint32_t* neighbors_up,
                                  const float* dists_up) {
  LB2_API_BEGIN
  load_hnsw(index, IndexKind::SQ, max_level, m, ef_construction, levels, counts0, neighbors0, dists0,
            counts_up, neighbors_up, dists_up);
  LB2_API_END
}

lb2_status lb2_index_load_hnsw_pq(lb2_index* index, uint32_t max_level, uint32_t m, uint32_t ef_construction,
                                  const uint8_t* levels, const uint32_t* counts0, const uint32_t* neighbors0,
                                  const float* dists0, const uint32_t* counts_up, const uint32_t* neighbors_up,
                                  const float* dists_up) {
  LB2_API_BEGIN
  load_hnsw(index, IndexKind::PQ, max_level, m, ef_construction, levels, counts0, neighbors0, dists0,
            counts_up, neighbors_up, dists_up);
  LB2_API_END
}

lb2_status lb2_index_load_hnsw_flat(lb2_index* index, uint32_t max_level, uint32_t m, uint32_t ef_construction,
                                    const uint8_t* levels, const uint32_t* counts0, const uint32_t* neighbors0,
                                    const float* dists0, const uint32_t* counts_up, const uint32_t* neighbors_up,
                                    const float* dists_up) {
  LB2_API_BEGIN
  load_hnsw(index, IndexKind::FLAT, max_level, m, ef_construction, levels, counts0, neighbors0,
            dists0, counts_up, neighbors_up, dists_up);
  LB2_API_END
}

lb2_status lb2_index_hnsw_sq_info(const lb2_index* index, uint32_t* max_level, uint32_t* m, uint32_t* ef_construction,
                                  uint64_t* num_upper_rows) {
  LB2_API_BEGIN
  hnsw_info(graph_of(index, IndexKind::SQ), max_level, m, ef_construction, num_upper_rows);
  LB2_API_END
}

lb2_status lb2_index_hnsw_pq_info(const lb2_index* index, uint32_t* max_level, uint32_t* m, uint32_t* ef_construction,
                                  uint64_t* num_upper_rows) {
  LB2_API_BEGIN
  hnsw_info(graph_of(index, IndexKind::PQ), max_level, m, ef_construction, num_upper_rows);
  LB2_API_END
}

lb2_status lb2_index_hnsw_flat_info(const lb2_index* index, uint32_t* max_level, uint32_t* m,
                                    uint32_t* ef_construction, uint64_t* num_upper_rows) {
  LB2_API_BEGIN
  hnsw_info(graph_of(index, IndexKind::FLAT), max_level, m, ef_construction, num_upper_rows);
  LB2_API_END
}

lb2_status lb2_index_export_hnsw_sq(const lb2_index* index, uint8_t* levels_out, uint32_t* counts0_out,
                                    uint32_t* neighbors0_out, float* dists0_out, uint32_t* counts_up_out,
                                    uint32_t* neighbors_up_out, float* dists_up_out) {
  LB2_API_BEGIN
  export_hnsw(index, graph_of(index, IndexKind::SQ), levels_out, counts0_out, neighbors0_out,
              dists0_out, counts_up_out, neighbors_up_out, dists_up_out);
  LB2_API_END
}

lb2_status lb2_index_export_hnsw_pq(const lb2_index* index, uint8_t* levels_out, uint32_t* counts0_out,
                                    uint32_t* neighbors0_out, float* dists0_out, uint32_t* counts_up_out,
                                    uint32_t* neighbors_up_out, float* dists_up_out) {
  LB2_API_BEGIN
  export_hnsw(index, graph_of(index, IndexKind::PQ), levels_out, counts0_out, neighbors0_out,
              dists0_out, counts_up_out, neighbors_up_out, dists_up_out);
  LB2_API_END
}

lb2_status lb2_index_export_hnsw_flat(const lb2_index* index, uint8_t* levels_out, uint32_t* counts0_out,
                                      uint32_t* neighbors0_out, float* dists0_out, uint32_t* counts_up_out,
                                      uint32_t* neighbors_up_out, float* dists_up_out) {
  LB2_API_BEGIN
  export_hnsw(index, graph_of(index, IndexKind::FLAT), levels_out, counts0_out, neighbors0_out,
              dists0_out, counts_up_out, neighbors_up_out, dists_up_out);
  LB2_API_END
}

lb2_status lb2_index_export_rq(const lb2_index* index, void* centroids_out, void* rotation_out,
                               uint64_t* part_offsets_out, uint8_t* codes_out, float* add_out, float* scale_out,
                               uint64_t* row_ids_out) {
  LB2_API_BEGIN
  LB2_REQUIRE(index && index->kind == IndexKind::RQ, "not an IVF_RQ index");
  export_common(index, centroids_out, part_offsets_out, codes_out, row_ids_out);
  cudaStream_t s = ctx().stream;
  const size_t cd = index->code_dim(), n = index->n;
  if (rotation_out)
    LB2_CUDA(cudaMemcpyAsync(rotation_out, index->rq_rot.p, sizeof(float) * cd * cd, cudaMemcpyDefault, s));
  if (add_out && n) LB2_CUDA(cudaMemcpyAsync(add_out, index->rq_add.p, sizeof(float) * n, cudaMemcpyDefault, s));
  if (scale_out && n) LB2_CUDA(cudaMemcpyAsync(scale_out, index->rq_scale.p, sizeof(float) * n, cudaMemcpyDefault, s));
  sync_stream();
  LB2_API_END
}

lb2_status lb2_index_search(lb2_index* index, const void* queries, uint64_t nq, uint32_t k,
                            uint32_t nprobes, uint64_t* row_ids_out, float* dists_out,
                            uint32_t* counts_out) {
  LB2_API_BEGIN
  const lb2_search_params sp = {k, nprobes};
  index_search_impl(index, queries, nq, sp, row_ids_out, dists_out, counts_out);
  LB2_API_END
}

lb2_status lb2_index_search_refine(lb2_index* index, const void* vectors, uint64_t num_vectors,
                                   const void* queries, uint64_t nq, uint32_t k, uint32_t nprobes,
                                   uint32_t refine_factor, uint64_t* row_ids_out, float* dists_out,
                                   uint32_t* counts_out) {
  LB2_API_BEGIN
  LB2_REQUIRE(vectors && refine_factor > 0, "bad argument");
  const lb2_search_params sp = {k, nprobes, refine_factor, vectors, num_vectors};
  index_search_impl(index, queries, nq, sp, row_ids_out, dists_out, counts_out);
  LB2_API_END
}

lb2_status lb2_index_search_ex(lb2_index* index, const void* queries, uint64_t nq,
                               const lb2_search_params* sp, uint64_t* row_ids_out, float* dists_out,
                               uint32_t* counts_out) {
  LB2_API_BEGIN
  LB2_REQUIRE(sp, "null search params");
  LB2_REQUIRE(sp->refine_factor == 0 || sp->refine_vectors, "refine_factor > 0 needs refine_vectors");
  index_search_impl(index, queries, nq, *sp, row_ids_out, dists_out, counts_out);
  LB2_API_END
}

// the probe rule of lb2_index_search_probed, its checks and its staged arguments (alive as long as the object)
namespace {
struct ProbedSearch {
  InArg<uint64_t> mask;
  DevBuf<uint64_t> no_ids;  // an iterable, empty allow list
  OutArg<uint32_t> np_out;
  ProbeRule pr;
  ProbedSearch(const lb2_search_params* sp, const lb2_probe_params* pp, uint64_t nq, uint32_t* nprobes_out) {
    LB2_REQUIRE(sp->nprobes == 0, "nprobes must be 0: the probe parameters decide the probes");
    LB2_REQUIRE(sp->refine_factor == 0 || sp->refine_vectors, "refine_factor > 0 needs refine_vectors");
    LB2_REQUIRE(pp->minimum_nprobes >= 1, "minimum_nprobes must be at least 1");
    LB2_REQUIRE(pp->maximum_nprobes == 0 || pp->maximum_nprobes >= pp->minimum_nprobes,
                "maximum_nprobes %u is below minimum_nprobes %u", pp->maximum_nprobes, pp->minimum_nprobes);
    LB2_REQUIRE(pp->late_width >= 1, "late_width must be at least 1");
    LB2_REQUIRE(sp->allow_bitmap || (!pp->has_max_len && !pp->mask_ids), "max_len and mask_ids need an allow bitmap");
    if (current_comm() && current_comm()->nranks > 1)
      fail(LB2_UNSUPPORTED, "a search with minimum / maximum nprobes on a row-sharded index is not implemented");
    mask.set(pp->mask_ids, pp->mask_ids ? pp->num_mask_ids : 0);
    if (pp->mask_ids && pp->num_mask_ids == 0) no_ids.alloc(1);
    np_out.set(nprobes_out, nq);
    pr.min_np = pp->minimum_nprobes;
    pr.max_np = pp->maximum_nprobes;
    pr.late_width = pp->late_width;
    pr.k = sp->k;
    pr.has_max_len = pp->has_max_len != 0;
    pr.max_len = pp->max_len;
    pr.mask_ids = pp->mask_ids ? (mask.get() ? mask.get() : no_ids.p) : nullptr;
    pr.num_mask_ids = pp->mask_ids ? pp->num_mask_ids : 0;
    pr.nprobes_out = np_out.get();
  }
};
}  // namespace

lb2_status lb2_index_search_probed(lb2_index* index, const void* queries, uint64_t nq, const lb2_search_params* sp,
                                   const lb2_probe_params* pp, uint64_t* row_ids_out, float* dists_out,
                                   uint32_t* counts_out, uint32_t* nprobes_out) {
  LB2_API_BEGIN
  LB2_REQUIRE(sp && pp && index, "null argument");
  ProbedSearch ps(sp, pp, nq, nprobes_out);
  index_search_impl(index, queries, nq, *sp, row_ids_out, dists_out, counts_out, &ps.pr);
  ps.np_out.commit();
  sync_stream();
  LB2_API_END
}

lb2_status lb2_index_search_hnsw(lb2_index* index, const void* queries, uint64_t nq, const lb2_search_params* sp,
                                 const lb2_probe_params* pp, uint32_t ef, uint64_t* row_ids_out, float* dists_out,
                                 uint32_t* counts_out, uint32_t* nprobes_out) {
  LB2_API_BEGIN
  LB2_REQUIRE(sp && index, "null argument");
  LB2_REQUIRE(index->hnsw, "not an IVF_HNSW_SQ, IVF_HNSW_PQ or IVF_HNSW_FLAT index");
  LB2_REQUIRE(!nprobes_out || pp, "nprobes_out needs probe parameters");
  if (pp) {
    ProbedSearch ps(sp, pp, nq, nprobes_out);
    index_search_impl(index, queries, nq, *sp, row_ids_out, dists_out, counts_out, &ps.pr, ef);
    ps.np_out.commit();
  } else {
    LB2_REQUIRE(sp->refine_factor == 0 || sp->refine_vectors, "refine_factor > 0 needs refine_vectors");
    index_search_impl(index, queries, nq, *sp, row_ids_out, dists_out, counts_out, nullptr, ef);
  }
  sync_stream();
  LB2_API_END
}

// A batch of queries with their own parameters in one pass (include/lance_b200.h).  Every query's own call is
// checked first, so a refusal writes nothing.  The filters are staged once; each query's k', filter, range and ef
// go to the device as one QueryParam per query for the scan kernels and one QueryOut per query for the finish
// (refine or copy to rows of k_stride).  The lists are as long as the batch's largest k' and the probe grid as wide
// as its largest nprobes; a query's other slots probe the empty partition.  A batch with minimum / maximum nprobes
// queries runs the probe rule for every query, each with its own QueryProbe: a fixed nprobes p is minimum = maximum =
// p, which lb2_index_search_probed defines to equal lb2_index_search_ex.
// lb2_index_search_batch and lb2_index_search_candidates share everything up to the merged candidate lists:
// BatchPlan checks the batch (have_vectors: refine_factor > 0 is allowed), BatchSearch runs it.
namespace {
struct BatchPlan {
  uint32_t kmax = 0, kcmax = 0, npmax = 0, efmax = 0, Lmax = 0;
  bool any_refine = false, any_filter = false, any_range = false, any_probed = false;
  BatchPlan(const lb2_index* index, const void* queries, uint64_t nq, const lb2_query_params* params,
            const lb2_query_filter* filters, uint32_t num_filters, uint32_t late_width, bool have_vectors) {
    LB2_REQUIRE(index, "null index");
    LB2_REQUIRE(nq == 0 || (queries && params), "null queries or params");
    LB2_REQUIRE(num_filters == 0 || filters, "null filters");
    LB2_REQUIRE(late_width >= 1, "late_width must be at least 1");
    const uint32_t K = (uint32_t)index->K;
    for (uint64_t q = 0; q < nq; ++q) {
      const lb2_query_params& p = params[q];
      const unsigned long long qi = (unsigned long long)q;
      LB2_REQUIRE(p.k > 0, "query %llu: k must be positive", qi);
      LB2_REQUIRE(p.filter < num_filters || p.filter == UINT32_MAX, "query %llu: filter %u is not below num_filters %u",
                  qi, p.filter, num_filters);
      LB2_REQUIRE(p.ef == 0 || index->hnsw, "query %llu: ef is set on an index without HNSW graphs", qi);
      LB2_REQUIRE(p.refine_factor == 0 || have_vectors, "query %llu: refine_factor > 0 needs refine_vectors", qi);
      if (p.nprobes == 0) {  // lb2_index_search_probed's checks
        LB2_REQUIRE(p.minimum_nprobes >= 1, "query %llu: minimum_nprobes must be at least 1", qi);
        LB2_REQUIRE(p.maximum_nprobes == 0 || p.maximum_nprobes >= p.minimum_nprobes,
                    "query %llu: maximum_nprobes %u is below minimum_nprobes %u", qi, p.maximum_nprobes,
                    p.minimum_nprobes);
        LB2_REQUIRE(p.filter == UINT32_MAX || filters[p.filter].allow_bitmap ||
                        (!filters[p.filter].has_max_len && !filters[p.filter].mask_ids),
                    "query %llu: max_len and mask_ids need an allow bitmap", qi);
        any_probed = true;
      }
      const uint64_t kc = (uint64_t)p.k * std::max<uint32_t>(1, p.refine_factor);
      if (kc > 1024)
        fail(LB2_UNSUPPORTED, "query %llu: k * refine_factor = %llu > 1024 is not implemented", qi, (unsigned long long)kc);
      const uint32_t ef = p.ef ? p.ef : (uint32_t)(kc + kc / 2);
      if (index->hnsw && ef < kc)
        fail(LB2_INVALID_ARG, "query %llu: %s: ef = %u must be greater than or equal to k = %u", qi, index->hnsw->kind,
             ef, (uint32_t)kc);
      kmax = std::max(kmax, p.k);
      kcmax = std::max(kcmax, (uint32_t)kc);
      npmax = std::max(npmax, std::min(p.nprobes, K));
      const uint32_t mx = p.nprobes ? p.nprobes : p.maximum_nprobes;
      Lmax = std::max(Lmax, mx ? std::min(mx, K) : K);
      efmax = std::max(efmax, ef);
      any_refine |= p.refine_factor > 0;
      any_filter |= p.filter != UINT32_MAX || p.has_lower_bound || p.has_upper_bound;
      any_range |= p.has_lower_bound || p.has_upper_bound;
    }
  }
};

// the batch's scan up to the merged lists: cid / cdist [nq][kcmax], ccnt [nq], each query's QueryOut in qo; nprobes
// (device, nullable) receives nprobes_out.  nq > 0.
struct BatchSearch {
  const SearchQueries q;
  DevBuf<uint64_t> cid;
  DevBuf<float> cdist;
  DevBuf<uint32_t> ccnt;
  DevBuf<QueryOut> qo;
  std::vector<uint32_t> qnp_h;
  BatchSearch(lb2_index* index, const void* queries, uint64_t nq, const lb2_query_params* params,
              const lb2_query_filter* filters, uint32_t num_filters, uint32_t late_width, const BatchPlan& b,
              uint32_t* nprobes)
      : q(index, queries, nq), cid((size_t)nq * b.kcmax), cdist((size_t)nq * b.kcmax), ccnt(nq), qo(nq), qnp_h(nq) {
    const uint32_t K = (uint32_t)index->K;
    const int d = index->d;
    // the filters, staged once each (with the probe rule also their allow lists' ids), and their allowed rows per
    // partition in one launch: IVF_HNSW_*'s `remained`, and the probe rule's c_p (row num_filters: no prefilter)
    const size_t words = (size_t)((index->n + 63) / 64);
    std::vector<InArg<uint64_t>> allow(num_filters), ids(num_filters);
    std::vector<const uint64_t*> allow_h(num_filters + 1, nullptr), ids_h(num_filters, nullptr);
    DevBuf<uint64_t> no_ids(1);  // an iterable, empty allow list
    for (uint32_t f = 0; f < num_filters; ++f) {
      allow[f].set(filters[f].allow_bitmap, filters[f].allow_bitmap ? words : 0);
      allow_h[f] = allow[f].get();
      if (b.any_probed && filters[f].mask_ids) {
        ids[f].set(filters[f].mask_ids, filters[f].num_mask_ids);
        ids_h[f] = ids[f].get() ? ids[f].get() : no_ids.p;
      }
    }
    DevBuf<uint32_t> acnt;
    if ((index->hnsw && num_filters) || b.any_probed) {
      DevBuf<const uint64_t*> tab(num_filters + 1);
      h2d(tab.p, allow_h.data(), num_filters + 1);
      acnt.alloc((size_t)(num_filters + 1) * K);
      partition_counts_table(index->part_offsets.p, (int)K, tab.p, (int)num_filters + 1, acnt.p);
    }
    std::vector<QueryProbe> qpr_h(b.any_probed ? nq : 0);
    bool any_iterable = false;
    std::vector<QueryParam> qp_h(nq);
    std::vector<QueryOut> qo_h(nq);
    for (uint64_t i = 0; i < nq; ++i) {
      const lb2_query_params& p = params[i];
      const bool filtered = p.filter != UINT32_MAX && allow_h[p.filter];
      const int kc = (int)p.k * (int)std::max<uint32_t>(1, p.refine_factor);
      qp_h[i].flt = make_filter(filtered ? allow_h[p.filter] : nullptr, p.has_lower_bound != 0, p.lower_bound,
                                p.has_upper_bound != 0, p.upper_bound);
      qp_h[i].k = kc;
      qp_h[i].ef = p.ef ? p.ef : (uint32_t)(kc + kc / 2);
      qp_h[i].acnt = filtered && acnt.p ? acnt.p + (size_t)p.filter * K : nullptr;
      qo_h[i] = QueryOut{kc, (int)p.k, p.refine_factor > 0, (int)(p.has_lower_bound != 0),
                         (int)(p.has_upper_bound != 0), p.lower_bound, p.upper_bound};
      qnp_h[i] = std::min(p.nprobes, K);
      if (b.any_probed) {  // a fixed nprobes p: minimum = maximum = p, no shortcut
        const uint32_t f = p.filter == UINT32_MAX ? num_filters : p.filter;
        const bool probed = p.nprobes == 0;
        const uint32_t mx = probed ? p.maximum_nprobes : p.nprobes;
        const uint64_t* mids = probed && f < num_filters ? ids_h[f] : nullptr;
        qpr_h[i] = QueryProbe{probed ? p.minimum_nprobes : p.nprobes, mx ? std::min(mx, K) : K, p.k, (uint32_t)kc,
                              p.has_lower_bound || p.has_upper_bound, probed && f < num_filters && filters[f].has_max_len,
                              probed && f < num_filters ? filters[f].max_len : 0, mids,
                              mids ? filters[f].num_mask_ids : 0, acnt.p + (size_t)(allow_h[f] ? f : num_filters) * K};
        any_iterable |= mids != nullptr;
      }
    }
    DevBuf<QueryParam> qp(nq);
    DevBuf<uint32_t> qnp(nq);
    h2d(qp.p, qp_h.data(), nq);
    h2d(qo.p, qo_h.data(), nq);
    h2d(qnp.p, qnp_h.data(), nq);
    DevBuf<QueryProbe> qpr(qpr_h.size());
    if (b.any_probed) h2d(qpr.p, qpr_h.data(), nq);
    TagScope tg("search");
    IvfSearch s{index->centroids.p, index->K, d, index->metric, index->part_offsets.p, index->row_ids.p, q.get(), nq,
                (int)b.kcmax, (int)b.npmax, cid.p, cdist.p, ccnt.p, ScanFilter{}, nullptr};
    s.qp = qp.p;
    s.qp_host = qp_h.data();
    s.qnp = qnp.p;
    s.any_filter = b.any_filter;
    s.any_range = b.any_range;
    ProbeRule pr;
    if (b.any_probed) {
      pr.max_np = b.Lmax;
      pr.late_width = late_width;
      pr.mask_ids = any_iterable ? no_ids.p : nullptr;  // non-null: lists get a shortcut slot
      pr.nprobes_out = nprobes;
      pr.qpr = qpr.p;
      s.pr = &pr;
    }
    search_kind(index, s, b.efmax);
    if (nprobes && !b.any_probed) h2d(nprobes, qnp_h.data(), nq);
  }
};
}  // namespace

lb2_status lb2_index_search_batch(lb2_index* index, const void* queries, uint64_t nq, const lb2_query_params* params,
                                  const lb2_query_filter* filters, uint32_t num_filters, const void* refine_vectors,
                                  uint64_t num_vectors, uint32_t late_width, uint32_t k_stride, uint64_t* row_ids_out,
                                  float* dists_out, uint32_t* counts_out, uint32_t* nprobes_out) {
  LB2_API_BEGIN
  const BatchPlan b(index, queries, nq, params, filters, num_filters, late_width, refine_vectors != nullptr);
  LB2_REQUIRE(k_stride >= b.kmax, "k_stride %u is below the largest k %u", k_stride, b.kmax);
  if (current_comm() && current_comm()->nranks > 1)
    fail(LB2_UNSUPPORTED, "a batch search on a row-sharded index is not implemented");
  if (nq == 0) {
    sync_stream();
    return LB2_OK;
  }
  const int d = index->d;
  OutArg<uint64_t> oi(row_ids_out, (size_t)nq * k_stride);
  OutArg<float> od(dists_out, (size_t)nq * k_stride);
  OutArg<uint32_t> oc(counts_out, nq);
  OutArg<uint32_t> onp(nprobes_out, nq);
  BatchSearch bs(index, queries, nq, params, filters, num_filters, late_width, b, onp.get());
  {
    TagScope tg("search");
    InArg<uint8_t> v(b.any_refine ? refine_vectors : nullptr, (size_t)num_vectors * d * dtype_size(index->dtype));
    refine_batch_f32(bs.q.q.get(), nq, d, index->metric, v.get(), (int)index->dtype, num_vectors, bs.cdist.p,
                     bs.cid.p, bs.ccnt.p, (int)b.kcmax, bs.qo.p, (int)k_stride, oi.get(), od.get(), oc.get());
  }
  oi.commit(); od.commit(); oc.commit(); onp.commit();
  sync_stream();
  LB2_API_END
}

// The index half of a refined batch (include/lance_b200.h): BatchSearch's merged lists, each query's k' of them, into
// rows of kc_stride, and optionally the batch's distinct row ids with every slot's position among them.
lb2_status lb2_index_search_candidates(lb2_index* index, const void* queries, uint64_t nq,
                                       const lb2_query_params* params, const lb2_query_filter* filters,
                                       uint32_t num_filters, uint32_t late_width, uint32_t kc_stride,
                                       uint64_t* cand_ids_out, float* cand_dists_out, uint32_t* cand_counts_out,
                                       uint32_t* nprobes_out, uint64_t* distinct_ids_out, uint64_t* num_distinct_out,
                                       uint64_t* positions_out) {
  LB2_API_BEGIN
  const BatchPlan b(index, queries, nq, params, filters, num_filters, late_width, true);
  LB2_REQUIRE(kc_stride >= b.kcmax, "kc_stride %u is below the largest k * max(1, refine_factor) %u", kc_stride,
              b.kcmax);
  LB2_REQUIRE(nq == 0 || (cand_ids_out && cand_dists_out && cand_counts_out), "null candidate outputs");
  LB2_REQUIRE(!distinct_ids_out == !positions_out && !distinct_ids_out == !num_distinct_out,
              "distinct_ids_out, num_distinct_out and positions_out go together");
  if (current_comm() && current_comm()->nranks > 1)
    fail(LB2_UNSUPPORTED, "a batch search on a row-sharded index is not implemented");
  const size_t slots = (size_t)nq * kc_stride;
  OutArg<uint64_t> om(num_distinct_out, 1);
  if (nq == 0) {
    if (om.get()) LB2_CUDA(cudaMemsetAsync(om.get(), 0, sizeof(uint64_t), ctx().stream));
    om.commit();
    sync_stream();
    return LB2_OK;
  }
  OutArg<uint64_t> oi(cand_ids_out, slots);
  OutArg<float> od(cand_dists_out, slots);
  OutArg<uint32_t> oc(cand_counts_out, nq);
  OutArg<uint32_t> onp(nprobes_out, nq);
  OutArg<uint64_t> odi(distinct_ids_out, slots), opos(positions_out, slots);
  BatchSearch bs(index, queries, nq, params, filters, num_filters, late_width, b, onp.get());
  {
    TagScope tg("search");
    candidate_rows(bs.cid.p, bs.cdist.p, bs.ccnt.p, nq, (int)b.kcmax, bs.qo.p, (int)kc_stride, oi.get(), od.get(),
                   oc.get());
    if (odi.get()) distinct_ids(oi.get(), slots, odi.get(), om.get(), opos.get());
  }
  oi.commit(); od.commit(); oc.commit(); onp.commit(); odi.commit(); om.commit(); opos.commit();
  sync_stream();
  LB2_API_END
}

// taken rows in host memory up to this size cross to the device in one copy; a larger batch is staged in query slabs,
// each slab's own taken rows gathered into a pinned buffer of this size
static constexpr size_t kTakenStageBytes = (size_t)512 << 20;
namespace {
struct PinnedHostBuf {
  void* p = nullptr;
  explicit PinnedHostBuf(size_t bytes) { LB2_CUDA(cudaMallocHost(&p, bytes ? bytes : 1)); }
  PinnedHostBuf(const PinnedHostBuf&) = delete;
  PinnedHostBuf& operator=(const PinnedHostBuf&) = delete;
  ~PinnedHostBuf() { cudaFreeHost(p); }
};
}  // namespace

// The exact re-rank of the rows the caller took (include/lance_b200.h): refine_batch_f32 with the taken rows as its
// row source, so it is lb2_index_search_batch's refine arithmetic with a row found by position instead of row id.
lb2_status lb2_index_refine_taken(lb2_index* index, const void* queries, uint64_t nq, const lb2_query_params* params,
                                  uint32_t kc_stride, const uint64_t* cand_ids, const float* cand_dists,
                                  const uint32_t* cand_counts, const void* taken, uint64_t m, const uint64_t* positions,
                                  uint32_t k_stride, uint64_t* row_ids_out, float* dists_out, uint32_t* counts_out) {
  LB2_API_BEGIN
  LB2_REQUIRE(index, "null index");
  LB2_REQUIRE(nq == 0 || (queries && params && cand_ids && cand_dists && cand_counts), "null queries, params or candidates");
  uint32_t kmax = 0;
  bool any_refine = false;
  std::vector<QueryOut> qo_h(nq);
  for (uint64_t q = 0; q < nq; ++q) {
    const lb2_query_params& p = params[q];
    const unsigned long long qi = (unsigned long long)q;
    LB2_REQUIRE(p.k > 0, "query %llu: k must be positive", qi);
    const uint64_t kc = (uint64_t)p.k * std::max<uint32_t>(1, p.refine_factor);
    if (kc > 1024)
      fail(LB2_UNSUPPORTED, "query %llu: k * refine_factor = %llu > 1024 is not implemented", qi, (unsigned long long)kc);
    LB2_REQUIRE(kc <= kc_stride, "query %llu: k * max(1, refine_factor) = %llu is above kc_stride %u", qi,
                (unsigned long long)kc, kc_stride);
    kmax = std::max(kmax, p.k);
    any_refine |= p.refine_factor > 0;
    qo_h[q] = QueryOut{(int)kc, (int)p.k, p.refine_factor > 0, (int)(p.has_lower_bound != 0),
                       (int)(p.has_upper_bound != 0), p.lower_bound, p.upper_bound};
  }
  LB2_REQUIRE(k_stride >= kmax, "k_stride %u is below the largest k %u", k_stride, kmax);
  LB2_REQUIRE(!any_refine || positions, "refine_factor > 0 needs positions");
  LB2_REQUIRE(!any_refine || m == 0 || taken, "null taken rows");
  if (nq == 0) {
    sync_stream();
    return LB2_OK;
  }
  const int d = index->d;
  const size_t row_bytes = (size_t)d * dtype_size(index->dtype), slots = (size_t)nq * kc_stride;
  VecIn q(queries, (size_t)nq * d, index->dtype);  // the original query, as the refine of a search takes it
  DevBuf<QueryOut> qo(nq);
  h2d(qo.p, qo_h.data(), nq);
  InArg<uint64_t> ci(cand_ids, slots);
  InArg<float> cd(cand_dists, slots);
  InArg<uint32_t> cc(cand_counts, nq);
  OutArg<uint64_t> oi(row_ids_out, (size_t)nq * k_stride);
  OutArg<float> od(dists_out, (size_t)nq * k_stride);
  OutArg<uint32_t> oc(counts_out, nq);
  TagScope tg("search");
  auto refine = [&](uint64_t q0, uint64_t n, const void* rows, uint64_t nrows, const uint64_t* pos) {
    refine_batch_f32(q.get() + q0 * d, n, d, index->metric, rows, (int)index->dtype, nrows, cd.get() + q0 * kc_stride,
                     ci.get() + q0 * kc_stride, cc.get() + q0, (int)kc_stride, qo.p + q0, (int)k_stride,
                     oi.get() + q0 * k_stride, od.get() + q0 * k_stride, oc.get() ? oc.get() + q0 : nullptr, pos);
  };
  if (!any_refine) {
    refine(0, nq, nullptr, 0, nullptr);
  } else if (m * row_bytes <= kTakenStageBytes || is_device_ptr(taken)) {
    InArg<uint8_t> t(taken, m * row_bytes);
    InArg<uint64_t> pos(positions, slots);
    refine(0, nq, t.get(), m, pos.get());
  } else {
    // query slabs: each slab's distinct positions (on the device, positions >= m left out so they still score NaN),
    // its rows gathered on the host into the pinned buffer, its positions renumbered into that buffer
    const size_t stage_rows = std::max<size_t>(kc_stride, kTakenStageBytes / row_bytes);
    const uint64_t slab = std::max<uint64_t>(1, stage_rows / kc_stride);
    InArg<uint64_t> pos(positions, slots);
    PinnedHostBuf stage(stage_rows * row_bytes), sel((size_t)slab * kc_stride * sizeof(uint64_t));
    DevBuf<uint8_t> rows(stage_rows * row_bytes);
    DevBuf<uint64_t> ldist((size_t)slab * kc_stride), lpos((size_t)slab * kc_stride), lm(1);
    const uint8_t* src = static_cast<const uint8_t*>(taken);
    uint8_t* dst = static_cast<uint8_t*>(stage.p);
    const uint64_t* local = static_cast<const uint64_t*>(sel.p);
    for (uint64_t q0 = 0; q0 < nq; q0 += slab) {
      const uint64_t n = std::min<uint64_t>(slab, nq - q0);
      distinct_ids(pos.get() + q0 * kc_stride, n * kc_stride, ldist.p, lm.p, lpos.p, m);
      uint64_t nl = 0;
      d2h(&nl, lm.p, 1);
      sync_stream();  // (also: the previous slab has read the staging buffer)
      d2h(static_cast<uint64_t*>(sel.p), ldist.p, nl);
      sync_stream();
      for (uint64_t r = 0; r < nl; ++r) memcpy(dst + r * row_bytes, src + local[r] * row_bytes, row_bytes);
      h2d(rows.p, dst, nl * row_bytes);
      refine(q0, n, rows.p, nl, lpos.p);
    }
    sync_stream();  // before the pinned buffer is released
  }
  oi.commit(); od.commit(); oc.commit();
  sync_stream();
  LB2_API_END
}

lb2_status lb2_index_search_combined(lb2_index* index, const void* queries, uint64_t nq, const lb2_search_params* sp,
                                     const lb2_probe_params* pp, const lb2_unindexed_rows* u, uint64_t* row_ids_out,
                                     float* dists_out, uint32_t* counts_out, uint32_t* nprobes_out) {
  LB2_API_BEGIN
  LB2_REQUIRE(index && sp, "null argument");
  LB2_REQUIRE(sp->k > 0, "k must be positive");
  LB2_REQUIRE(sp->refine_vectors, "the combined search re-scores the index's rows exactly: refine_vectors is required");
  LB2_REQUIRE(u && u->row_ids, "the unindexed rows and their row ids are required");
  LB2_REQUIRE(u->n == 0 || u->vectors, "null unindexed vectors");
  LB2_REQUIRE(!nprobes_out || pp, "nprobes_out needs probe parameters");
  if (current_comm() && current_comm()->nranks > 1)
    fail(LB2_UNSUPPORTED, "a combined search on a row-sharded index is not implemented");
  const int k = (int)sp->k, d = index->d;
  flat_search_check(d, index->dtype, index->metric, (int)std::min<uint32_t>(sp->k, 1025));
  std::unique_ptr<ProbedSearch> ps;
  if (pp) ps.reset(new ProbedSearch(sp, pp, nq, nprobes_out));
  // the index's rows: refined, so their distances are exact (scanner.rs:2884-2905)
  lb2_search_params s = *sp;
  s.refine_factor = std::max<uint32_t>(1, sp->refine_factor);
  const size_t nk = (size_t)nq * k;
  DevBuf<uint64_t> ids(std::max<size_t>(1, 2 * nk));
  DevBuf<float> dists(std::max<size_t>(1, 2 * nk));
  DevBuf<uint32_t> cnts(std::max<uint64_t>(1, 2 * nq));
  index_search_impl(index, queries, nq, s, ids.p, dists.p, cnts.p, ps ? &ps->pr : nullptr);
  // the unindexed rows: flat_knn with the index metric on the original query (scanner.rs:2993-3013)
  VecIn q(queries, (size_t)nq * d, index->dtype);
  InArg<uint64_t> rid(u->row_ids, u->n), allow(u->allow_bitmap, u->allow_bitmap ? (size_t)((u->n + 63) / 64) : 0);
  FlatFilter flt;
  flt.allow = allow.get();
  flt.has_lower = sp->has_lower_bound != 0;
  flt.has_upper = sp->has_upper_bound != 0;
  flt.lower = sp->lower_bound;
  flt.upper = sp->upper_bound;
  flat_search(q.get(), nq, d, index->metric, u->vectors, u->n, index->dtype, rid.get(), flt, k, ids.p + nk,
              dists.p + nk, cnts.p + nq);
  // the union by (_distance, _rowid), first k
  OutArg<uint64_t> oi(row_ids_out, nk);
  OutArg<float> od(dists_out, nk);
  OutArg<uint32_t> oc(counts_out, nq);
  {
    TagScope tg("search");
    merge_lists("merge_combined", nq, dists.p, ids.p, cnts.p, 2, k, nk, nk, (size_t)k, nq, 1, oi.get(), od.get(),
                oc.get());
  }
  oi.commit(); od.commit(); oc.commit();
  if (ps) ps->np_out.commit();
  sync_stream();
  LB2_API_END
}

// knn_combined for a mixed batch (include/lance_b200.h): BatchSearch and refine_batch_f32 with every refine factor
// raised to max(1, rf), flat_search_batch over the unindexed rows, and merge_lists with each query's own k.  Both
// halves are rows of k_stride, so the merge writes the output rows directly.
lb2_status lb2_index_search_combined_batch(lb2_index* index, const void* queries, uint64_t nq,
                                           const lb2_query_params* params, const lb2_query_filter* filters,
                                           uint32_t num_filters, const void* refine_vectors, uint64_t num_vectors,
                                           uint32_t late_width, const lb2_unindexed_batch* u, uint32_t k_stride,
                                           uint64_t* row_ids_out, float* dists_out, uint32_t* counts_out,
                                           uint32_t* nprobes_out) {
  LB2_API_BEGIN
  LB2_REQUIRE(index, "null index");
  LB2_REQUIRE(nq == 0 || params, "null queries or params");
  LB2_REQUIRE(refine_vectors, "the combined search re-scores the index's rows exactly: refine_vectors is required");
  std::vector<lb2_query_params> ip(params, params + nq);
  for (lb2_query_params& p : ip) p.refine_factor = std::max<uint32_t>(1, p.refine_factor);
  const BatchPlan b(index, queries, nq, ip.data(), filters, num_filters, late_width, true);
  LB2_REQUIRE(k_stride >= b.kmax, "k_stride %u is below the largest k %u", k_stride, b.kmax);
  LB2_REQUIRE(u && u->rows.row_ids, "the unindexed rows and their row ids are required");
  LB2_REQUIRE(u->rows.n == 0 || u->rows.vectors, "null unindexed vectors");
  LB2_REQUIRE(num_filters == 0 || u->filter_bitmaps, "null unindexed filter_bitmaps");
  if (current_comm() && current_comm()->nranks > 1)
    fail(LB2_UNSUPPORTED, "a combined search on a row-sharded index is not implemented");
  const int d = index->d;
  flat_search_batch_check(d, index->dtype, index->metric, (int)std::max<uint32_t>(1, b.kmax));
  if (nq == 0) {
    sync_stream();
    return LB2_OK;
  }
  const size_t nk = (size_t)nq * k_stride;
  OutArg<uint64_t> oi(row_ids_out, nk);
  OutArg<float> od(dists_out, nk);
  OutArg<uint32_t> oc(counts_out, nq);
  OutArg<uint32_t> onp(nprobes_out, nq);
  DevBuf<uint64_t> ids(2 * nk);
  DevBuf<float> dists(2 * nk);
  DevBuf<uint32_t> cnts(2 * nq);
  // the index's rows, refined so that their distances are exact (scanner.rs:2884-2905)
  BatchSearch bs(index, queries, nq, ip.data(), filters, num_filters, late_width, b, onp.get());
  {
    TagScope tg("search");
    InArg<uint8_t> v(refine_vectors, (size_t)num_vectors * d * dtype_size(index->dtype));
    refine_batch_f32(bs.q.q.get(), nq, d, index->metric, v.get(), (int)index->dtype, num_vectors, bs.cdist.p,
                     bs.cid.p, bs.ccnt.p, (int)b.kcmax, bs.qo.p, (int)k_stride, ids.p, dists.p, cnts.p);
  }
  // the unindexed rows: flat_knn with the index metric on the original query, each query with its own bitmap
  // (scanner.rs:2993-3013)
  const lb2_unindexed_rows& r = u->rows;
  const size_t words = (size_t)((r.n + 63) / 64);
  InArg<uint64_t> rid(r.row_ids, r.n), allow(r.allow_bitmap, r.allow_bitmap ? words : 0);
  std::vector<InArg<uint64_t>> bm(num_filters);
  std::vector<const uint64_t*> bm_dev(num_filters);
  for (uint32_t f = 0; f < num_filters; ++f) {
    bm[f].set(u->filter_bitmaps[f], u->filter_bitmaps[f] ? words : 0);
    bm_dev[f] = bm[f].get();
  }
  const std::vector<FlatQuery> fq = flat_queries(params, nq, bm_dev, allow.get());
  flat_search_batch(bs.q.q.get(), nq, d, index->metric, r.vectors, r.n, index->dtype, rid.get(), fq.data(),
                    (int)k_stride, ids.p + nk, dists.p + nk, cnts.p + nq);
  // the union by (_distance, _rowid), first k_q
  std::vector<QueryParam> qp_h(nq);
  for (uint64_t q = 0; q < nq; ++q) qp_h[q].k = (int)params[q].k;
  DevBuf<QueryParam> qp(nq);
  h2d(qp.p, qp_h.data(), nq);
  {
    TagScope tg("search");
    merge_lists("merge_combined", nq, dists.p, ids.p, cnts.p, 2, (int)k_stride, nk, nk, (size_t)k_stride, nq, 1,
                oi.get(), od.get(), oc.get(), 2, qp.p);
  }
  oi.commit(); od.commit(); oc.commit(); onp.commit();
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
  index_search_impl(index, queries, nq, *sp, row_ids_out, dists_out, counts_out);
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
  index_search_impl(index, queries, nq, *sp, li.p, ld.p, lc.p);
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

lb2_status lb2_index_update(const lb2_index* old, const void* new_centroids, uint32_t new_k, const uint32_t* part_map,
                            const uint32_t* add_part_ids, const uint8_t* add_codes, const uint64_t* add_row_ids,
                            uint64_t n_add, const uint64_t* remove_row_ids, uint64_t n_remove, lb2_index** out) {
  LB2_API_BEGIN
  if (old && old->kind == IndexKind::FLAT && old->hnsw)
    fail(LB2_UNSUPPORTED, "lb2_index_update: IVF_HNSW_FLAT indexes are not implemented");
  LB2_REQUIRE(old && out && old->kind == IndexKind::PQ, "lb2_index_update takes an IVF_PQ index");
  if (old->hnsw) fail(LB2_UNSUPPORTED, "lb2_index_update: IVF_HNSW_PQ indexes are not implemented");
  LB2_REQUIRE(n_add == 0 || (add_part_ids && add_codes && add_row_ids), "added rows need partition ids, codes and row ids");
  lb2_optimize_params p = {};
  p.new_centroids = new_centroids;
  p.new_k = new_k;
  p.part_map = part_map;
  p.add_part_ids = add_part_ids;
  p.add_payload = add_codes;
  p.add_row_ids = add_row_ids;
  p.n_add = n_add;
  p.remove_row_ids = remove_row_ids;
  p.n_remove = n_remove;
  *out = index_merge(old, p, "index_update").release();
  LB2_API_END
}

lb2_status lb2_index_optimize(const lb2_index* old, const lb2_optimize_params* p, lb2_index** out) {
  LB2_API_BEGIN
  LB2_REQUIRE(old && p && out, "null argument");
  *out = index_merge(old, *p, "index_optimize").release();
  LB2_API_END
}

lb2_status lb2_index_repartition(const lb2_index* shard, lb2_index** owned_out) {
  LB2_API_BEGIN
  LB2_REQUIRE(shard && owned_out, "null argument");
  if (shard->kind == IndexKind::RQ) fail(LB2_UNSUPPORTED, "lb2_index_repartition: IVF_RQ indexes are not implemented");
  if (shard->hnsw) fail(LB2_UNSUPPORTED, "lb2_index_repartition: %s indexes are not implemented", shard->hnsw->kind);
  Comm* cm = current_comm();
  const int G = cm ? cm->nranks : 1, me = cm ? cm->rank : 0;
  const int K = shard->K;
  const int rb = (int)shard->row_bytes();
  const uint8_t* payload = shard->payload().p;
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
  std::vector<size_t> s_off(G), r_off(G);
  std::vector<uint64_t> s_rows(G, 0), r_rows(G, 0), send_base(K);
  for (int p = 0; p < K; ++p) s_rows[p % G] += mine[p];
  {
    std::vector<uint64_t> run(G, 0);
    uint64_t acc = 0;
    std::vector<uint64_t> gbase(G);
    for (int g = 0; g < G; ++g) { gbase[g] = acc; acc += s_rows[g]; }
    for (int p = 0; p < K; ++p) { send_base[p] = gbase[p % G] + run[p % G]; run[p % G] += mine[p]; }
    for (int g = 0; g < G; ++g) s_off[g] = gbase[g];
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
      r_off[r] = acc; acc += r_rows[r];
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
    for (int g = 0; g < G; ++g) { so[g] = s_off[g] * rb; sb[g] = s_rows[g] * rb; ro[g] = r_off[g] * rb; rbv[g] = r_rows[g] * rb; }
    comm_alltoallv_bytes(sp.p, so.data(), sb.data(), rp.p, ro.data(), rbv.data());
    for (int g = 0; g < G; ++g) { so[g] = s_off[g] * 8; sb[g] = s_rows[g] * 8; ro[g] = r_off[g] * 8; rbv[g] = r_rows[g] * 8; }
    comm_alltoallv_bytes(si.p, so.data(), sb.data(), ri.p, ro.data(), rbv.data());
  }
  std::unique_ptr<lb2_index> ix = make_index(shard->kind, K, shard->d, shard->metric, shard->dtype);
  copy_model(shard, ix.get());
  ix->n = n_new;
  ix->part_offsets.alloc(K + 1);
  h2d(ix->part_offsets.p, new_off.data(), (size_t)K + 1);
  DevBuf<uint8_t>& dstp = ix->payload();
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
  build_skew(ix.get());
  sync_stream();
  *owned_out = ix.release();
  LB2_API_END
}

lb2_status lb2_index_set_partition_index(lb2_index* index, lb2_partition_index_mode mode, uint64_t seed,
                                         uint32_t insert_batch) {
  LB2_API_BEGIN
  LB2_REQUIRE(index, "null argument");
  set_partition_index(index, (uint32_t)mode, seed, insert_batch);
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

}  // extern "C"
