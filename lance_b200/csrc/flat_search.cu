// flat_search.cu -- flat KNN over a vector column, batched over queries: the exact distance of every (query, row)
// pair by the refine plan's per-element-type rule (row_distance.cuh), the rows a bitmap and a [lower, upper) range
// admit, and the k smallest (distance, row id) pairs of every query.
//
// Replaces  flat_knn                             rust/lance/src/dataset/scanner.rs:3336-3411, 2912-2941
//           compute_distance                     lance-index/src/vector/flat.rs:94-150
//           SortExec(_distance, _rowid).fetch(k) scanner.rs:3450-3466
//
// One CTA scores a tile of FS_Q queries (f32 in shared memory) against a range of rows, which it streams through
// shared memory FS_R rows at a time: each row is read from memory once per query tile.  Each half-warp owns a 4 x 4
// register tile of (query, row) pairs and, as lane l, the elements of lane l of the rule: one element load from shared
// memory feeds four pairs.  The 16 lane partials of a pair meet in shared memory, where one lane folds them in the
// rule's order.  A pair that the filter admits and that precedes the query's current k-th (distance, row id) is
// appended to the query's pending buffer; a full buffer is merged into the CTA's sorted list of the query by rank
// (merge-path ranks: position in its own run + count of the other run before it), the list living in the output
// candidate array.  The per-query top-k by (distance, row id) is contained in the union of the CTAs' lists, which
// merge_list_tree (ivf_search.cu) merges per query.
//
// flat_search_batch runs the same scan for queries that differ in k, range and bitmap: the batch kernel loads its
// tile's entries of a per-query table into shared memory, and each folded (query, row) pair reads its own query's
// bitmap bit, bounds and k-th threshold; a query's list is cut at its own k.  The launches are those of a uniform
// batch of the largest k.
#include <algorithm>
#include <memory>
#include <vector>

#include "common.cuh"
#include "exact.cuh"
#include "flat_search.cuh"
#include "ivf_search.cuh"
#include "row_distance.cuh"
#include "scan.cuh"
#include "staging.cuh"
#include "topk.cuh"

namespace lb2 {

constexpr int FS_Q = 16;                  // queries per CTA: 4 groups of 4
constexpr int FS_R = 16;                  // rows per tile: 4 groups of 4
constexpr int FS_P = 128;                 // pending candidates per query between two merges
constexpr int FS_RED = 16 * 2 * 17 + 16;  // per half-warp: 16 pairs x 2 partials x 16 lanes (stride 17), 16 tails
constexpr int FS_MIN_ROWS = 2048;         // the fewest rows a CTA is given when row ranges are split for parallelism

// row stride of the query tile: = 4 (mod 8) words, so the two half-warps of a warp (query groups g, g + 1: 4 rows
// apart) read disjoint bank halves
__host__ __device__ inline int fs_qstride(int d) { return (d + 7) / 8 * 8 + 4; }
__host__ __device__ inline size_t fs_region_bytes(int d, size_t es) {
  const size_t rows = ((size_t)FS_R * d * es + 15) / 16 * 16;
  const size_t red = sizeof(float) * 16 * FS_RED;
  return rows > red ? rows : red;
}
static size_t fs_smem_bytes(int d, size_t es) {
  return sizeof(float) * FS_Q * fs_qstride(d) + fs_region_bytes(d, es) + (size_t)FS_Q * FS_P * (8 + 4);
}

// the FS_R-row tile [src, src + bytes) -> shared memory, as wide as the alignment allows
__device__ __forceinline__ void fs_copy_tile(unsigned char* dst, const unsigned char* src, size_t bytes) {
  const uintptr_t a = reinterpret_cast<uintptr_t>(src) | bytes;
  if ((a & 15) == 0) {
    for (size_t i = threadIdx.x; i < bytes / 16; i += 256)
      reinterpret_cast<uint4*>(dst)[i] = reinterpret_cast<const uint4*>(src)[i];
  } else if ((a & 3) == 0) {
    for (size_t i = threadIdx.x; i < bytes / 4; i += 256)
      reinterpret_cast<uint32_t*>(dst)[i] = reinterpret_cast<const uint32_t*>(src)[i];
  } else {
    for (size_t i = threadIdx.x; i < bytes; i += 256) dst[i] = src[i];
  }
}

// Merge query qi's np pending candidates into its sorted list of nw <= k (wd / wi, global memory), keeping the k
// smallest (key, id).  Every rank is computed before anything is written; block-wide, with barriers.
__device__ __forceinline__ void fs_merge(int k, float* wd, uint64_t* wi, const int32_t* pkey, const uint64_t* pid,
                                         uint32_t* s_pcnt, uint32_t* s_wcnt, int32_t* s_wkey, uint64_t* s_wid, int qi) {
  const int tid = threadIdx.x;
  const uint32_t np = s_pcnt[qi], nw = s_wcnt[qi];
  const uint32_t nn = min((uint32_t)k, nw + np);
  float mf[4];
  int32_t mk[4];
  uint64_t mi[4];
  uint32_t mr[4];
#pragma unroll
  for (int m = 0; m < 4; ++m) {  // k <= 1024: at most 4 list entries per thread
    const uint32_t w = tid + 256 * m;
    mr[m] = ~0u;
    if (w >= nw) continue;
    mf[m] = wd[w];
    mk[m] = total_order_key(mf[m]);
    mi[m] = wi[w];
    uint32_t r = w;
    for (uint32_t j = 0; j < np; ++j) r += ki_less(pkey[j], pid[j], mk[m], mi[m]) ? 1u : 0u;
    mr[m] = r;
  }
  int32_t key = 0;
  uint64_t id = 0;
  uint32_t pr = ~0u;
  if ((uint32_t)tid < np) {  // np <= FS_P < 256
    key = pkey[tid];
    id = pid[tid];
    uint32_t r = 0;
    for (uint32_t j = 0; j < np; ++j) r += ki_less(pkey[j], pid[j], key, id) ? 1u : 0u;
    uint32_t lo = 0, hi = nw;  // list entries before it
    while (lo < hi) {
      const uint32_t mid = (lo + hi) >> 1;
      if (ki_less(total_order_key(wd[mid]), wi[mid], key, id)) lo = mid + 1; else hi = mid;
    }
    pr = r + lo;
  }
  __syncthreads();
#pragma unroll
  for (int m = 0; m < 4; ++m) {
    if (mr[m] >= nn) continue;
    wd[mr[m]] = mf[m];
    wi[mr[m]] = mi[m];
    if (mr[m] == nn - 1) { s_wkey[qi] = mk[m]; s_wid[qi] = mi[m]; }
  }
  if (pr < nn) {
    wd[pr] = key_to_float(key);
    wi[pr] = id;
    if (pr == nn - 1) { s_wkey[qi] = key; s_wid[qi] = id; }
  }
  if (tid == 0) {
    s_pcnt[qi] = 0;
    s_wcnt[qi] = nn;
  }
  __syncthreads();
}

// grid (query tiles, row ranges of rows_per_cta rows); rows [0, n) of this launch are rows [r0, r0 + n) of the column.
// The list of query q and row range y is list list0 + y of the nl lists per query of cand_* ([nq][nl][k]).
// BATCH: every query's own k (<= k, the lists' stride) and filter from s_fq, the tile's entries of the FlatQuery table
// (flat_search_batch_scan_kernel); the single-parameter kernel is compiled without them.
template <int METRIC, class T, bool BATCH>
__device__ __forceinline__ void fs_scan(const float* __restrict__ queries, uint64_t nq, int d, const T* __restrict__ rows,
                                        uint64_t n, uint64_t r0, uint64_t rows_per_cta,
                                        const uint64_t* __restrict__ row_ids, const FlatFilter flt, int k, int nl,
                                        int list0, float* cand_d, uint64_t* cand_id, uint32_t* __restrict__ cand_cnt,
                                        const FlatQuery* s_fq) {
  constexpr int RULE = refine_rule<METRIC, T>();
  extern __shared__ __align__(16) unsigned char fs_smem[];
  const int qstride = fs_qstride(d);
  float* qs = reinterpret_cast<float*>(fs_smem);                                  // [FS_Q][qstride]
  unsigned char* region = fs_smem + sizeof(float) * FS_Q * qstride;               // the row tile, then the partials
  const T* rs = reinterpret_cast<const T*>(region);
  float* red = reinterpret_cast<float*>(region);
  uint64_t* pid = reinterpret_cast<uint64_t*>(region + fs_region_bytes(d, sizeof(T)));  // [FS_Q][FS_P]
  int32_t* pkey = reinterpret_cast<int32_t*>(pid + FS_Q * FS_P);                      // [FS_Q][FS_P]
  __shared__ uint32_t s_pcnt[FS_Q], s_wcnt[FS_Q];
  __shared__ int32_t s_wkey[FS_Q];
  __shared__ uint64_t s_wid[FS_Q];
  __shared__ float s_qnorm[FS_Q];

  const int tid = threadIdx.x, l = tid & 15, h = tid >> 4, qg = h & 3, rg = h >> 2;
  const unsigned hmask = 0xffffu << (16 * (h & 1));
  const uint64_t q0 = (uint64_t)blockIdx.x * FS_Q;
  const int nqt = nq - q0 < (uint64_t)FS_Q ? (int)(nq - q0) : FS_Q;
  const uint64_t b0 = (uint64_t)blockIdx.y * rows_per_cta, b1 = min(n, b0 + rows_per_cta);
  const size_t list = list0 + blockIdx.y;
  for (int i = tid; i < FS_Q * d; i += 256) {
    const int qi = i / d, e = i - qi * d;
    qs[qi * qstride + e] = qi < nqt ? queries[(q0 + qi) * d + e] : 0.0f;
  }
  if (tid < FS_Q) { s_pcnt[tid] = 0; s_wcnt[tid] = 0; }
  __syncthreads();
  if (METRIC == METRIC_COSINE) {  // norm_l2(query): 16 lanes + sqrt (norm_l2.rs:106-130), half-warp h for query h
    float a = 0.0f;
    for (int e = l; e < d; e += 16) a = fmaf(qs[h * qstride + e], qs[h * qstride + e], a);
#pragma unroll
    for (int o = 8; o >= 1; o >>= 1) a += __shfl_xor_sync(hmask, a, o, 16);
    if (l == 0) s_qnorm[h] = sqrtf(a);
  }
  auto list_d = [&](int qi) { return cand_d + ((q0 + qi) * nl + list) * k; };
  auto list_id = [&](int qi) { return cand_id + ((q0 + qi) * nl + list) * k; };
  float* my = red + h * FS_RED;
  // lane l folds pair l of its half-warp's tile: query qg * 4 + l / 4, row rg * 4 + l % 4
  const int fq = qg * 4 + (l >> 2), fr = rg * 4 + (l & 3);
  for (uint64_t t0 = b0; t0 < b1; t0 += FS_R) {
    const int nr = b1 - t0 < (uint64_t)FS_R ? (int)(b1 - t0) : FS_R;
    fs_copy_tile(region, reinterpret_cast<const unsigned char*>(rows + t0 * d), (size_t)nr * d * sizeof(T));
    __syncthreads();
    LaneAcc<RULE, METRIC> acc[4][4];
    rule_walk<RULE>(d, l, [&](int e, auto part) {
      float qv[4], vv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) qv[i] = qs[(qg * 4 + i) * qstride + e];
#pragma unroll
      for (int j = 0; j < 4; ++j) vv[j] = ldf<T>(rs + (size_t)(rg * 4 + j) * d, e);
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j].template step<decltype(part)::value>(qv[i], vv[j]);
    });
    __syncthreads();  // the row tile is read: its space takes the partials
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int p = i * 4 + j;
        my[(p * 2) * 17 + l] = RULE == RULE_U8 ? __uint_as_float(acc[i][j].u) : acc[i][j].a;
        if (RULE == RULE_DOT32 || RULE == RULE_COSINE) my[(p * 2 + 1) * 17 + l] = acc[i][j].b;
        if ((RULE == RULE_LANES16 || RULE == RULE_DOT32) && l == 0) my[16 * 2 * 17 + p] = acc[i][j].s;
      }
    __syncwarp(hmask);
    const float* pa = my + (l * 2) * 17;
    const float* pb = my + (l * 2 + 1) * 17;
    const float dist = fold_partials<RULE, METRIC>([&](int i) { return pa[i]; }, [&](int i) { return pb[i]; },
                                                   [&](int i) { return __float_as_uint(pa[i]); }, my[16 * 2 * 17 + l],
                                                   METRIC == METRIC_COSINE ? s_qnorm[fq] : 0.0f);
    const uint64_t r = r0 + t0 + fr;  // the row's position in the column
    // LanceFilterExec(_distance >= lower AND _distance < upper) and the caller's bitmap (scanner.rs:3342-3377)
    auto offer = [&](const FlatFilter& f, int kq) {
      if (fq < nqt && fr < nr && row_allowed(f.allow, r) && (!f.has_lower || dist >= f.lower) &&
          (!f.has_upper || dist < f.upper)) {
        const int32_t key = total_order_key(dist);
        const uint64_t id = row_ids ? row_ids[r] : r;
        if (s_wcnt[fq] < (uint32_t)kq || ki_less(key, id, s_wkey[fq], s_wid[fq])) {
          const uint32_t at = atomicAdd(&s_pcnt[fq], 1u);
          pkey[fq * FS_P + at] = key;
          pid[fq * FS_P + at] = id;
        }
      }
    };
    if constexpr (BATCH) offer(s_fq[fq].flt, s_fq[fq].k);
    else offer(flt, k);
    __syncthreads();
    for (int qi = 0; qi < nqt; ++qi)  // a buffer that might not take the next tile's rows is merged
      if (s_pcnt[qi] > FS_P - FS_R)
        fs_merge(BATCH ? s_fq[qi].k : k, list_d(qi), list_id(qi), pkey + qi * FS_P, pid + qi * FS_P, s_pcnt, s_wcnt,
                 s_wkey, s_wid, qi);
  }
  for (int qi = 0; qi < nqt; ++qi)
    if (s_pcnt[qi] > 0)
      fs_merge(BATCH ? s_fq[qi].k : k, list_d(qi), list_id(qi), pkey + qi * FS_P, pid + qi * FS_P, s_pcnt, s_wcnt,
               s_wkey, s_wid, qi);
  if (tid < nqt) cand_cnt[(q0 + tid) * nl + list] = s_wcnt[tid];
}

template <int METRIC, class T>
__global__ void __launch_bounds__(256)
flat_search_scan_kernel(const float* __restrict__ queries, uint64_t nq, int d, const T* __restrict__ rows, uint64_t n,
                        uint64_t r0, uint64_t rows_per_cta, const uint64_t* __restrict__ row_ids, const FlatFilter flt,
                        int k, int nl, int list0, float* cand_d, uint64_t* cand_id, uint32_t* __restrict__ cand_cnt) {
  fs_scan<METRIC, T, false>(queries, nq, d, rows, n, r0, rows_per_cta, row_ids, flt, k, nl, list0, cand_d, cand_id,
                            cand_cnt, nullptr);
}

// the batch version: query q's k and filter are fq[q] (flat_search_batch); k is the lists' stride, the largest k
template <int METRIC, class T>
__global__ void __launch_bounds__(256)
flat_search_batch_scan_kernel(const float* __restrict__ queries, uint64_t nq, int d, const T* __restrict__ rows,
                              uint64_t n, uint64_t r0, uint64_t rows_per_cta, const uint64_t* __restrict__ row_ids,
                              const FlatQuery* __restrict__ fq, int k, int nl, int list0, float* cand_d,
                              uint64_t* cand_id, uint32_t* __restrict__ cand_cnt) {
  __shared__ FlatQuery s_fq[FS_Q];
  const uint64_t q0 = (uint64_t)blockIdx.x * FS_Q;
  if (threadIdx.x < FS_Q) s_fq[threadIdx.x] = q0 + threadIdx.x < nq ? fq[q0 + threadIdx.x] : FlatQuery{};
  // (fs_scan's first barrier orders these writes before any read)
  fs_scan<METRIC, T, true>(queries, nq, d, rows, n, r0, rows_per_cta, row_ids, FlatFilter{}, k, nl, list0, cand_d,
                           cand_id, cand_cnt, s_fq);
}

template <bool BATCH, class F>
static void with_scan_kernel(int metric, lb2_dtype dt, F&& f) {
  dispatch_metric_elem<true>(metric, (int)dt, [&](auto m, auto e) {
    using T = typename decltype(e)::type;
    if constexpr (BATCH) f(flat_search_batch_scan_kernel<decltype(m)::value, T>, T{});
    else f(flat_search_scan_kernel<decltype(m)::value, T>, T{});
  });
}

template <bool BATCH>
static void scan_check(int d, lb2_dtype dt, int metric, int k) {
  if (k > 1024) fail(LB2_UNSUPPORTED, "k = %d > 1024 is not implemented", k);
  const size_t dyn = fs_smem_bytes(d, dtype_size(dt));
  size_t need = 0;
  with_scan_kernel<BATCH>(metric, dt, [&](auto kern, auto) { need = smem_with_static(kern, dyn); });
  if (need > ctx().smem_optin)
    fail(LB2_UNSUPPORTED, "dimension %d: the flat search's tile of %d queries and %d rows needs %zu bytes of shared "
         "memory, the device has %zu", d, FS_Q, FS_R, need, ctx().smem_optin);
}
void flat_search_check(int d, lb2_dtype dt, int metric, int k) { scan_check<false>(d, dt, metric, k); }
void flat_search_batch_check(int d, lb2_dtype dt, int metric, int kmax) { scan_check<true>(d, dt, metric, kmax); }

// row ranges per launch over `rows` rows for nqt query tiles: enough CTAs for four per SM, each at least FS_MIN_ROWS
static int fs_ranges(uint64_t rows, uint64_t nqt) {
  const uint64_t want = cdiv(4ull * ctx().num_sms, nqt);
  return (int)std::max<uint64_t>(1, std::min<uint64_t>(want, rows / FS_MIN_ROWS));
}

// The scan of both entry points: query slabs whose candidate lists (stride k) hold at most about 256 MB, a launch per
// staged chunk of host rows (one for device rows), and each slab's lists merged by merge_list_tree into [qn][k] at
// out_ids + s0 * k (merged(s0, qn) runs after each slab's merge).  fq (device, BATCH only): the per-query table.
template <bool BATCH, class Merged>
static void fs_run(const float* queries, uint64_t nq, int d, int metric, const void* vectors, uint64_t n, lb2_dtype dt,
                   const uint64_t* row_ids, const FlatFilter& flt, const FlatQuery* fq, int k, uint64_t* out_ids,
                   float* out_dists, uint32_t* out_counts, Merged&& merged) {
  const size_t dyn = fs_smem_bytes(d, dtype_size(dt));
  std::unique_ptr<Source> src;
  const void* nat = nullptr;
  uint64_t step = std::max<uint64_t>(n, 1);
  if (n) {
    src.reset(new Source(vectors, n, d, dt));
    nat = src->native_device();
    if (!nat) step = chunk_step(*src);
  }
  // lists per query: every launch's row ranges (a launch per staged chunk)
  auto lists = [&](uint64_t qn) {
    int nl = 0;
    for (uint64_t r = 0; r < n; r += step) nl += fs_ranges(std::min(step, n - r), cdiv(qn, FS_Q));
    return std::max(nl, 1);
  };
  // query slabs: candidate lists of at most about 256 MB
  uint64_t slab = nq;
  while (slab > FS_Q && slab * lists(slab) * k * 12 > (256ull << 20)) slab = (slab / 2 + FS_Q - 1) / FS_Q * FS_Q;
  for (uint64_t s0 = 0; s0 < nq; s0 += slab) {
    const uint64_t qn = std::min(slab, nq - s0), nqt = cdiv(qn, FS_Q);
    const int nl = lists(qn);
    DevBuf<float> cd(qn * nl * k);
    DevBuf<uint64_t> cid(qn * nl * k);
    DevBuf<uint32_t> ccnt(qn * nl);
    ccnt.zero();
    int list0 = 0;
    auto scan = [&](const void* rows, uint64_t r0, uint64_t cnt) {
      const int nr = fs_ranges(cnt, nqt);
      const uint64_t per = (cdiv(cnt, nr) + FS_R - 1) / FS_R * FS_R;
      with_scan_kernel<BATCH>(metric, dt, [&](auto kern, auto t) {
        using T = decltype(t);
        set_smem(kern, dyn);
        if constexpr (BATCH)
          LB2_LAUNCH("scan", kern, dim3((unsigned)nqt, (unsigned)nr), 256, dyn, queries + s0 * d, qn, d,
                     static_cast<const T*>(rows), cnt, r0, per, row_ids, fq + s0, k, nl, list0, cd.p, cid.p, ccnt.p);
        else
          LB2_LAUNCH("scan", kern, dim3((unsigned)nqt, (unsigned)nr), 256, dyn, queries + s0 * d, qn, d,
                     static_cast<const T*>(rows), cnt, r0, per, row_ids, flt, k, nl, list0, cd.p, cid.p, ccnt.p);
      });
      list0 += nr;
    };
    if (nat) scan(nat, 0, n);
    else if (n) for_each_chunk(*src, [&](const float* xf, const void* xnat, uint64_t r0, uint64_t rows) {
      scan(xnat ? xnat : xf, r0, rows);
    });
    merge_list_tree("merge", qn, cd.p, cid.p, ccnt.p, nl, k, out_ids + s0 * k, out_dists + s0 * k,
                    out_counts ? out_counts + s0 : nullptr);
    merged(s0, qn);
  }
}

void flat_search(const float* queries, uint64_t nq, int d, int metric, const void* vectors, uint64_t n, lb2_dtype dt,
                 const uint64_t* row_ids, const FlatFilter& flt, int k, uint64_t* out_ids, float* out_dists,
                 uint32_t* out_counts) {
  flat_search_check(d, dt, metric, k);
  if (nq == 0) return;
  TagScope tg("flat_search");
  fs_run<false>(queries, nq, d, metric, vectors, n, dt, row_ids, flt, nullptr, k, out_ids, out_dists, out_counts,
                [](uint64_t, uint64_t) {});
}

// Each slab's lists are merged to the slab's largest k (every list holds at most its own query's k, so the first k_q
// of query q's merged row are its top k_q), then cut to k_q into rows of k_stride by candidate_rows.
void flat_search_batch(const float* queries, uint64_t nq, int d, int metric, const void* vectors, uint64_t n,
                       lb2_dtype dt, const uint64_t* row_ids, const FlatQuery* fq_host, int k_stride,
                       uint64_t* out_ids, float* out_dists, uint32_t* out_counts) {
  int kmax = 1;
  for (uint64_t q = 0; q < nq; ++q) kmax = std::max(kmax, fq_host[q].k);
  flat_search_batch_check(d, dt, metric, kmax);
  if (nq == 0) return;
  TagScope tg("flat_search");
  DevBuf<FlatQuery> fq(nq);
  h2d(fq.p, fq_host, nq);
  std::vector<QueryOut> qo_h(nq);
  for (uint64_t q = 0; q < nq; ++q) qo_h[q] = QueryOut{fq_host[q].k, fq_host[q].k, 0, 0, 0, 0.0f, 0.0f};
  DevBuf<QueryOut> qo(nq);
  h2d(qo.p, qo_h.data(), nq);
  DevBuf<uint64_t> mi(nq * kmax);
  DevBuf<float> md(nq * kmax);
  DevBuf<uint32_t> mc(nq), oc;
  if (!out_counts) {
    oc.alloc(nq);
    out_counts = oc.p;
  }
  fs_run<true>(queries, nq, d, metric, vectors, n, dt, row_ids, FlatFilter{}, fq.p, kmax, mi.p, md.p, mc.p,
               [&](uint64_t s0, uint64_t qn) {
                 candidate_rows(mi.p + s0 * kmax, md.p + s0 * kmax, mc.p + s0, qn, kmax, qo.p + s0, k_stride,
                                out_ids + s0 * k_stride, out_dists + s0 * k_stride, out_counts + s0);
               });
}

}  // namespace lb2
