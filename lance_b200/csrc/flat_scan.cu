// flat_scan.cu -- the exact-distance query kernels: the IVF_FLAT partition scan, the refine step over raw vectors
// and the top-k of a distance array.
//
// Replaces  FlatDistanceCal::distance_all        lance-index/src/vector/flat/storage.rs:397-403
//           FlatIndex::search heap top-k         lance-index/src/vector/flat/index.rs:82-177
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <type_traits>

#include "common.cuh"
#include "exact.cuh"
#include "ivf_search.cuh"
#include "row_distance.cuh"
#include "scan.cuh"
#include "topk.cuh"

namespace lb2 {

// ------------------------------------------------------------------------------------------------
// IVF_FLAT: exact distances of the query to every row of a probed partition
// (FlatDistanceCal::distance_all, lance-index/src/vector/flat/storage.rs:397-403) + top-k.
// 16 lanes per row: lane l owns the reference's lane-accumulator l (elements 16c + l), so the L2 /
// dot results are bit-identical to l2.rs:57-91 / dot.rs:30-58; cosine follows cosine.rs:143-174 in
// structure (f32 FMA lanes) and is checked to the reference's own tolerance.
// ------------------------------------------------------------------------------------------------
template <int METRIC, class T>
__global__ void __launch_bounds__(256)
ivfflat_scan_kernel(const float* __restrict__ queries, int d, const uint32_t* __restrict__ probe_ids,
                    int np, const uint64_t* __restrict__ part_offsets,
                    const T* __restrict__ vectors, const uint64_t* __restrict__ row_ids, int k,
                    float* __restrict__ cand_d, uint64_t* __restrict__ cand_id,
                    uint32_t* __restrict__ cand_cnt, const ScanFilter flt0, const QueryParam* __restrict__ qp) {
  extern __shared__ float smem[];
  float* qs = smem;                          // [d]
  __shared__ float s_qnorm;
  const int tid = threadIdx.x, l = tid & 15;
  const unsigned hmask = 0xffffu << (16 * ((tid >> 4) & 1));
  size_t qi, slot;
  uint32_t p, n_p;
  uint64_t off;
  if (!slot_partition(probe_ids, np, part_offsets, cand_cnt, qi, slot, p, off, n_p)) return;
  const int kq = query_k(qp, qi, k);  // k: the lists' stride
  const ScanFilter flt = query_filter(qp, qi, flt0);
  const SlotSmem s(qs + d, kq + 1);
  for (int t = tid; t < d; t += 256) qs[t] = queries[qi * d + t];
  __syncthreads();
  if (METRIC == METRIC_COSINE && tid < 32) {  // norm_l2(query): 16 lanes + sqrt (norm_l2.rs:106-130)
    float a = 0.0f;
    for (int e = (tid & 15); e < d; e += 16) a = fmaf(qs[e], qs[e], a);
#pragma unroll
    for (int o = 8; o >= 1; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o, 16);
    if (tid == 0) s_qnorm = sqrtf(a);
  }
  __syncthreads();
  const float qn = METRIC == METRIC_COSINE ? s_qnorm : 0.0f;
  auto fill = [&](uint32_t c0, uint32_t clen) {
    for (uint32_t j = tid >> 4; j < clen; j += 16) {  // 16 rows per pass, 16 lanes each
      const float dist = flat_row_distance<METRIC, T>(qs, vectors + (off + c0 + j) * (uint64_t)d, d, l, hmask, qn);
      if (l == 0) s.ukey[j] = (uint32_t)total_order_key(dist) ^ 0x80000000u;
    }
  };
  const uint32_t cnt = slot_topk(s, n_p, kq, flt, off, false, fill);
  write_slot(s, cnt, slot, k, off, row_ids, cand_d, cand_id, cand_cnt);
}

// FlatIndex::search over a distance array (flat/index.rs:97-127): the heap's final content (the exact top-k of one
// slot, position = index into dists), written ascending by (distance, row id).
__global__ void __launch_bounds__(256)
flat_topk_kernel(const float* __restrict__ dists, const uint64_t* __restrict__ row_ids, uint64_t n,
                 int k, const ScanFilter flt, uint64_t* __restrict__ out_id, float* __restrict__ out_d,
                 uint32_t* __restrict__ out_cnt) {
  extern __shared__ float smem[];
  const SlotSmem s(smem, k + 1);
  auto fill = [&](uint32_t c0, uint32_t clen) {
    for (uint32_t j = threadIdx.x; j < clen; j += 256) s.ukey[j] = (uint32_t)total_order_key(dists[c0 + j]) ^ 0x80000000u;
  };
  const uint32_t cnt = slot_topk(s, (uint32_t)n, k, flt, 0, false, fill);
  emit_ascending<256>(
      cnt, cnt,
      [&](uint32_t i, int32_t& key, uint64_t& id) {
        key = (int32_t)(s.nkey[i] ^ 0x80000000u);
        id = row_ids ? row_ids[s.npos[i]] : (uint64_t)s.npos[i];
        return true;
      },
      [&](uint32_t r, uint32_t, int32_t key, uint64_t id) {
        out_d[r] = key_to_float(key);
        out_id[r] = id;
      });
  if (threadIdx.x == 0) *out_cnt = cnt;
}

void ivfflat_search(const IvfSearch& s, const void* vectors, int vdt) {
  const int d = s.d, k = s.k;
  const size_t smem = sizeof(float) * (size_t)d + slot_smem_bytes(k);
  size_t need = 0;
  dispatch_metric_elem<false>(s.metric, vdt, [&](auto m, auto e) {
    need = smem_with_static(ivfflat_scan_kernel<decltype(m)::value, typename decltype(e)::type>, smem);
  });
  if (!ivf_search_begin(s, need, "dimension %zu too large for the flat scan", (size_t)d)) return;
  run_ivf_search(s, [&](const ScanSlots& sl) {
    dispatch_metric_elem<false>(s.metric, vdt, [&](auto m, auto e) {
      using T = typename decltype(e)::type;
      auto kern = ivfflat_scan_kernel<decltype(m)::value, T>;
      set_smem(kern, smem);
      LB2_LAUNCH("flat_scan", kern, dim3(sl.np, (unsigned)sl.qn), 256, smem, s.queries + sl.q0 * d, d, sl.probe_ids,
                 sl.np, sl.offsets, reinterpret_cast<const T*>(vectors), s.row_ids, k, sl.cand_d, sl.cand_id,
                 sl.cand_cnt, s.flt, s.qp_at(sl.q0));
    });
  });
}

// ------------------------------------------------------------------------------------------------
// refine: exact distances of k' = k * refine_factor candidates from the raw vectors, then the k
// best by (distance, row id)  (scanner.rs:2884-2905, flat.rs:95-148)
// ------------------------------------------------------------------------------------------------
// Where the refine kernel reads candidate c's row: null scores NaN, as a row the column does not hold.
// ColumnRows: by row id from the dense column (lb2_index_search_ex / _batch's refine_vectors).
template <class T>
struct ColumnRows {
  const T* v;
  uint64_t n;
  __device__ const T* row(size_t, uint32_t, uint64_t id, int d) const { return id < n ? v + id * (uint64_t)d : nullptr; }
};
// TakenRows: by the candidate's position in the rows the caller took (lb2_index_refine_taken), [nq][stride]
template <class T>
struct TakenRows {
  const T* v;
  uint64_t m;
  const uint64_t* pos;
  int stride;
  __device__ const T* row(size_t qi, uint32_t c, uint64_t, int d) const {
    const uint64_t p = pos[qi * stride + c];
    return p < m ? v + p * (uint64_t)d : nullptr;
  }
};

// BATCH: per-query values from qo (refine_batch_f32); the single-parameter refine is compiled without them
template <int METRIC, class T, bool BATCH, class Rows>
__global__ void __launch_bounds__(256)
refine_kernel(const float* __restrict__ queries, int d, const Rows rows, const uint64_t* __restrict__ cand_id,
              const uint32_t* __restrict__ cand_cnt, int kc, int k, uint64_t* __restrict__ out_id,
              float* __restrict__ out_d, uint32_t* __restrict__ out_cnt, int has_lower, float lower, int has_upper,
              float upper, const float* __restrict__ cand_d, const QueryOut* __restrict__ qo, int k_stride) {
  extern __shared__ float smem[];
  float* qs = smem;       // [d]
  float* cd = qs + d;     // [kc]
  __shared__ float s_qnorm;
  const size_t qi = blockIdx.x;
  const int tid = threadIdx.x, l = tid & 15;
  const unsigned hmask = 0xffffu << (16 * ((tid >> 4) & 1));
  const uint64_t* ids = cand_id + qi * kc;
  if constexpr (BATCH) {  // a batch: this query's own k' (kc is the lists' stride), k, range; output rows of k_stride
    const QueryOut& o = qo[qi];
    has_lower = o.has_lower; lower = o.lower; has_upper = o.has_upper; upper = o.upper;
    if (!o.refine) {  // the merged list is the result: its first k, ascending already
      const uint32_t r = min(cand_cnt[qi], (uint32_t)o.k);
      for (int e = tid; e < k_stride; e += 256) {
        out_id[qi * k_stride + e] = (uint32_t)e < r ? ids[e] : ~0ull;
        out_d[qi * k_stride + e] = (uint32_t)e < r ? cand_d[qi * kc + e] : __int_as_float(0x7f800000);
      }
      if (tid == 0 && out_cnt) out_cnt[qi] = r;
      return;
    }
  }
  const int kcq = BATCH ? qo[qi].kc : kc, os = BATCH ? k_stride : k;
  if constexpr (BATCH) k = qo[qi].k;
  const uint32_t cnt = min(cand_cnt[qi], (uint32_t)kcq);
  for (int t = tid; t < d; t += 256) qs[t] = queries[qi * d + t];
  __syncthreads();
  if (METRIC == METRIC_COSINE && tid < 32) {
    float a = 0.0f;
    for (int e = (tid & 15); e < d; e += 16) a = fmaf(qs[e], qs[e], a);
#pragma unroll
    for (int o = 8; o >= 1; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o, 16);
    if (tid == 0) s_qnorm = sqrtf(a);
  }
  __syncthreads();
  const float qn = METRIC == METRIC_COSINE ? s_qnorm : 0.0f;
  for (uint32_t c = tid >> 4; c < cnt; c += 16) {
    const T* row = rows.row(qi, c, ids[c], d);
    float dist = __int_as_float(0x7fc00000);
    if (row) dist = refine_row_distance<METRIC, T>(qs, row, d, l, hmask, qn);
    if (l == 0) cd[c] = dist;
  }
  __syncthreads();
  auto passes = [&](float dv) {  // LanceFilterExec(_distance >= lower AND _distance < upper): SQL compares
    return (!has_lower || dv >= lower) && (!has_upper || dv < upper);
  };
  const uint32_t r = emit_ascending<256>(
      min(cnt, (uint32_t)k), cnt,
      [&](uint32_t c, int32_t& key, uint64_t& id) {
        key = total_order_key(cd[c]);
        id = ids[c];
        return passes(cd[c]);
      },
      [&](uint32_t r, uint32_t c, int32_t, uint64_t id) {
        out_id[qi * os + r] = id;
        out_d[qi * os + r] = cd[c];
      });
  for (uint32_t e = r + tid; e < (uint32_t)os; e += 256) {
    out_id[qi * os + e] = ~0ull;
    out_d[qi * os + e] = __int_as_float(0x7f800000);
  }
  if (tid == 0 && out_cnt) out_cnt[qi] = r;
}

void refine_f32(const float* queries, uint64_t nq, int d, int metric, const void* vectors, int vdt,
                uint64_t num_vectors, const uint64_t* cand_id, const uint32_t* cand_cnt, int kc, int k,
                uint64_t* out_id, float* out_d, uint32_t* out_cnt, int has_lower, float lower, int has_upper,
                float upper) {
  if (nq == 0) return;
  const size_t smem = sizeof(float) * ((size_t)d + kc);
  dispatch_metric_elem<true>(metric, vdt, [&](auto m, auto e) {
    using T = typename decltype(e)::type;
    auto kern = refine_kernel<decltype(m)::value, T, false, ColumnRows<T>>;
    set_smem(kern, smem);
    LB2_LAUNCH("refine", kern, (unsigned)nq, 256, smem, queries, d,
               ColumnRows<T>{reinterpret_cast<const T*>(vectors), num_vectors}, cand_id, cand_cnt, kc, k, out_id,
               out_d, out_cnt, has_lower, lower, has_upper, upper, (const float*)nullptr, (const QueryOut*)nullptr, k);
  });
}

void refine_batch_f32(const float* queries, uint64_t nq, int d, int metric, const void* vectors, int vdt,
                      uint64_t num_vectors, const float* cand_d, const uint64_t* cand_id, const uint32_t* cand_cnt,
                      int kc, const QueryOut* qo, int k_stride, uint64_t* out_id, float* out_d, uint32_t* out_cnt,
                      const uint64_t* positions) {
  if (nq == 0) return;
  const size_t smem = sizeof(float) * ((size_t)d + kc);
  dispatch_metric_elem<true>(metric, vdt, [&](auto m, auto e) {
    using T = typename decltype(e)::type;
    auto launch = [&](auto kern, auto rows) {
      set_smem(kern, smem);
      LB2_LAUNCH("refine", kern, (unsigned)nq, 256, smem, queries, d, rows, cand_id, cand_cnt, kc, k_stride, out_id,
                 out_d, out_cnt, 0, 0.0f, 0, 0.0f, cand_d, qo, k_stride);
    };
    const T* v = reinterpret_cast<const T*>(vectors);
    if (positions)
      launch(refine_kernel<decltype(m)::value, T, true, TakenRows<T>>, TakenRows<T>{v, num_vectors, positions, kc});
    else
      launch(refine_kernel<decltype(m)::value, T, true, ColumnRows<T>>, ColumnRows<T>{v, num_vectors});
  });
}

// lb2_index_search_candidates' rows: query q's merged list (stride kc, its own k' = qo[q].kc entries at most) into
// a row of `stride`, unused slots UINT64_MAX / +inf
__global__ void candidate_rows_kernel(const uint64_t* __restrict__ cid, const float* __restrict__ cdist,
                                      const uint32_t* __restrict__ ccnt, int kc, const QueryOut* __restrict__ qo,
                                      int stride, uint64_t* __restrict__ out_id, float* __restrict__ out_d,
                                      uint32_t* __restrict__ out_cnt) {
  const size_t qi = blockIdx.x;
  const uint32_t r = min(ccnt[qi], (uint32_t)qo[qi].kc);
  for (int e = threadIdx.x; e < stride; e += blockDim.x) {
    out_id[qi * stride + e] = (uint32_t)e < r ? cid[qi * kc + e] : ~0ull;
    out_d[qi * stride + e] = (uint32_t)e < r ? cdist[qi * kc + e] : __int_as_float(0x7f800000);
  }
  if (threadIdx.x == 0) out_cnt[qi] = r;
}

void candidate_rows(const uint64_t* cid, const float* cdist, const uint32_t* ccnt, uint64_t nq, int kc,
                    const QueryOut* qo, int stride, uint64_t* out_id, float* out_d, uint32_t* out_cnt) {
  if (nq == 0) return;
  LB2_LAUNCH("candidate_rows", candidate_rows_kernel, (unsigned)nq, 256, 0, cid, cdist, ccnt, kc, qo, stride, out_id,
             out_d, out_cnt);
}

// ------------------------------------------------------------------------------------------------
// lb2_distance_batch where the reference's arithmetic depends on the element type (l2_distance_batch /
// dot_distance_batch, l2.rs:194-203, dot.rs:164-172): u8 L2 / dot and 16-bit dot.  Half-warp per row of `to`, read
// in its own type; `from` as f32.
// ------------------------------------------------------------------------------------------------
template <int METRIC, class T>
__global__ void __launch_bounds__(256)
distance_batch_kernel(const float* __restrict__ from, const T* __restrict__ to, uint64_t n, int d,
                      float* __restrict__ out) {
  const uint64_t row = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 4;
  if (row >= n) return;  // a whole half-warp leaves: the shuffles below only name its own lanes
  const int l = threadIdx.x & 15;
  const unsigned hmask = 0xffffu << (16 * ((threadIdx.x >> 4) & 1));
  float dist;
  if constexpr (std::is_same<T, uint8_t>::value) dist = u8_row_distance<METRIC>(from, to + row * d, d, l, hmask);
  else dist = dot32_row_distance<T>(from, to + row * d, d, l, hmask);
  if (l == 0) out[row] = dist;
}

bool distance_batch_typed_applies(int dt, int metric) {
  return metric != METRIC_COSINE && (dt == LB2_U8 || (metric == METRIC_DOT && (dt == LB2_F16 || dt == LB2_BF16)));
}

void distance_batch_typed(const float* from, const void* to, int dt, uint64_t n, int d, int metric, float* out) {
  if (!distance_batch_typed_applies(dt, metric)) fail(LB2_UNSUPPORTED, "no typed distance for dtype %d, metric %d", dt, metric);
  if (n == 0) return;
  auto launch = [&](auto kern, auto rows) {
    LB2_LAUNCH("distance_batch", kern, cdiv(n * 16, 256), 256, 0, from, rows, n, d, out);
  };
  if (dt == LB2_U8 && metric == METRIC_DOT)
    launch(distance_batch_kernel<METRIC_DOT, uint8_t>, static_cast<const uint8_t*>(to));
  else if (dt == LB2_U8)
    launch(distance_batch_kernel<METRIC_L2, uint8_t>, static_cast<const uint8_t*>(to));
  else if (dt == LB2_F16)
    launch(distance_batch_kernel<METRIC_DOT, __half>, static_cast<const __half*>(to));
  else
    launch(distance_batch_kernel<METRIC_DOT, __nv_bfloat16>, static_cast<const __nv_bfloat16*>(to));
}

void flat_topk_f32(const float* dists, const uint64_t* row_ids, uint64_t n, int k, const ScanFilter& flt,
                   uint64_t* out_id, float* out_d, uint32_t* out_cnt) {
  if (k > 1024) fail(LB2_UNSUPPORTED, "k > 1024 is not implemented");
  LB2_LAUNCH("flat_topk", flat_topk_kernel, 1, 256, slot_smem_bytes(k), dists, row_ids, n, k, flt, out_id, out_d, out_cnt);
}

}  // namespace lb2
