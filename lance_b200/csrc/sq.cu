// sq.cu -- the 8-bit scalar quantizer of IVF_SQ (lance-index/src/vector/sq.rs, sq/builder.rs).
//
// Replaces  ScalarQuantizer::update_bounds   sq.rs:67-89 (the bounds of ScalarQuantizer::build, :152-182)
//           scale_to_u8                      sq.rs:263-277 (quantize / transform, and the query's codes,
//                                            sq/storage.rs:404-430)
//           SQDistCalculator::distance_all   sq/storage.rs:432-468 (the partition scan of a search)
//
// The bounds are a min / max: exact in f32 and widened to f64 afterwards, so any reduction order gives the
// reference's fold.  The encoding is restated in f64 with explicitly rounded operations (no mul-add contraction).
#include <algorithm>
#include <cfloat>
#include <vector>

#include "common.cuh"
#include "exact.cuh"
#include "ivf_search.cuh"
#include "sq.cuh"
#include "topk.cuh"

namespace lb2 {

constexpr int SQ_BOUNDS_THREADS = 256;

// per-block (min, max) of the non-NaN elements; +inf / -inf when the block saw none
__global__ void __launch_bounds__(SQ_BOUNDS_THREADS)
sq_bounds_kernel(const float* __restrict__ x, uint64_t count, float2* __restrict__ block_out) {
  float mn = __int_as_float(0x7f800000), mx = __int_as_float(0xff800000);
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (uint64_t)gridDim.x * blockDim.x) {
    const float v = x[i];
    mn = fminf(mn, v);  // fminf / fmaxf return the other operand when one is NaN, like f64::min / f64::max
    mx = fmaxf(mx, v);
  }
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) {
    mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  }
  __shared__ float s_mn[SQ_BOUNDS_THREADS / 32], s_mx[SQ_BOUNDS_THREADS / 32];
  const int warp = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) { s_mn[warp] = mn; s_mx[warp] = mx; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < SQ_BOUNDS_THREADS / 32; ++w) { mn = fminf(mn, s_mn[w]); mx = fmaxf(mx, s_mx[w]); }
    block_out[blockIdx.x] = make_float2(mn, mx);
  }
}

void sq_bounds_f32(const float* x, uint64_t count, double* lower, double* upper) {
  double lo = DBL_MAX, hi = -DBL_MAX;  // (f64::MAX, f64::MIN): what the fold starts from
  if (count) {
    const unsigned nb = (unsigned)std::min<uint64_t>(cdiv(count, SQ_BOUNDS_THREADS), 4ull * ctx().num_sms);
    DevBuf<float2> part(nb);
    std::vector<float2> h(nb);
    LB2_LAUNCH("sq_bounds", sq_bounds_kernel, nb, SQ_BOUNDS_THREADS, 0, x, count, part.p);
    d2h(h.data(), part.p, nb);
    sync_stream();
    for (const float2& b : h) {  // +inf never lowers f64::MAX, -inf never raises f64::MIN
      lo = std::min(lo, (double)b.x);
      hi = std::max(hi, (double)b.y);
    }
  }
  *lower = lo;
  *upper = hi;
}

__global__ void sq_encode_kernel(const float* __restrict__ x, uint64_t count, double lower, double upper,
                                 uint8_t* __restrict__ codes) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  if (lower == upper) {
    codes[i] = 0;
    return;
  }
  const double range = __dsub_rn(upper, lower);
  const double v = __ddiv_rn(__dmul_rn(__dsub_rn((double)x[i], lower), 255.0), range);
  // `v as u8`: NaN -> 0, truncation toward zero, saturating at 0 and 255
  codes[i] = v != v ? 0 : v <= 0.0 ? 0 : v >= 255.0 ? 255 : (uint8_t)v;
}

void sq_encode_f32(const float* x, uint64_t count, double lower, double upper, uint8_t* codes) {
  if (count) LB2_LAUNCH("sq_encode", sq_encode_kernel, cdiv(count, 256), 256, 0, x, count, lower, upper, codes);
}

// ------------------------------------------------------------------------------------------------
// IVF_SQ: SQDistCalculator::distance_all (lance-index/src/vector/sq/storage.rs:432-468) + top-k.
// A row's distance is an exact u32 integer sum over its d code bytes -- l2_distance_uint_scalar
// (lance-linalg/src/distance/l2.rs:44-49) for L2 / cosine, the u8 dot (dot.rs:152-161) for dot -- so
// any split of a row over lanes and any reduction order gives the reference's integer; d * 255^2 < 2^32
// (checked on the host) keeps it from wrapping.  Then inverse_scalar_dist (sq.rs:279-287) in f32:
// (f * (rf * rf)) / 255^2 with f = s as f32 (dot: 1 - s as f32); r2 = rf * rf comes from the host.
// 8 lanes per row; VEC4: d % 16 == 0, 16-byte loads, otherwise 4-byte words.
// ------------------------------------------------------------------------------------------------
template <int METRIC, bool VEC4>
__global__ void __maxnreg__(128)  // 256 threads; under __launch_bounds__(256) ptxas spills the selection's state
ivfsq_scan_kernel(const uint8_t* __restrict__ qcodes, int d, float r2, const uint32_t* __restrict__ probe_ids, int np,
                  const uint64_t* __restrict__ part_offsets, const uint8_t* __restrict__ codes,
                  const uint64_t* __restrict__ row_ids, int k, float* __restrict__ cand_d, uint64_t* __restrict__ cand_id,
                  uint32_t* __restrict__ cand_cnt, const ScanFilter flt0, const QueryParam* __restrict__ qp) {
  extern __shared__ uint4 sq_smem[];
  const int nw = d >> 2;                                   // 4-byte words per row
  uint32_t* qw = reinterpret_cast<uint32_t*>(sq_smem);     // the query's codes, [nw] words (16-byte aligned)
  const int tid = threadIdx.x, l = tid & 7;
  const unsigned gmask = 0xffu << (8 * ((tid >> 3) & 3));  // the row's 8 lanes
  size_t qi, slot;
  uint32_t p, n_p;
  uint64_t off;
  if (!slot_partition(probe_ids, np, part_offsets, cand_cnt, qi, slot, p, off, n_p)) return;
  const int kq = query_k(qp, qi, k);  // k: the lists' stride
  const ScanFilter flt = query_filter(qp, qi, flt0);
  const SlotSmem s(qw + ((nw + 3) & ~3), kq + 1);
  const uint32_t* qsrc = reinterpret_cast<const uint32_t*>(qcodes + qi * (size_t)d);  // d % 4 == 0: word aligned
  for (int t = tid; t < nw; t += 256) qw[t] = qsrc[t];
  __syncthreads();
  auto fill = [&](uint32_t c0, uint32_t clen) {
    for (uint32_t j = tid >> 3; j < clen; j += 32) {  // 32 rows per pass, 8 lanes each
      const uint8_t* row = codes + (off + c0 + j) * (uint64_t)d;
      uint32_t acc = 0;
      if constexpr (VEC4) {
        const uint4* r4 = reinterpret_cast<const uint4*>(row);
        const uint4* q4 = reinterpret_cast<const uint4*>(qw);
        for (int w = l; w < (nw >> 2); w += 8) {
          const uint4 x = __ldg(r4 + w), q = q4[w];
          acc = sq_word<METRIC>(x.x, q.x, acc);
          acc = sq_word<METRIC>(x.y, q.y, acc);
          acc = sq_word<METRIC>(x.z, q.z, acc);
          acc = sq_word<METRIC>(x.w, q.w, acc);
        }
      } else {
        const uint32_t* r1 = reinterpret_cast<const uint32_t*>(row);
        for (int w = l; w < nw; w += 8) acc = sq_word<METRIC>(__ldg(r1 + w), qw[w], acc);
      }
#pragma unroll
      for (int o = 4; o >= 1; o >>= 1) acc += __shfl_xor_sync(gmask, acc, o, 8);
      if (l == 0) {
        s.ukey[j] = (uint32_t)total_order_key(sq_distance<METRIC>(acc, r2)) ^ 0x80000000u;
      }
    }
  };
  const uint32_t cnt = slot_topk(s, n_p, kq, flt, off, false, fill);
  write_slot(s, cnt, slot, k, off, row_ids, cand_d, cand_id, cand_cnt);
}

void ivfsq_search(const IvfSearch& s, const uint8_t* codes, float r2, const uint8_t* qcodes) {
  const int d = s.d, k = s.k;
  const size_t smem = (size_t)(d + 15) / 16 * 16 + slot_smem_bytes(k);
  auto with_kernel = [&](auto f) {
    const bool vec4 = d % 16 == 0;
    if (s.metric == METRIC_DOT) {
      if (vec4) f(ivfsq_scan_kernel<METRIC_DOT, true>); else f(ivfsq_scan_kernel<METRIC_DOT, false>);
    } else {  // cosine: L2 on the normalised vectors' codes (sq/storage.rs:436-440)
      if (vec4) f(ivfsq_scan_kernel<METRIC_L2, true>); else f(ivfsq_scan_kernel<METRIC_L2, false>);
    }
  };
  size_t need = 0;
  with_kernel([&](auto kern) { need = smem_with_static(kern, smem); });
  if (!ivf_search_begin(s, need, "dimension %zu too large for the SQ scan", (size_t)d)) return;
  run_ivf_search(s, [&](const ScanSlots& sl) {
    with_kernel([&](auto kern) {
      set_smem(kern, smem);
      LB2_LAUNCH("sq_scan", kern, dim3(sl.np, (unsigned)sl.qn), 256, smem, qcodes + sl.q0 * d, d, r2, sl.probe_ids,
                 sl.np, sl.offsets, codes, s.row_ids, k, sl.cand_d, sl.cand_id, sl.cand_cnt, s.flt,
                 s.qp_at(sl.q0));
    });
  });
}

}  // namespace lb2
