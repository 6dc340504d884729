// row_distance.cuh -- the exact distance of a query to a stored row, per element type and metric: the one definition
// that the IVF_FLAT scan, the refine step, lb2_distance_batch's typed rule (flat_scan.cu) and the flat search
// (flat_search.cu) share, so that refine and flat search cannot drift apart.
//
// A rule has three parts, each in the reference's order:
//  * the elements lane l of a half-warp owns and how it accumulates them (rule_walk, LaneAcc::step);
//  * the sequential tail, which every lane computes redundantly (LaneAcc::s);
//  * the fold of the 16 lane partials into the distance (fold_partials).
// A per-row caller (row_distance) folds with shuffles.  The flat search's register tile keeps one LaneAcc per (query,
// row) pair and folds the same partials out of shared memory; the operations and their order are the same.
//
// Replaces  l2 / dot / cosine per element type   lance-linalg/src/distance/{l2,dot,cosine}.rs
//           compute_distance's per-type choice    lance-index/src/vector/flat.rs:94-150
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <type_traits>

#include "common.cuh"
#include "exact.cuh"

namespace lb2 {

// element of a stored / raw vector as f32 (l2.rs:100-106,156: f16 / bf16 elements are converted one by one)
template <class T> __device__ __forceinline__ float ldf(const T* p, int e);
template <> __device__ __forceinline__ float ldf<float>(const float* p, int e) { return p[e]; }
template <> __device__ __forceinline__ float ldf<__half>(const __half* p, int e) { return __half2float(p[e]); }
template <> __device__ __forceinline__ float ldf<__nv_bfloat16>(const __nv_bfloat16* p, int e) { return __bfloat162float(p[e]); }
template <> __device__ __forceinline__ float ldf<uint8_t>(const uint8_t* p, int e) { return (float)p[e]; }

// the rules:
//  LANES16: 16 f32 lanes (lane l owns elements 16c + l), no FMA contraction, the d % 16 tail summed first, the lanes
//           folded 0..15 (l2.rs:57-91, dot.rs:30-58 with LANES = 16);
//  DOT32:   dot_scalar::<T, f32, 32> (dot.rs:30-58): lane l owns accumulators l and l + 16, the d % 32 tail first,
//           the 32 sums folded 0..31;
//  U8:      exact integer sums (wrapping like the reference's release build), one conversion to f32 (l2.rs:44-49,
//           dot.rs:152-161); the query holds u8 values as f32;
//  COSINE:  cosine.rs:143-174 in structure: 16 f32 FMA lanes for <q, y> and <y, y>, a 4-level xor tree, checked to
//           the reference's own tolerance.
enum RuleKind { RULE_LANES16 = 0, RULE_DOT32 = 1, RULE_U8 = 2, RULE_COSINE = 3 };

// the IVF_FLAT scan's rule: its storage is f32 (flat/storage.rs:352-365), whatever the element type
template <int METRIC> __host__ __device__ constexpr int scan_rule() {
  return METRIC == METRIC_COSINE ? RULE_COSINE : RULE_LANES16;
}
// The refine plan's and flat_knn's rule: compute_distance takes the function of the key's own element type
// (flat.rs:94-150):
//  * f16 dot: the 32-lane dot_scalar (the fp16 C kernel is not compiled in, dot.rs:133);
//  * u8 L2 / dot: exact integer sums;
//  * everything else (f32, f16 L2, bf16, cosine) as the scan: the reference refuses bf16 keys there, so bf16 keeps
//    the scan's 16-lane rule (DESIGN.md section 5).
template <int METRIC, class T> __host__ __device__ constexpr int refine_rule() {
  return METRIC == METRIC_COSINE                                          ? RULE_COSINE
         : std::is_same<T, uint8_t>::value                                ? RULE_U8
         : (std::is_same<T, __half>::value && METRIC == METRIC_DOT)       ? RULE_DOT32
                                                                          : RULE_LANES16;
}

// lane l's partial sums of one (query, row) pair
template <int RULE, int METRIC>
struct LaneAcc {
  float a = 0.0f;   // LANES16, DOT32: the sum of lane l; COSINE: <q, y>
  float b = 0.0f;   // DOT32: the sum of lane l + 16; COSINE: <y, y>
  float s = 0.0f;   // LANES16, DOT32: the sequential tail, the same on every lane
  uint32_t u = 0;   // U8: the integer sum of lane l
  // PART 0: an element the lane owns; 1: DOT32's element 16 further on; 2: a tail element
  template <int PART>
  __device__ __forceinline__ void step(float q, float v) {
    if constexpr (RULE == RULE_COSINE) {
      a = fmaf(q, v, a);
      b = fmaf(v, v, b);
    } else if constexpr (RULE == RULE_U8) {
      const int x = __float2int_rn(q), y = __float2int_rn(v);
      u += METRIC == METRIC_DOT ? (uint32_t)(x * y) : (uint32_t)((x - y) * (x - y));
    } else if constexpr (PART == 0) {
      a = f_add(a, term<METRIC>(q, v));
    } else if constexpr (PART == 1) {
      b = f_add(b, term<METRIC>(q, v));
    } else {
      s = f_add(s, term<METRIC>(q, v));
    }
  }
};

// lane l's elements in the reference's order per accumulator: f(e, part) with part a std::integral_constant
template <int RULE, class F>
__device__ __forceinline__ void rule_walk(int d, int l, F&& f) {
  using P0 = std::integral_constant<int, 0>;
  using P1 = std::integral_constant<int, 1>;
  using P2 = std::integral_constant<int, 2>;
  if constexpr (RULE == RULE_COSINE || RULE == RULE_U8) {
    for (int e = l; e < d; e += 16) f(e, P0{});
  } else if constexpr (RULE == RULE_DOT32) {
    const int n32 = d & ~31;
    for (int e = l; e < n32; e += 32) {
      f(e, P0{});
      f(e + 16, P1{});
    }
    for (int e = n32; e < d; ++e) f(e, P2{});
  } else {
    const int n16 = d & ~15;
    for (int e = l; e < n16; e += 16) f(e, P0{});
    for (int e = n16; e < d; ++e) f(e, P2{});
  }
}

__device__ __forceinline__ float cosine_finish(float xy, float yy, float q_norm) { return 1.0f - xy / q_norm / sqrtf(yy); }

// The value the xor-shuffle tree (offsets 8, 4, 2, 1) leaves on every lane, from the 16 lane partials a(0..15): at
// each level lane i adds lane i ^ off, and f32 addition is commutative, so this is bit for bit the shuffle result.
template <class A>
__device__ __forceinline__ float tree16(A a) {
  float v[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) v[i] = a(i);
#pragma unroll
  for (int off = 8; off >= 1; off >>= 1) {
#pragma unroll
    for (int i = 0; i < off; ++i) v[i] = v[i] + v[i + off];
  }
  return v[0];
}

// The distance from the lane partials of one pair: a(i), b(i), u(i) read lane i's LaneAcc fields, s is the tail.
// LANES16 / DOT32 fold 0..15 (DOT32: then lanes 16..31) onto the tail; U8 sums exactly; COSINE takes the xor tree.
template <int RULE, int METRIC, class A, class B, class U>
__device__ __forceinline__ float fold_partials(A a, B b, U u, float s, float q_norm) {
  if constexpr (RULE == RULE_COSINE) {
    return cosine_finish(tree16(a), tree16(b), q_norm);
  } else if constexpr (RULE == RULE_U8) {
    uint32_t acc = 0;
#pragma unroll
    for (int i = 0; i < 16; ++i) acc += u(i);
    return finish<METRIC>(__uint2float_rn(acc));
  } else {
    float t = 0.0f;
#pragma unroll
    for (int i = 0; i < 16; ++i) t = f_add(t, a(i));
    if constexpr (RULE == RULE_DOT32) {
#pragma unroll
      for (int i = 0; i < 16; ++i) t = f_add(t, b(i));
    }
    return finish<METRIC>(f_add(s, t));
  }
}

// One row, one half-warp (lane l of the 16 lanes in `mask`): q is the query as f32, q_norm its norm (cosine only).
// Cosine and u8 reduce with the xor tree, which gives the same value as fold_partials in fewer shuffles.
template <int RULE, int METRIC, class T>
__device__ __forceinline__ float row_distance(const float* __restrict__ q, const T* __restrict__ v, int d, int l,
                                              unsigned mask, float q_norm) {
  LaneAcc<RULE, METRIC> acc;
  rule_walk<RULE>(d, l, [&](int e, auto part) { acc.template step<decltype(part)::value>(q[e], ldf<T>(v, e)); });
  if constexpr (RULE == RULE_COSINE) {
#pragma unroll
    for (int off = 8; off >= 1; off >>= 1) {
      acc.a += __shfl_xor_sync(mask, acc.a, off, 16);
      acc.b += __shfl_xor_sync(mask, acc.b, off, 16);
    }
    return cosine_finish(acc.a, acc.b, q_norm);
  } else if constexpr (RULE == RULE_U8) {
#pragma unroll
    for (int off = 8; off >= 1; off >>= 1) acc.u += __shfl_xor_sync(mask, acc.u, off, 16);
    return finish<METRIC>(__uint2float_rn(acc.u));
  } else {
    return fold_partials<RULE, METRIC>([&](int i) { return __shfl_sync(mask, acc.a, i, 16); },
                                       [&](int i) { return __shfl_sync(mask, acc.b, i, 16); },
                                       [](int) { return 0u; }, acc.s, q_norm);
  }
}

// lb2_distance_batch's cosine (cosine_distance_batch, cosine.rs:143-174,266-290) over one warp: lane l owns elements
// l, l + 32, .. and accumulates <x, y> with FMA; the 32 partials are folded with the xor tree (offsets 16 .. 1).
// <x, x> is cos32_sum(x, x).  The distance of `from` to `to` is cos32_finish(<from, to>, <from, from>, <to, to>).
template <class T, class U>
__device__ __forceinline__ float cos32_sum(const T* __restrict__ x, const U* __restrict__ y, int d, int lane) {
  float s = 0.0f;
  for (int e = lane; e < d; e += 32) s = fmaf(ldf<T>(x, e), ldf<U>(y, e), s);
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  return s;
}
// <x, x>, <x, y> and <y, y> as three cos32_sum would give them, in one pass over x and y
template <class T, class U>
__device__ __forceinline__ void cos32_sums(const T* __restrict__ x, const U* __restrict__ y, int d, int lane,
                                           float& xx, float& xy, float& yy) {
  xx = 0.0f, xy = 0.0f, yy = 0.0f;
  for (int e = lane; e < d; e += 32) {
    const float a = ldf<T>(x, e), b = ldf<U>(y, e);
    xx = fmaf(a, a, xx);
    xy = fmaf(a, b, xy);
    yy = fmaf(b, b, yy);
  }
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) {
    xx += __shfl_xor_sync(0xffffffffu, xx, o);
    xy += __shfl_xor_sync(0xffffffffu, xy, o);
    yy += __shfl_xor_sync(0xffffffffu, yy, o);
  }
}
// cos32_sum's value computed by one thread: the 32 lane partials in registers, folded as the xor tree folds them onto
// lane 0 (at offset o, partial i < o takes partial i + o; f32 addition is commutative)
__device__ __forceinline__ float cos32_sum_thread(const float* __restrict__ x, const float* __restrict__ y, int d) {
  float v[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) v[i] = 0.0f;
  for (int c = 0; c < d; c += 32) {
#pragma unroll
    for (int i = 0; i < 32; ++i)
      if (c + i < d) v[i] = fmaf(x[c + i], y[c + i], v[i]);
  }
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) {
#pragma unroll
    for (int i = 0; i < o; ++i) v[i] = v[i] + v[i + o];
  }
  return v[0];
}
__device__ __forceinline__ float cos32_finish(float xy, float from_sq, float to_sq) {
  return 1.0f - xy / sqrtf(from_sq) / sqrtf(to_sq);
}

// One pair by one thread: the 16 lanes of the rule as 16 LaneAcc in registers, folded as fold_partials folds them (the
// value row_distance leaves on its lanes).  Not for cosine, whose per-row form is the xor tree of row_distance.
template <int RULE, int METRIC, class T>
__device__ __forceinline__ float thread_distance(const float* __restrict__ q, const T* __restrict__ v, int d) {
  static_assert(RULE != RULE_COSINE, "thread_distance: cosine folds with the xor tree");
  LaneAcc<RULE, METRIC> acc[16];
#pragma unroll
  for (int l = 0; l < 16; ++l)
    rule_walk<RULE>(d, l, [&](int e, auto part) { acc[l].template step<decltype(part)::value>(q[e], ldf<T>(v, e)); });
  return fold_partials<RULE, METRIC>([&](int i) { return acc[i].a; }, [&](int i) { return acc[i].b; },
                                     [&](int i) { return acc[i].u; }, acc[0].s, 0.0f);
}

// the IVF_FLAT scan: FlatDistanceCal::distance_all (flat/storage.rs:397-403)
template <int METRIC, class T = float>
__device__ __forceinline__ float flat_row_distance(const float* __restrict__ q, const T* __restrict__ v, int d, int l,
                                                   unsigned mask, float q_norm) {
  return row_distance<scan_rule<METRIC>(), METRIC, T>(q, v, d, l, mask, q_norm);
}
// u8 L2 / dot (lb2_distance_batch and refine)
template <int METRIC>
__device__ __forceinline__ float u8_row_distance(const float* __restrict__ q, const uint8_t* __restrict__ v, int d,
                                                 int l, unsigned mask) {
  return row_distance<RULE_U8, METRIC, uint8_t>(q, v, d, l, mask, 0.0f);
}
// 16-bit dot with 32 lanes: bf16 always (dot.rs:78-83), f16 without the fp16 C kernel (dot.rs:133)
template <class T>
__device__ __forceinline__ float dot32_row_distance(const float* __restrict__ q, const T* __restrict__ v, int d,
                                                    int l, unsigned mask) {
  return row_distance<RULE_DOT32, METRIC_DOT, T>(q, v, d, l, mask, 0.0f);
}
// the refine plan (and flat_knn): the key's element type decides (refine_rule)
template <int METRIC, class T>
__device__ __forceinline__ float refine_row_distance(const float* __restrict__ q, const T* __restrict__ v, int d,
                                                     int l, unsigned mask, float q_norm) {
  return row_distance<refine_rule<METRIC, T>(), METRIC, T>(q, v, d, l, mask, q_norm);
}

// f(metric, element) with the metric as a std::integral_constant and the element type as a type_tag
template <class T> struct type_tag { using type = T; };
template <bool WITH_U8, class F>
static void dispatch_metric_elem(int metric, int vdt, F&& f) {
  auto by_elem = [&](auto m) {
    if (vdt == LB2_F16) f(m, type_tag<__half>{});
    else if (vdt == LB2_BF16) f(m, type_tag<__nv_bfloat16>{});
    else if constexpr (WITH_U8) {
      if (vdt == LB2_U8) f(m, type_tag<uint8_t>{}); else f(m, type_tag<float>{});
    } else f(m, type_tag<float>{});
  };
  if (metric == METRIC_DOT) by_elem(std::integral_constant<int, METRIC_DOT>{});
  else if (metric == METRIC_COSINE) by_elem(std::integral_constant<int, METRIC_COSINE>{});
  else by_elem(std::integral_constant<int, METRIC_L2>{});
}

}  // namespace lb2
