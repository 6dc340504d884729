// search.cu -- query-time kernels.
//
// Replaces  kmeans_find_partitions               lance-index/src/vector/kmeans.rs:1134-1158
//           IVFIndex::preprocess_query           rust/lance/src/index/vector/ivf/v2.rs:316-332
//           build_distance_table_l2/_dot         lance-index/src/vector/pq/distance.rs:24-92
//           compute_pq_distance (+ Dot fix-up)   pq/distance.rs:109-144, pq/storage.rs:921-962
//           FlatIndex::search heap top-k         lance-index/src/vector/flat/index.rs:82-177
//           SortExec(_distance,_rowid).fetch(k)  rust/lance/src/dataset/scanner.rs:3450-3466
//
// One CTA per (query, probed partition): the residual query and its M x 256 f32 lookup table are
// built in shared memory (never written to HBM), the partition's codes are streamed once with
// 128-bit loads, each row's distance is the reference's m-ascending f32 sum (bit-exact), and
// warp-level sorting networks (k <= 16) or a block radix select produce the k smallest (distance,
// position) pairs.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <type_traits>

#include "assign.cuh"
#include "comm.cuh"
#include "common.cuh"
#include "exact.cuh"
#include "probe.cuh"
#include "rq.cuh"
#include "search.cuh"

namespace lb2 {

// prefilter (PreFilter::mask, lance-index/src/prefilter.rs:27-51; FlatIndex::search :129-165): one bit
// per STORAGE position (partition-sorted order); a cleared bit removes the row from the scan.  Filtered
// rows get the maximal key, so they can only surface when fewer than k allowed rows exist, and the
// output stage drops them by re-testing the bit.
__device__ __forceinline__ bool row_allowed(const uint64_t* __restrict__ allow, uint64_t pos) {
  return allow == nullptr || ((allow[pos >> 6] >> (pos & 63)) & 1ull) != 0;
}
// range query (flat/index.rs:100-115): a row enters the heap iff lower <= dist < upper in f32::total_cmp
// order; an absent bound is f32::MIN / f32::MAX (NOT -inf / +inf), exactly as the reference unwraps them
__device__ __forceinline__ bool key_in_range(const ScanFilter& f, int32_t key) {
  return !f.range || (key >= f.lo_key && key < f.hi_key);
}

// ---- Rust std BinaryHeap<OrderedNode> restated (alloc::collections::binary_heap: push = sift_up,
// pop = swap with the last + sift_down_to_bottom + sift_up) on (unsigned order key, position) pairs.
// OrderedNode compares by distance only (graph.rs:117-121), so WHICH of several rows tied at the k-th
// distance survives FlatIndex::search's `if root.dist > dist { pop; push }` loop (flat/index.rs:116-126)
// depends on this exact sift order.  The parallel selections below return the k smallest (distance,
// position) pairs, which is the same SET unless more rows tie at the k-th distance than fit; exactly
// then (detected by selecting k + 1) the slot is replayed sequentially through this heap.
__device__ __forceinline__ void rheap_sift_up(uint32_t* hk, uint32_t* hp, uint32_t pos) {
  const uint32_t ek = hk[pos], ep = hp[pos];
  while (pos > 0) {
    const uint32_t parent = (pos - 1) >> 1;
    if (ek <= hk[parent]) break;
    hk[pos] = hk[parent];
    hp[pos] = hp[parent];
    pos = parent;
  }
  hk[pos] = ek;
  hp[pos] = ep;
}
__device__ __forceinline__ void rheap_push(uint32_t* hk, uint32_t* hp, uint32_t& len, uint32_t key, uint32_t pos) {
  hk[len] = key;
  hp[len] = pos;
  rheap_sift_up(hk, hp, len);
  ++len;
}
__device__ __forceinline__ void rheap_pop(uint32_t* hk, uint32_t* hp, uint32_t& len) {
  --len;
  if (len == 0) return;
  const uint32_t ek = hk[len], ep = hp[len];  // the last element moves to the root, then sinks to the bottom
  uint32_t pos = 0, child = 1;
  const uint32_t end = len;
  while (child + 1 < end) {
    if (hk[child] <= hk[child + 1]) child += 1;
    hk[pos] = hk[child];
    hp[pos] = hp[child];
    pos = child;
    child = 2 * pos + 1;
  }
  if (child + 1 == end) {
    hk[pos] = hk[child];
    hp[pos] = hp[child];
    pos = child;
  }
  hk[pos] = ek;
  hp[pos] = ep;
  rheap_sift_up(hk, hp, pos);
}
// FlatIndex::search's insertion rule for one row (flat/index.rs:116-126); keys are unsigned order keys
__device__ __forceinline__ void rheap_offer(uint32_t* hk, uint32_t* hp, uint32_t& len, uint32_t k, uint32_t key,
                                            uint32_t pos) {
  if (len < k) {
    rheap_push(hk, hp, len, key, pos);
  } else if (hk[0] > key) {
    rheap_pop(hk, hp, len);
    rheap_push(hk, hp, len, key, pos);
  }
}


// ------------------------------------------------------------------------------------------------
// block-level helpers
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool ki_less(int32_t k1, uint64_t i1, int32_t k2, uint64_t i2) {
  return k1 < k2 || (k1 == k2 && i1 < i2);
}

// argmin over (key, tie) proposed by every thread of a 256/128-thread block; returns the winning
// thread id (all threads get it).  Threads with nothing to propose pass has=false.
template <int NT>
__device__ inline int block_argmin(bool has, int32_t key, uint64_t tie, int32_t* s_key,
                                   uint64_t* s_tie, int* s_tid) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  int who = has ? tid : -1;
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) {
    const int32_t ok = __shfl_xor_sync(0xffffffffu, key, off);
    const uint64_t ot = __shfl_xor_sync(0xffffffffu, tie, off);
    const int ow = __shfl_xor_sync(0xffffffffu, who, off);
    if (ow >= 0 && (who < 0 || ki_less(ok, ot, key, tie))) {
      key = ok; tie = ot; who = ow;
    }
  }
  if (lane == 0) { s_key[warp] = key; s_tie[warp] = tie; s_tid[warp] = who; }
  __syncthreads();
  if (tid == 0) {
    int bw = s_tid[0];
    int32_t bk = s_key[0];
    uint64_t bt = s_tie[0];
    for (int w = 1; w < NT / 32; ++w)
      if (s_tid[w] >= 0 && (bw < 0 || ki_less(s_key[w], s_tie[w], bk, bt))) {
        bw = s_tid[w]; bk = s_key[w]; bt = s_tie[w];
      }
    s_tid[NT / 32] = bw;
  }
  __syncthreads();
  const int winner = s_tid[NT / 32];
  __syncthreads();
  return winner;
}

// Ordered emission: round r finds the smallest (key, tie) strictly after round r - 1's among the candidates
// i in [0, n) for which cand(i, key, tie) returns true, and emit(r, i, key, tie) runs on the thread that proposed
// it.  Stops after `rounds` rounds or when no candidate is left; returns the number of rounds that emitted.
template <int NT, class Cand, class Emit>
__device__ __forceinline__ uint32_t emit_ascending(uint32_t rounds, uint32_t n, Cand cand, Emit emit) {
  __shared__ int32_t s_key[NT / 32];
  __shared__ uint64_t s_tie[NT / 32];
  __shared__ int s_tid[NT / 32 + 1];
  __shared__ int32_t prev_key;
  __shared__ uint64_t prev_tie;
  const int tid = threadIdx.x;
  uint32_t r = 0;
  for (; r < rounds; ++r) {
    int32_t bk = 0;
    uint64_t bt = 0;
    uint32_t bi = 0;
    bool has = false;
    const int32_t pk = r ? prev_key : 0;
    const uint64_t pt = r ? prev_tie : 0;
    for (uint32_t i = tid; i < n; i += NT) {
      int32_t key;
      uint64_t tie;
      if (!cand(i, key, tie) || (r && !ki_less(pk, pt, key, tie))) continue;  // none, or already emitted
      if (!has || ki_less(key, tie, bk, bt)) { bk = key; bt = tie; bi = i; has = true; }
    }
    const int w = block_argmin<NT>(has, bk, bt, s_key, s_tie, s_tid);
    if (w < 0) break;
    if (tid == w) {
      prev_key = bk;
      prev_tie = bt;
      emit(r, bi, bk, bt);
    }
    __syncthreads();
  }
  return r;
}

// ------------------------------------------------------------------------------------------------
// coarse probe selection: nprobes smallest (distance, id), ascending (kmeans.rs:1152-1157)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128)
select_probes_kernel(const float* __restrict__ all_dists, int K, int nprobes,
                     uint32_t* __restrict__ ids, float* __restrict__ dists) {
  const float* row = all_dists + (size_t)blockIdx.x * K;
  emit_ascending<128>(
      nprobes, K,
      [&](uint32_t c, int32_t& key, uint64_t& tie) {
        key = total_order_key(row[c]);
        tie = c;
        return true;
      },
      [&](uint32_t r, uint32_t c, int32_t, uint64_t) {
        ids[(size_t)blockIdx.x * nprobes + r] = c;
        dists[(size_t)blockIdx.x * nprobes + r] = row[c];
      });
}

// LUT[m][c] = dist(q_m, cb[m][c])  (pq/distance.rs:38-56).  For the common sub-vector widths the
// codeword is fetched with 128-bit loads and the reference-order sum is fully unrolled.
template <int METRIC, int DS>
__device__ __forceinline__ float lut_entry_fixed(const float* __restrict__ qm, const float* __restrict__ cw) {
  float qv[DS], cv[DS];
#pragma unroll
  for (int t = 0; t < DS; t += 4) {
    const float4 a = *reinterpret_cast<const float4*>(qm + t);
    const float4 b = __ldg(reinterpret_cast<const float4*>(cw + t));
    qv[t] = a.x; qv[t + 1] = a.y; qv[t + 2] = a.z; qv[t + 3] = a.w;
    cv[t] = b.x; cv[t + 1] = b.y; cv[t + 2] = b.z; cv[t + 3] = b.w;
  }
  if (DS < 16) {  // tail-only path (l2.rs:69-79): plain left-to-right sum
    float s = 0.0f;
#pragma unroll
    for (int t = 0; t < DS; ++t) s = f_add(s, term<METRIC>(qv[t], cv[t]));
    return finish<METRIC>(f_add(s, 0.0f));
  } else {        // DS == 16: one chunk of 16 lanes, summed lane 0..15
    float t0 = 0.0f;
#pragma unroll
    for (int t = 0; t < 16; ++t) t0 = f_add(t0, f_add(0.0f, term<METRIC>(qv[t], cv[t])));
    return finish<METRIC>(f_add(0.0f, t0));
  }
}
template <int METRIC>
__device__ __forceinline__ void build_lut_smem(float* lut, const float* qr, const float* __restrict__ codebook,
                                               int M, int ds, int tid) {
  if (ds == 8) {
    for (int idx = tid; idx < M * 256; idx += 256)
      lut[idx] = lut_entry_fixed<METRIC, 8>(qr + (idx >> 8) * 8, codebook + (size_t)idx * 8);
  } else if (ds == 4) {
    for (int idx = tid; idx < M * 256; idx += 256)
      lut[idx] = lut_entry_fixed<METRIC, 4>(qr + (idx >> 8) * 4, codebook + (size_t)idx * 4);
  } else if (ds == 16) {
    for (int idx = tid; idx < M * 256; idx += 256)
      lut[idx] = lut_entry_fixed<METRIC, 16>(qr + (idx >> 8) * 16, codebook + (size_t)idx * 16);
  } else {
    for (int idx = tid; idx < M * 256; idx += 256)
      lut[idx] = dist_exact_thread<METRIC>(qr + (idx >> 8) * ds, codebook + (size_t)idx * ds, ds);
  }
}

// ------------------------------------------------------------------------------------------------
// the fused (residual query -> LUT -> code scan -> top-k) kernels: one CTA per (query, probed
// partition).  Partitions are processed in chunks of <= SCAN_CHUNK rows, the winners of a chunk
// joining the next chunk's candidate pool.
// ------------------------------------------------------------------------------------------------
constexpr int SCAN_CHUNK = 4096;

__device__ __forceinline__ float key_to_float(int32_t key) {
  return __int_as_float(key ^ (int32_t)((uint32_t)(key >> 31) >> 1));
}

// arguments shared by the fused scan kernels (one slot = one (query, probed partition) pair)
struct ScanArgs {
  const float* queries; int d; const float* centroids; const float* codebook; int M, ds;
  const uint32_t* probe_ids; int np; const uint64_t* part_offsets; const uint8_t* codes;
  const uint64_t* row_ids; int k; float* cand_d; uint64_t* cand_id; uint32_t* cand_cnt;
  ScanFilter flt;
};

// the residual query of partition p (v2.rs:316-332) and its LUT, in shared memory (256 threads)
template <int METRIC, int NBITS>
__device__ __forceinline__ void stage_query_lut(float* lut, float* qr, const ScanArgs& a, size_t qi, uint32_t p) {
  const float* q = a.queries + qi * a.d;
  for (int t = threadIdx.x; t < a.d; t += 256)
    qr[t] = METRIC == METRIC_DOT ? q[t] : __fsub_rn(q[t], a.centroids[(size_t)p * a.d + t]);
  __syncthreads();
  if (NBITS == 8) {
    build_lut_smem<METRIC>(lut, qr, a.codebook, a.M, a.ds, threadIdx.x);
  } else {
    for (int idx = threadIdx.x; idx < a.M * 16; idx += 256)
      lut[idx] = dist_exact_thread<METRIC>(qr + (idx / 16) * a.ds, a.codebook + (size_t)idx * a.ds, a.ds);
  }
  __syncthreads();
}

// one row's 8-bit ADC distance: the reference's m-ascending f32 sum of LUT[m][code[m]] (pq/distance.rs:109-144)
__device__ __forceinline__ float pq8_row_distance(const float* lut, const uint8_t* __restrict__ rp, int M) {
  float dist = 0.0f;
  if ((M & 15) == 0) {
    const uint4* rp4 = reinterpret_cast<const uint4*>(rp);
    for (int c16 = 0; c16 < M / 16; ++c16) {
      const uint4 v = __ldg(rp4 + c16);
      const uint32_t w[4] = {v.x, v.y, v.z, v.w};
      const float* l0 = lut + c16 * 16 * 256;
#pragma unroll
      for (int aa = 0; aa < 4; ++aa)
#pragma unroll
        for (int bb = 0; bb < 4; ++bb)
          dist = f_add(dist, l0[(aa * 4 + bb) * 256 + ((w[aa] >> (8 * bb)) & 0xff)]);
    }
  } else {
    for (int m = 0; m < M; ++m) dist = f_add(dist, lut[m * 256 + rp[m]]);
  }
  return dist;
}

// The 4-bit quantisation range (qmax - qmin) / 255 and the dequantisation q * range + qmin as x86 (where the reference
// runs) evaluates them when the table is not finite: r = a op b, but an invalid operation (0 * Inf, Inf - Inf) gives
// the default NaN 0xFFC00000, whose sign bit puts it before every number in f32::total_cmp order, and a NaN operand
// passes through.  The device's own NaN is 0x7FFFFFFF, which orders after every number.
__device__ __forceinline__ float x86_nan(float r, float a, float b) {
  return r == r ? r : a != a ? a : b != b ? b : __int_as_float(0xffc00000);
}
__device__ __forceinline__ float pq4_dequantize(uint32_t q, const float* params) {
  const float qf = (float)q, p = x86_nan(__fmul_rn(qf, params[1]), qf, params[1]);
  return x86_nan(__fadd_rn(p, params[0]), p, params[0]);
}

// 4-bit table quantisation (pq/distance.rs:147-242), one block of 256 threads: qmin = min(table) (f32::min ignores
// NaN), qmax = max of the flat rows' distances flat_dist(j), j < flat_num, in total order; qt = the table quantised
// to u8, params = {qmin, (qmax - qmin) / 255}.  r_mx / r_mn: 256 entries of reduction scratch each.
template <class FlatDist>
__device__ __forceinline__ void pq4_quantize(const float* lut, int M, uint64_t flat_num, FlatDist flat_dist, uint8_t* qt,
                             float* params, int32_t* r_mx, float* r_mn) {
  const int tid = threadIdx.x;
  int32_t mx = (int32_t)0x80000000;
  for (uint64_t j = tid; j < flat_num; j += 256) mx = max(mx, total_order_key(flat_dist(j)));
  float mn = __int_as_float(0x7f800000);
  for (int i = tid; i < M * 16; i += 256) mn = fminf(mn, lut[i]);
  r_mx[tid] = mx;
  r_mn[tid] = mn;
  __syncthreads();
  for (int o = 128; o >= 1; o >>= 1) {
    if (tid < o) {
      r_mx[tid] = max(r_mx[tid], r_mx[tid + o]);
      r_mn[tid] = fminf(r_mn[tid], r_mn[tid + o]);
    }
    __syncthreads();
  }
  const float qmax = key_to_float(r_mx[0]), qmin = r_mn[0];
  __syncthreads();
  const float factor = __fdiv_rn(255.0f, __fsub_rn(qmax, qmin));
  for (int i = tid; i < M * 16; i += 256) {
    const float v = roundf(__fmul_rn(__fsub_rn(lut[i], qmin), factor));  // f32::round: half away from zero
    qt[i] = (v != v) ? 0 : v <= 0.0f ? 0 : v >= 255.0f ? 255 : (uint8_t)v;  // `as u8`: saturating, NaN -> 0
  }
  if (tid == 0) {
    params[0] = qmin;
    const float span = x86_nan(__fsub_rn(qmax, qmin), qmax, qmin);
    params[1] = x86_nan(__fdiv_rn(span, 255.0f), span, 255.0f);
  }
  __syncthreads();
}

// ------------------------------------------------------------------------------------------------
// Exact top-k of one slot (16 < k <= 1024 in the PQ scan, every k in the IVF_FLAT scan and lb2_flat_topk), 256
// threads.  A row's distance is an unsigned order key (unsigned order == f32::total_cmp order); the caller's fill
// step writes the keys of rows [c0, c0 + clen) to ukey.  Per chunk of SCAN_CHUNK rows the kk = k + 1 smallest
// (key, position) pairs of the chunk and the winners carried from earlier chunks are found by a 4-pass MSB radix
// select over shared-memory keys (256-bin histograms): everything below the kk-th key is kept, ties AT it are
// resolved by position (earliest rows survive).  Selecting one more than asked for exposes ties that overflow the
// k-th place; those slots are replayed through the reference's heap.
// ------------------------------------------------------------------------------------------------
// shared memory of one slot (u32 words): ukey[SCAN_CHUNK + kk] (a chunk's keys, then the carried winners' keys),
// cpos[kk] (the carried winners' positions), nkey[kk] / npos[kk] (the next winners; the result; the replay heap)
__host__ __device__ constexpr size_t slot_smem_bytes(int k) {
  return sizeof(uint32_t) * (SCAN_CHUNK + 4 * (size_t)(k + 1));
}
struct SlotSmem {
  uint32_t *ukey, *cpos, *nkey, *npos;
  __device__ SlotSmem(void* base, int kk)
      : ukey(static_cast<uint32_t*>(base)), cpos(ukey + SCAN_CHUNK + kk), nkey(cpos + kk), npos(nkey + kk) {}
};

// a row the prefilter (bit at off + row) or the range removes
__device__ __forceinline__ bool slot_excluded(const ScanFilter& f, uint64_t off, uint32_t row, uint32_t ukey) {
  return !row_allowed(f.allow, off + row) || !key_in_range(f, (int32_t)(ukey ^ 0x80000000u));
}

// The kk smallest (key, position) pairs of rows [0, n); excluded rows take the maximal key, so they only surface when
// fewer than kk rows are left.  Returns their number; they are left unordered at ukey[SCAN_CHUNK ..) / cpos.
// max_admitted: some admitted row has the maximal key too (a NaN distance), so it ties with the excluded rows.
template <class Fill>
__device__ __forceinline__ uint32_t slot_select(const SlotSmem& s, uint32_t n, uint32_t kk, const ScanFilter& flt, uint64_t off,
                                Fill fill, bool& max_admitted) {
  __shared__ uint32_t hist[256], s_wsum[8];
  __shared__ uint32_t s_prefix, s_need, s_eq, s_out, s_maxadm;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const bool filtering = flt.allow != nullptr || flt.range;
  uint32_t nw = 0;
  // once kk winners are carried, a chunk row whose key is >= lim (>= the kk-th carried key) cannot enter: kk
  // carried winners precede it in (key, position) order.  Such rows are left out of the pool.
  uint32_t lim = 0xffffffffu;
  bool full = false;
  if (tid == 0) s_maxadm = 0;  // ordered before any store by the barrier after the first fill
  for (uint32_t c0 = 0; c0 < n; c0 += SCAN_CHUNK) {
    const uint32_t clen = min((uint32_t)SCAN_CHUNK, n - c0);
    fill(c0, clen);
    __syncthreads();
    if (filtering) {
      for (uint32_t j = tid; j < clen; j += 256) {
        if (slot_excluded(flt, off, c0 + j, s.ukey[j])) s.ukey[j] = 0xffffffffu;
        else if (s.ukey[j] == 0xffffffffu) s_maxadm = 1;
      }
      __syncthreads();
    }
    // pool element i: i < clen -> (ukey[i], c0 + i), else the carried winner i - clen at ukey[SCAN_CHUNK ..)
    const uint32_t pool = clen + nw;
    auto key_at = [&](uint32_t i) { return i < clen ? s.ukey[i] : s.ukey[SCAN_CHUNK + (i - clen)]; };
    auto pos_at = [&](uint32_t i) { return i < clen ? c0 + i : s.cpos[i - clen]; };
    auto pooled = [&](uint32_t i, uint32_t kv) { return !full || i >= clen || kv < lim; };
    if (pool <= kk) {
      for (uint32_t i = tid; i < pool; i += 256) { s.nkey[i] = key_at(i); s.npos[i] = pos_at(i); }
      __syncthreads();
      for (uint32_t i = tid; i < pool; i += 256) { s.ukey[SCAN_CHUNK + i] = s.nkey[i]; s.cpos[i] = s.npos[i]; }
      nw = pool;
      full = nw == kk;
      __syncthreads();
      continue;
    }
    if (tid == 0) { s_prefix = 0; s_need = kk; }
    uint32_t mask = 0;
    for (int shift = 24; shift >= 0; shift -= 8) {
      hist[tid] = 0;
      __syncthreads();
      const uint32_t prefix = s_prefix, need = s_need;
      for (uint32_t i = tid; i < pool; i += 256) {
        const uint32_t kv = key_at(i);
        if (pooled(i, kv) && (kv & mask) == prefix) atomicAdd(&hist[(kv >> shift) & 255u], 1u);
      }
      __syncthreads();
      // the bin of the need-th key: the one whose inclusive prefix sum first reaches `need` (bin = thread)
      const uint32_t h = hist[tid];
      uint32_t cum = h;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t v = __shfl_up_sync(0xffffffffu, cum, o);
        if (lane >= o) cum += v;
      }
      if (lane == 31) s_wsum[warp] = cum;
      __syncthreads();
      for (int w = 0; w < warp; ++w) cum += s_wsum[w];
      if (cum >= need && cum - h < need) {
        s_need = need - (cum - h);
        s_prefix = prefix | ((uint32_t)tid << shift);
        s_eq = h;
      }
      mask |= 0xffu << shift;
      __syncthreads();
    }
    const uint32_t T = s_prefix, need = s_need, eq = s_eq;  // take all keys < T and `need` of the `eq` keys == T
    if (tid == 0) s_out = 0;
    __syncthreads();
    for (uint32_t i = tid; i < pool; i += 256) {
      const uint32_t kv = key_at(i);
      if (pooled(i, kv) && (kv < T || (kv == T && eq == need))) {
        const uint32_t at = atomicAdd(&s_out, 1u);
        s.nkey[at] = kv;
        s.npos[at] = pos_at(i);
      }
    }
    __syncthreads();
    if (eq != need)  // ties at the last key: the `need` smallest positions survive (rare)
      emit_ascending<256>(
          need, pool,
          [&](uint32_t i, int32_t& key, uint64_t& tie) {
            const uint32_t kv = key_at(i);
            key = 0;
            tie = pos_at(i);
            return kv == T && pooled(i, kv);
          },
          [&](uint32_t, uint32_t, int32_t, uint64_t tie) {
            const uint32_t at = s_out;
            s.nkey[at] = T;
            s.npos[at] = (uint32_t)tie;
            s_out = at + 1;
          });
    const uint32_t got = s_out;  // == kk
    __syncthreads();
    for (uint32_t i = tid; i < got; i += 256) { s.ukey[SCAN_CHUNK + i] = s.nkey[i]; s.cpos[i] = s.npos[i]; }
    nw = got;
    full = true;
    lim = T;
    __syncthreads();
  }
  max_admitted = n > 0 && s_maxadm != 0;  // every pass of the loop ends in a barrier
  return nw;
}

// The finish, on the nw <= kk winners in (key, position) order: excluded winners at the end are dropped (they carry
// the maximal key; an admitted row whose key is the maximal one, e.g. a NaN distance, keeps the excluded winners before
// it).  If kk winners remain and the last two share a key, more rows tie at the k-th distance than fit and the
// reference's heap decides: returns false.  So it does when excluded winners were dropped from the end of a full
// selection while an admitted row shares their key (max_admitted): admitted rows behind the kk may then belong in the
// result.  Otherwise leaves the admitted winners among the first k at nkey / npos (unordered), sets *cnt and returns
// true.
__device__ __forceinline__ bool slot_finish(const SlotSmem& s, uint32_t nw, uint32_t kk, bool max_admitted,
                            const ScanFilter& flt, uint64_t off, uint32_t* cnt) {
  __shared__ uint32_t s_kept, s_max, s_maxcnt, s_last, s_mid, s_out;
  const int tid = threadIdx.x;
  if (tid == 0) { s_kept = 0; s_max = 0; s_maxcnt = 0; s_last = 0; s_mid = 0; s_out = 0; }
  __syncthreads();
  for (uint32_t i = tid; i < nw; i += 256) {
    const uint32_t key = s.ukey[SCAN_CHUNK + i], pos = s.cpos[i];
    if (slot_excluded(flt, off, pos, key)) continue;
    atomicAdd(&s_kept, 1u);
    atomicMax(&s_max, key);
    if (key == 0xffffffffu) atomicMax(&s_last, pos + 1);  // 1 + the last admitted position at the maximal key
  }
  __syncthreads();
  const uint32_t mx = s_max, last = s_last;
  for (uint32_t i = tid; i < nw; i += 256) {
    const uint32_t key = s.ukey[SCAN_CHUNK + i], pos = s.cpos[i];
    if (slot_excluded(flt, off, pos, key)) {
      if (pos + 1 < last) atomicAdd(&s_mid, 1u);  // excluded, but in front of an admitted winner
    } else if (key == mx) {
      atomicAdd(&s_maxcnt, 1u);
    }
  }
  __syncthreads();
  const uint32_t kept = s_kept, mid = s_mid;
  const bool at_k = kept + mid == kk;
  if (at_k && s_maxcnt + mid >= 2) return false;  // block-uniform
  if (nw == kk && !at_k && max_admitted) return false;
  for (uint32_t i = tid; i < nw; i += 256) {
    const uint32_t key = s.ukey[SCAN_CHUNK + i], pos = s.cpos[i];
    if (slot_excluded(flt, off, pos, key) || (at_k && key == mx)) continue;  // at_k: the (k+1)-th is the unique max
    const uint32_t at = atomicAdd(&s_out, 1u);
    s.nkey[at] = key;
    s.npos[at] = pos;
  }
  __syncthreads();
  *cnt = s_out;
  return true;
}

// The reference's own loop (flat/index.rs:116-165): rows in storage order, keys filled one chunk ahead of the single
// thread that drives the heap.  Leaves the heap's content at nkey / npos and returns its size.
template <class Fill>
__device__ __forceinline__ uint32_t slot_replay(const SlotSmem& s, uint32_t n, uint32_t k, const ScanFilter& flt, uint64_t off,
                                Fill fill) {
  __shared__ uint32_t s_len;
  const bool filtering = flt.allow != nullptr || flt.range;
  uint32_t len = 0;
  for (uint32_t c0 = 0; c0 < n; c0 += SCAN_CHUNK) {
    const uint32_t clen = min((uint32_t)SCAN_CHUNK, n - c0);
    fill(c0, clen);
    __syncthreads();
    if (threadIdx.x == 0) {
      for (uint32_t j = 0; j < clen; ++j) {
        const uint32_t key = s.ukey[j];
        if (filtering && slot_excluded(flt, off, c0 + j, key)) continue;
        rheap_offer(s.nkey, s.npos, len, k, key, c0 + j);
      }
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) s_len = len;
  __syncthreads();
  return s_len;
}

// The exact top-k of a slot of n rows: <= k winners at nkey / npos (unordered); returns their number.  replay: go
// straight to the heap loop.
template <class Fill>
__device__ __forceinline__ uint32_t slot_topk(const SlotSmem& s, uint32_t n, int k, const ScanFilter& flt, uint64_t off, bool replay,
                              Fill fill) {
  if (!replay) {
    uint32_t cnt;
    bool max_admitted;
    const uint32_t nw = slot_select(s, n, k + 1, flt, off, fill, max_admitted);
    if (slot_finish(s, nw, k + 1, max_admitted, flt, off, &cnt)) return cnt;
    __syncthreads();
  }
  return slot_replay(s, n, k, flt, off, fill);
}

// a slot's winners -> its candidate list (unordered)
__device__ __forceinline__ void write_slot(const SlotSmem& s, uint32_t cnt, size_t slot, int k, uint64_t off,
                                           const uint64_t* __restrict__ row_ids, float* __restrict__ cand_d,
                                           uint64_t* __restrict__ cand_id, uint32_t* __restrict__ cand_cnt) {
  for (uint32_t i = threadIdx.x; i < cnt; i += 256) {
    cand_d[slot * k + i] = key_to_float((int32_t)(s.nkey[i] ^ 0x80000000u));
    cand_id[slot * k + i] = row_ids[off + s.npos[i]];
  }
  if (threadIdx.x == 0) cand_cnt[slot] = cnt;
}

template <int METRIC, int NBITS>
__device__ void radix_slot(const ScanArgs& a, size_t slot, bool replay) {
  extern __shared__ float smem[];
  const int M = a.M, d = a.d, k = a.k, np = a.np;
  float* lut = smem;                         // [M*16] (4-bit) or [M*256] (8-bit)
  float* qr = lut + M * (NBITS == 4 ? 16 : 256);  // [d]
  const SlotSmem s(qr + d, k + 1);
  const int tid = threadIdx.x;
  const int pi = (int)(slot % np);
  const size_t qi = slot / np;
  const uint32_t p = a.probe_ids[qi * np + pi];
  const uint64_t off = a.part_offsets[p];
  const uint32_t n_p = (uint32_t)(a.part_offsets[p + 1] - off);
  if (n_p == 0) {
    if (tid == 0) a.cand_cnt[slot] = 0;
    return;
  }
  stage_query_lut<METRIC, NBITS>(lut, qr, a, qi, p);
  const int cw = NBITS == 4 ? M / 2 : M;  // code bytes per row
  const uint8_t* pc = a.codes + off * cw;
  const float dot_fix = (float)M - 1.0f;
  // ---- 4-bit (pq/distance.rs:147-242): rows [0, flat_num) and the last n_p % 16 rows are exact f32 sums;
  // the others go through the table quantised to u8.  With a prefilter the reference scores row by row with
  // DistCalculator::distance (exact, pq/storage.rs:895-916), so every row is exact then.
  __shared__ uint8_t qt[NBITS == 4 ? 256 * 16 : 1];  // M <= 256 sub-vectors x 16 entries
  __shared__ float s_q[2];                                // qmin, (qmax - qmin) / 255
  const uint32_t flat_num = NBITS == 4 ? min((uint32_t)max(200, k), n_p) : 0;
  const uint32_t rem16 = NBITS == 4 ? n_p % 16 : 0;
  auto exact4 = [&](uint32_t j) -> float {  // two adds per byte, byte order
    const uint8_t* rp = pc + (size_t)j * cw;
    float dist = 0.0f;
    for (int i = 0; i < cw; ++i) {
      const uint8_t c = rp[i];
      dist = f_add(dist, lut[(2 * i) * 16 + (c & 0xF)]);
      dist = f_add(dist, lut[(2 * i + 1) * 16 + (c >> 4)]);
    }
    return dist;
  };
  if (NBITS == 4 && a.flt.allow == nullptr)  // the selection's (still unused) key buffer is the scratch
    pq4_quantize(lut, M, flat_num, exact4, qt, s_q, reinterpret_cast<int32_t*>(s.ukey),
                 reinterpret_cast<float*>(s.ukey + 256));
  auto fill = [&](uint32_t c0, uint32_t clen) {
    for (uint32_t j = tid; j < clen; j += 256) {
      const uint32_t row = c0 + j;
      float dist;
      if constexpr (NBITS == 4) {
        if (a.flt.allow != nullptr || row < flat_num || row >= n_p - rem16) {
          dist = exact4(row);
        } else {
          const uint8_t* rp = pc + (size_t)row * cw;
          uint32_t qs = 0;  // saturating u8 adds of non-negative terms == min(255, sum)
          for (int i2 = 0; i2 < cw; ++i2) {
            const uint8_t c = rp[i2];
            qs += qt[(2 * i2) * 16 + (c & 0xF)];
            qs += qt[(2 * i2 + 1) * 16 + (c >> 4)];
          }
          dist = pq4_dequantize(min(qs, 255u), s_q);
        }
      } else {
        dist = pq8_row_distance(lut, pc + (size_t)row * M, M);
      }
      // pq/storage.rs:957-958; a NaN passes through, as on x86 (the device's own NaN would stay canonical anyway)
      if (METRIC == METRIC_DOT && dist == dist) dist = __fsub_rn(dist, dot_fix);
      s.ukey[j] = (uint32_t)total_order_key(dist) ^ 0x80000000u;
    }
  };
  const uint32_t cnt = slot_topk(s, n_p, k, a.flt, off, replay, fill);
  write_slot(s, cnt, slot, k, off, a.row_ids, a.cand_d, a.cand_id, a.cand_cnt);
}

// grid (np, nq): one CTA per slot; or, with a replay list (slots the fast kernel could not settle because of
// ties at the k-th distance), a small persistent grid that replays the listed slots
template <int METRIC, int NBITS>
__global__ void __launch_bounds__(256)
ivfpq_scan_radix_kernel(const ScanArgs a, const uint32_t* __restrict__ rlist, const uint32_t* __restrict__ rcount) {
  if (rlist) {
    const uint32_t cnt = *rcount;
    for (uint32_t i = blockIdx.x; i < cnt; i += gridDim.x) {
      radix_slot<METRIC, NBITS>(a, rlist[i], true);
      __syncthreads();
    }
    return;
  }
  radix_slot<METRIC, NBITS>(a, (size_t)blockIdx.y * a.np + blockIdx.x, false);
}

// ---- warp-wide sorting network on packed (key, position) words -------------------------------------
// A candidate is one u64: (order-preserving u32 of the distance) << 32 | position inside the partition,
// so an unsigned compare IS the (distance, position) order every selection step needs ("ties keep the
// earlier row").  PACK_INF (no candidate) sorts last.
constexpr uint64_t PACK_INF = ~0ull;
__device__ __forceinline__ uint64_t pack_cand(int32_t key, uint32_t pos) {
  return ((uint64_t)((uint32_t)key ^ 0x80000000u) << 32) | pos;
}
__device__ __forceinline__ int32_t cand_key(uint64_t c) { return (int32_t)((uint32_t)(c >> 32) ^ 0x80000000u); }
__device__ __forceinline__ uint32_t cand_pos(uint64_t c) { return (uint32_t)c; }

// End of a fast 8-bit slot, threads t = 0 .. nt - 1: win[0..nw) ascending by (key, position), nw <= k + 1.  If the
// k-th and the (k+1)-th share a key, more rows tie at the k-th distance than fit: which of them the reference's
// BinaryHeap keeps depends on its sift order, so the slot goes on the replay list (ivfpq_scan_radix_kernel in list
// mode restates that loop); so does a slot the kernel could not settle (replay).  Otherwise the first min(nw, k).
__device__ __forceinline__ void fast_slot_epilogue(const ScanArgs& a, uint32_t slot, uint64_t off, const uint64_t* win,
                                                   uint32_t nw, bool replay, int t, int nt, uint32_t* rlist,
                                                   uint32_t* rcount) {
  const int k = a.k;
  if (!replay && nw == (uint32_t)k + 1) {
    replay = cand_key(win[k]) == cand_key(win[k - 1]);
    nw = k;
  }
  if (replay) {
    if (t == 0) {
      rlist[atomicAdd(rcount, 1u)] = slot;
      a.cand_cnt[slot] = 0;
    }
    return;
  }
  for (uint32_t i = t; i < nw; i += nt) {
    a.cand_d[(size_t)slot * k + i] = key_to_float(cand_key(win[i]));
    a.cand_id[(size_t)slot * k + i] = a.row_ids[off + cand_pos(win[i])];
  }
  if (t == 0) a.cand_cnt[slot] = nw;
}

// bitonic merge of a 32-lane bitonic sequence into ascending order (5 compare-exchange steps)
__device__ __forceinline__ uint64_t warp_bitonic_merge32(uint64_t v, int lane) {
#pragma unroll
  for (int j = 16; j >= 1; j >>= 1) {
    const uint64_t o = __shfl_xor_sync(0xffffffffu, v, j);
    const bool keep_min = (lane & j) == 0;
    v = (keep_min == (o < v)) ? o : v;
  }
  return v;
}
// full ascending sort of one value per lane (15 compare-exchange steps)
__device__ __forceinline__ uint64_t warp_sort32(uint64_t v, int lane) {
#pragma unroll
  for (int k2 = 2; k2 <= 32; k2 <<= 1) {
#pragma unroll
    for (int j = k2 >> 1; j >= 1; j >>= 1) {
      const uint64_t o = __shfl_xor_sync(0xffffffffu, v, j);
      const bool keep_min = ((lane & j) == 0) == ((lane & k2) == 0);
      v = (keep_min == (o < v)) ? o : v;
    }
  }
  return v;
}
// the 32 smallest of a shared-memory list, ascending, one per lane (lane r = r-th smallest)
__device__ __forceinline__ uint64_t warp_smallest32(const uint64_t* list, uint32_t cnt, int lane) {
  uint64_t best = warp_sort32(lane < (int)cnt ? list[lane] : PACK_INF, lane);
  for (uint32_t base = 32; base < cnt; base += 32) {
    uint64_t v = warp_sort32(base + lane < cnt ? list[base + lane] : PACK_INF, lane);
    v = __shfl_sync(0xffffffffu, v, 31 - lane);  // descending: min(best, v) is bitonic
    best = warp_bitonic_merge32(v < best ? v : best, lane);
  }
  return best;
}

// k <= 16.  Per chunk of 4096 rows every WARP works on its own 512 rows without block barriers:
//   Tw = k-th smallest of its 32 lane minima (one 32-lane sort; an upper bound of the warp's k-th
//   smallest element), the <= (k-1)*16+1 elements <= Tw are compacted into the warp's shared-memory
//   list and sorted 32 at a time; then warp 0 merges the 8 x k warp winners with the winners carried
//   from earlier chunks the same way.  All comparisons are on packed (key, position) words.
constexpr int SCAN_KFAST = 16;
constexpr int SCAN_WLIST = (SCAN_KFAST - 1) * 16 + 1;  // 241

template <int METRIC, bool FILTER>
__global__ void __launch_bounds__(256, 6)
ivfpq_scan_kernel(const ScanArgs a, uint32_t* __restrict__ rlist, uint32_t* __restrict__ rcount) {
  constexpr int RPT = SCAN_CHUNK / 256;  // rows per thread and chunk (16)
  extern __shared__ float smem[];
  const int M = a.M, k = a.k, np = a.np;
  const int kk = k + 1;  // <= SCAN_KFAST: one more than asked for, to expose ties that overflow the k-th place
  const uint64_t* __restrict__ allow = a.flt.allow;
  float* lut = smem;          // [M*256]
  float* qr = lut + M * 256;  // [d]
  __shared__ uint64_t wl[8][SCAN_WLIST];                 // per-warp compacted candidates
  __shared__ uint64_t fin[8 * SCAN_KFAST + SCAN_KFAST];  // 8 x kk warp winners, then the carried winners
  __shared__ uint64_t car[SCAN_KFAST];
  __shared__ uint32_t s_nw;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int pi = blockIdx.x;
  const size_t qi = blockIdx.y;
  const uint32_t p = a.probe_ids[qi * np + pi];
  const uint64_t off = a.part_offsets[p];
  const uint32_t n_p = (uint32_t)(a.part_offsets[p + 1] - off);
  const size_t slot = qi * np + pi;
  if (n_p == 0) {
    if (tid == 0) a.cand_cnt[slot] = 0;
    return;
  }
  if (tid == 0) s_nw = 0;
  stage_query_lut<METRIC, 8>(lut, qr, a, qi, p);

  const uint8_t* pc = a.codes + off * M;
  const float dot_fix = (float)M - 1.0f;
  for (uint32_t c0 = 0; c0 < n_p; c0 += SCAN_CHUNK) {
    const uint32_t clen = min((uint32_t)SCAN_CHUNK, n_p - c0);
    int32_t key[RPT];
    uint64_t mine = PACK_INF;  // this lane's smallest candidate
    uint32_t livemask = 0;     // FILTER: bit u = row u of this thread passed the prefilter and the range
    // rows of warp w in this chunk: c0 + w*512 + lane + 32*u  (a warp owns a contiguous 512-row slab)
    const uint32_t wbase = warp * (RPT * 32);
#pragma unroll
    for (int u = 0; u < RPT; ++u) {
      const uint32_t j = wbase + lane + 32 * u;
      key[u] = 0x7fffffff;
      if (j < clen && (!FILTER || row_allowed(allow, off + c0 + j))) {
        float dist = pq8_row_distance(lut, pc + (size_t)(c0 + j) * M, M);
        if (METRIC == METRIC_DOT) dist = __fsub_rn(dist, dot_fix);  // pq/storage.rs:957-958
        const int32_t kv = total_order_key(dist);
        if (!FILTER || key_in_range(a.flt, kv)) {
          if (FILTER) livemask |= 1u << u;
          key[u] = kv;
          const uint64_t c = pack_cand(kv, c0 + j);
          mine = c < mine ? c : mine;
        }
      }
    }
    // ---- warp-local threshold: Tw = kk-th smallest lane minimum (PACK_INF if < kk lanes have rows)
    const uint64_t tw = __shfl_sync(0xffffffffu, warp_sort32(mine, lane), kk - 1);
    // ---- compact the warp's elements <= Tw (ballot-ranked: deterministic order, no atomics)
    uint32_t wcnt = 0;
#pragma unroll
    for (int u = 0; u < RPT; ++u) {
      const uint32_t j = wbase + lane + 32 * u;
      const bool live = FILTER ? ((livemask >> u) & 1u) != 0 : j < clen;
      const uint64_t c = pack_cand(key[u], c0 + j);
      const bool take = live && c <= tw;
      const unsigned bal = __ballot_sync(0xffffffffu, take);
      if (take) wl[warp][wcnt + __popc(bal & ((1u << lane) - 1))] = c;
      wcnt += __popc(bal);
    }
    __syncwarp();
    // ---- the warp's kk smallest -> block list (lane r holds the r-th smallest; PACK_INF = none)
    {
      const uint64_t best = warp_smallest32(wl[warp], wcnt, lane);
      if (lane < kk) fin[warp * SCAN_KFAST + lane] = best;
    }
    __syncthreads();
    if (warp == 0) {  // merge: 8 x kk warp winners + carried winners -> kk block winners
      const uint32_t nw = s_nw;
      if (lane < kk) fin[8 * SCAN_KFAST + lane] = lane < (int)nw ? car[lane] : PACK_INF;
      __syncwarp();
      // the winners sit at fin[w * 16 + r], r < kk: visit them 32 at a time (2 warps' slots per pass)
      uint64_t best = PACK_INF;
      for (int base = 0; base < 9 * SCAN_KFAST; base += 32) {
        const int i = base + lane;
        uint64_t v = (i < 9 * SCAN_KFAST && (i % SCAN_KFAST) < kk) ? fin[i] : PACK_INF;
        v = warp_sort32(v, lane);
        if (base == 0) {
          best = v;
        } else {
          v = __shfl_sync(0xffffffffu, v, 31 - lane);
          best = warp_bitonic_merge32(v < best ? v : best, lane);
        }
      }
      if (lane < kk) car[lane] = best;
      const unsigned got = __ballot_sync(0xffffffffu, lane < kk && best != PACK_INF);
      if (lane == 0) s_nw = __popc(got);
    }
    __syncthreads();
  }
  fast_slot_epilogue(a, (uint32_t)slot, off, car, s_nw, false, tid, 256, rlist, rcount);
}

// ------------------------------------------------------------------------------------------------
// Conflict-free scan for the headline shape (8-bit codes, M = 16 sub-spaces of 8 dimensions; C1 / C3).
//
// What bounds the scan above is the shared-memory gather: 32 lanes look up LUT[m][code] for the SAME m and random
// codes, i.e. random banks -- 3.3 wavefronts per request (ncu: 454 M bank conflicts per 10 000 x 10 probes) -- and
// every (query, partition) CTA re-reads the 128 KB codebook through L2.  This kernel removes both:
//
//  * the LUT is stored as [code][team][copy][m] (two copies per team, 256 B per code for the CTA's two teams):
//    sub-space m lives in bank m (copy 0) and 16 + m (copy 1).  Lane l works on sub-space (t - l) mod 16 at step t, lanes 0-15 on copy 0 and lanes 16-31 on copy 1,
//    so the 32 lookups of a request always hit 32 different banks: ONE wavefront.
//  * the reference's sum is m-ascending and sequential in f32, so a lane cannot start its row at m != 0.  Instead
//    the lanes are SKEWED IN TIME: lane l starts each row l steps late.  The index keeps, next to the row-major
//    codes, a skewed copy (`build_skew_codes`): per 512-row slab and lane the 16 rows of that lane (rows l + 32 i)
//    form one byte stream that is preceded by l mod 16 pad bytes and cut into 17 units of 16 bytes, unit (r, lane)
//    at (r * 32 + lane) * 16 -- one coalesced 128-bit load per lane and round, and byte t of a unit is a
//    compile-time register/byte position.  Two accumulators take the steps before / after the lane's row boundary,
//    selected by per-lane 0/1 weights through FFMA: fma(v, 1, acc) is the reference's separately rounded add,
//    fma(v, 0, acc) leaves acc unchanged (all LUT entries finite, checked while the LUT is built; a slot whose
//    LUT is not goes to the replay list).  Per lookup: one PRMT (code byte -> address bits 8-15, the lane's
//    bank bits into the low byte), LDS, 2 FFMA.
//  * persistent CTAs (one per SM, two teams of 8 warps) keep the codebook in shared memory (padded so that the
//    16 sub-spaces a half-warp reads are in different banks) and build each slot's LUT from there; thread (m, c)
//    keeps its residual sub-vector in registers.  Team barriers are named barriers, so one team scans while the
//    other builds its LUT.
// Distances, candidate order and the tie / replay rule are those of ivfpq_scan_kernel (same bits).
// ------------------------------------------------------------------------------------------------
constexpr int SKEW_ROUNDS = 17;                          // 16 rows per lane and slab + one unit of skew
constexpr int SKEW_SLAB_ROWS = 512;
constexpr int SKEW_SLAB_BYTES = SKEW_ROUNDS * 32 * 16;   // 8704
constexpr int SKEW_CB_STRIDE = 256 * 8 + 4;              // floats per sub-space in shared memory (+16 B pad)
constexpr int SKEW_LUT_BYTES = 256 * 256;                // both teams' LUTs, interleaved per code
constexpr int SKEW_LIST = 1024;                          // capacity of a team's candidate list (two teams)
constexpr int SKEW_SMALL_BYTES = 2 * SCAN_KFAST * 8 + 8 * 32 * 4 + 8 * 4 + 16;   // per team (sized for 8 warps): winners, lane minima, ...
// the LUT at shared address 0x10000: [base, 0x10000) holds 7 codebook sub-spaces + the small scratch, above the LUT
// come 9 sub-spaces and the two candidate lists; the dynamic allocation covers the highest address for base = 0
constexpr uint32_t SKEW_MAX_BASE = 0x10000u - (7 * SKEW_CB_STRIDE * 4 + 4 * SKEW_SMALL_BYTES);
constexpr int SKEW_SMEM_BYTES = 0x10000 + SKEW_LUT_BYTES + 112 + 9 * SKEW_CB_STRIDE * 4 + 2 * SKEW_LIST * 8;

__device__ __forceinline__ float lds_f32(uint32_t saddr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(saddr));
  return v;
}
template <int NT>
__device__ __forceinline__ void team_sync(int team) {
  asm volatile("bar.sync %0, %1;" ::"r"(team + 1), "n"(NT) : "memory");
}
template <int NT>
__device__ __forceinline__ bool team_or(int team, bool v) {
  uint32_t r;
  asm volatile(
      "{\n\t.reg .pred p, q;\n\tsetp.ne.u32 q, %2, 0;\n\tbar.red.or.pred p, %1, %3, q;\n\tselp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(r)
      : "r"(team + 1), "r"((uint32_t)v), "n"(NT)
      : "memory");
  return r != 0;
}

// slab_off[p] = number of 512-row slabs before partition p (exclusive scan of ceil(n_p / 512)); slab_off[K] = total
__global__ void __launch_bounds__(1024)
skew_offsets_kernel(const uint64_t* __restrict__ part_offsets, int K, uint64_t* __restrict__ slab_off) {
  __shared__ uint64_t part[1024];
  const int tid = threadIdx.x;
  const int per = (K + 1023) / 1024;
  const int b = tid * per, e = min(K, b + per);
  uint64_t s = 0;
  for (int p = b; p < e; ++p) s += (part_offsets[p + 1] - part_offsets[p] + SKEW_SLAB_ROWS - 1) / SKEW_SLAB_ROWS;
  part[tid] = s;
  __syncthreads();
  for (int o = 1; o < 1024; o <<= 1) {
    const uint64_t v = tid >= o ? part[tid - o] : 0;
    __syncthreads();
    part[tid] += v;
    __syncthreads();
  }
  uint64_t run = tid ? part[tid - 1] : 0;
  for (int p = b; p < e; ++p) {
    slab_off[p] = run;
    run += (part_offsets[p + 1] - part_offsets[p] + SKEW_SLAB_ROWS - 1) / SKEW_SLAB_ROWS;
  }
  if (tid == 1023) slab_off[K] = part[1023];
}

// one warp per slab: unit (r, lane) = bytes [16 r - l16, 16 r - l16 + 16) of the lane's row stream (rows lane + 32 i)
__global__ void __launch_bounds__(256)
skew_fill_kernel(const uint64_t* __restrict__ part_offsets, int K, const uint64_t* __restrict__ slab_off,
                 const uint8_t* __restrict__ codes, uint8_t* __restrict__ skew) {
  const uint64_t nslab = slab_off[K];
  const int lane = threadIdx.x & 31, l16 = lane & 15;
  for (uint64_t s = (uint64_t)blockIdx.x * 8 + (threadIdx.x >> 5); s < nslab; s += (uint64_t)gridDim.x * 8) {
    int lo = 0, hi = K;  // last p with slab_off[p] <= s  (empty partitions share their successor's offset)
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (slab_off[mid] <= s) lo = mid; else hi = mid;
    }
    const int p = lo;
    const uint64_t off = part_offsets[p];
    const uint32_t n_p = (uint32_t)(part_offsets[p + 1] - off);
    const uint32_t base = (uint32_t)(s - slab_off[p]) * SKEW_SLAB_ROWS;
    const uint4* rows = reinterpret_cast<const uint4*>(codes) + off;
    uint4* out = reinterpret_cast<uint4*>(skew + s * SKEW_SLAB_BYTES) + lane;
    uint4 prev = make_uint4(0, 0, 0, 0);
    for (int r = 0; r < SKEW_ROUNDS; ++r) {
      const uint32_t j = base + lane + 32 * r;
      const uint4 cur = (r < 16 && j < n_p) ? __ldg(rows + j) : make_uint4(0, 0, 0, 0);
      uint4 u = cur;
      if (l16) {  // bytes [16 - l16, 32 - l16) of prev|cur
        const uint32_t w[8] = {prev.x, prev.y, prev.z, prev.w, cur.x, cur.y, cur.z, cur.w};
        const int b0 = 16 - l16, wq = b0 >> 2, sh = (b0 & 3) * 8;
        uint32_t o[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          uint32_t lo32 = 0, hi32 = 0;
#pragma unroll
          for (int q = 0; q < 8; ++q) {  // static indexing of w[]
            if (q == wq + i) lo32 = w[q];
            if (q == wq + i + 1) hi32 = w[q];
          }
          o[i] = sh ? (lo32 >> sh) | (hi32 << (32 - sh)) : lo32;
        }
        u = make_uint4(o[0], o[1], o[2], o[3]);
      }
      out[r * 32] = u;
      prev = cur;
    }
  }
}

template <int METRIC, bool FILTER, int NTEAM>
__global__ void __launch_bounds__(512, 1)
ivfpq_scan_skew_kernel(const ScanArgs a, const uint64_t* __restrict__ slab_off, const uint8_t* __restrict__ skew,
                       uint32_t nslots, uint32_t* __restrict__ rlist, uint32_t* __restrict__ rcount) {
  extern __shared__ __align__(16) unsigned char sk_smem[];
  const int d = a.d, k = a.k, np = a.np;
  const int kk = k + 1;  // one more than asked for, to expose ties that overflow the k-th place
  const uint64_t* __restrict__ allow = a.flt.allow;
  // NTEAM = 2: teams of 8 warps, two LUT copies (no bank conflicts).  NTEAM = 4: teams of 4 warps, ONE copy each
  // (lanes l and l + 16 share a bank: two wavefronts per request) -- twice as many independent teams to fill the
  // issue slots a team leaves empty at its barriers and in its low-parallelism phases.
  constexpr int TT = 512 / NTEAM, TW = TT / 32, COPIES = NTEAM == 2 ? 2 : 1;
  constexpr int LIST = SKEW_LIST * 2 / NTEAM;          // candidate-list capacity per team
  constexpr uint32_t CHUNK = TW * SKEW_SLAB_ROWS;       // rows a team scans between two selections
  const int tid = threadIdx.x, team = tid / TT, ttid = tid % TT, lane = tid & 31, warp = ttid >> 5;
  const int l16 = lane & 15, half = lane >> 4;
  // Shared-memory map.  The LUT sits at SHARED ADDRESS 0x10000 exactly, so that a lookup address is
  // 0x10000 | code << 8 | bank bits -- all of it produced by the one byte permute.  The codebook is split around
  // it (sub-spaces 0-6 below, 7-15 above), the small per-team scratch goes below, the candidate lists above.
  const uint32_t sbase = (uint32_t)__cvta_generic_to_shared(sk_smem);
  if (sbase > SKEW_MAX_BASE) {  // never seen (the runtime reserves 1 KB: sbase = 0x400); the exact replay takes every slot
    for (uint32_t slot = blockIdx.x * 512 + tid; slot < nslots; slot += gridDim.x * 512) {
      rlist[atomicAdd(rcount, 1u)] = slot;
      a.cand_cnt[slot] = 0;
    }
    return;
  }
  unsigned char* lut_g = sk_smem + (0x10000u - sbase);                             // generic pointer to the LUT
  float* lut2 = reinterpret_cast<float*>(lut_g) + team * (16 * COPIES);            // [256 codes][64]: + copy * 16 + m
  float* cb_lo = reinterpret_cast<float*>(sk_smem);                                // sub-spaces 0..6
  // sub-spaces 7..15; the 112 bytes keep sub-space m in 16-byte bank group (m + 2 c + h) mod 8 on both sides of the LUT
  float* cb_hi = reinterpret_cast<float*>(lut_g + SKEW_LUT_BYTES + 112);
  unsigned char* tb = sk_smem + 7 * SKEW_CB_STRIDE * 4 + team * SKEW_SMALL_BYTES;  // small scratch (below the LUT)
  uint64_t* car = reinterpret_cast<uint64_t*>(tb);                                 // [2][SCAN_KFAST] winners so far
  int32_t* wmin = reinterpret_cast<int32_t*>(car + 2 * SCAN_KFAST);               // [TW][32] lane minima
  int32_t* s_tw = wmin + TW * 32;                                                  // [8] warp thresholds
  uint32_t* s_cnt = reinterpret_cast<uint32_t*>(s_tw + 8);                         // candidates in tl
  uint64_t* tl = reinterpret_cast<uint64_t*>(lut_g + SKEW_LUT_BYTES + 112 + 9 * SKEW_CB_STRIDE * 4) + team * LIST;

  // codebook -> shared memory, once per CTA (sub-space stride padded by 16 B)
  for (int i = tid; i < 16 * 256 * 2; i += 512) {
    const int e = i >> 1, m = e >> 8;
    const float4 v = __ldg(reinterpret_cast<const float4*>(a.codebook) + i);
    float* dstm = m < 7 ? cb_lo + m * SKEW_CB_STRIDE : cb_hi + (m - 7) * SKEW_CB_STRIDE;
    *reinterpret_cast<float4*>(dstm + (e & 255) * 8 + (i & 1) * 4) = v;
  }
  __syncthreads();

  // per-lane constants of the skewed schedule
  const int th = l16 ? l16 : 16;  // steps [0, th) of a round still belong to the row begun one round earlier
  float wA[16], wB[16];
  uint32_t lp[16];  // low address byte of LUT[.][team][this lane's copy][sub-space of step t]
#pragma unroll
  for (int t = 0; t < 16; ++t) {
    wA[t] = t < th ? 1.0f : 0.0f;
    wB[t] = t < th ? 0.0f : 1.0f;
    lp[t] = 0x10000u | (uint32_t)((team * (16 * COPIES) + (COPIES == 2 ? half * 16 : 0) + ((t - l16) & 15)) << 2);
  }
  const int sh = l16 != 0;  // the row finished in round u is row u - sh of the lane
  const int lm = ttid & 15;                  // LUT build: this thread's sub-space
  const float* cbm = lm < 7 ? cb_lo + lm * SKEW_CB_STRIDE : cb_hi + (lm - 7) * SKEW_CB_STRIDE;
  const float dot_fix = 16.0f - 1.0f;
  constexpr int32_t MAXKEY = 0x7fffffff;     // no live row carries it: the LUT is finite, sums are at most +inf
  int par = 0;                               // which half of car[] holds the winners

  // slot metadata is a chain of dependent global loads (probe id -> partition offsets -> slab offset): it is
  // fetched one slot ahead, and the first code unit of a slot is requested before its LUT is built
  const uint32_t stride = gridDim.x * NTEAM;
  uint32_t slot = blockIdx.x * NTEAM + team;
  uint32_t p_n = slot < nslots ? a.probe_ids[slot] : 0u;
  uint64_t off_n = a.part_offsets[p_n], end_n = a.part_offsets[p_n + 1], so_n = slab_off[p_n];
  for (; slot < nslots; slot += stride) {
    const size_t qi = slot / np;
    const uint32_t p = p_n;
    const uint64_t off = off_n;
    const uint32_t n_p = (uint32_t)(end_n - off_n);
    const uint8_t* sp = skew + so_n * SKEW_SLAB_BYTES;
    p_n = slot + stride < nslots ? a.probe_ids[slot + stride] : 0u;
    if (n_p == 0) {
      off_n = a.part_offsets[p_n]; end_n = a.part_offsets[p_n + 1]; so_n = slab_off[p_n];
      if (ttid == 0) a.cand_cnt[slot] = 0;
      continue;
    }
    const uint4* up0 = reinterpret_cast<const uint4*>(sp + (size_t)warp * SKEW_SLAB_BYTES) + lane;
    uint4 first_unit = make_uint4(0, 0, 0, 0);
    if ((uint32_t)warp * SKEW_SLAB_ROWS < n_p) first_unit = __ldg(up0);
    // ---- residual query of this thread's sub-space (v2.rs:316-332) and the LUT (pq/distance.rs:38-56).
    // No barrier is needed before lut2 is overwritten: every warp of the team left its scan before the last
    // team barrier of the previous slot.
    float qm[8];
    {
      const float4* q4 = reinterpret_cast<const float4*>(a.queries + qi * d + lm * 8);
      const float4* c4 = reinterpret_cast<const float4*>(a.centroids + (size_t)p * d + lm * 8);
      const float4 x0 = __ldg(q4), x1 = __ldg(q4 + 1);
      qm[0] = x0.x; qm[1] = x0.y; qm[2] = x0.z; qm[3] = x0.w; qm[4] = x1.x; qm[5] = x1.y; qm[6] = x1.z; qm[7] = x1.w;
      if (METRIC != METRIC_DOT) {
        const float4 y0 = __ldg(c4), y1 = __ldg(c4 + 1);
        const float cv[8] = {y0.x, y0.y, y0.z, y0.w, y1.x, y1.y, y1.z, y1.w};
#pragma unroll
        for (int t = 0; t < 8; ++t) qm[t] = __fsub_rn(qm[t], cv[t]);
      }
    }
    bool bad = false;
#pragma unroll 4
    for (int i = 0; i < 256 / (TT / 16); ++i) {
      const int c = (ttid >> 4) + (TT / 16) * i;
      const float4 b0 = *reinterpret_cast<const float4*>(cbm + c * 8);
      const float4 b1 = *reinterpret_cast<const float4*>(cbm + c * 8 + 4);
      const float cv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
      float s = 0.0f;
#pragma unroll
      for (int t = 0; t < 8; ++t) s = f_add(s, term<METRIC>(qm[t], cv[t]));
      const float val = finish<METRIC>(f_add(s, 0.0f));
      bad |= !(fabsf(val) < 1.0e30f);
      if (COPIES == 2) {
        lut2[c * 64 + half * 16 + lm] = val;
        lut2[c * 64 + (half ^ 1) * 16 + lm] = val;
      } else {
        lut2[c * 64 + lm] = val;
      }
    }
    off_n = a.part_offsets[p_n]; end_n = a.part_offsets[p_n + 1]; so_n = slab_off[p_n];
    bool replay = team_or<TT>(team, bad);
    uint32_t nw = 0;  // winners carried from earlier chunks (uniform)
    for (uint32_t c0 = 0; c0 < n_p && !replay; c0 += CHUNK) {
      const uint32_t clen = min(CHUNK, n_p - c0);
      const uint32_t wbase = warp * SKEW_SLAB_ROWS;
      if (ttid == 0) *s_cnt = 0;  // read last before the previous chunk's / slot's final barrier
      int32_t key[SKEW_ROUNDS];
      int32_t mk = MAXKEY;  // this lane's smallest live key
      if (wbase < clen) {   // warp-uniform: this warp's slab exists
        // rows of this lane: wbase + lane + 32 i < clen, i < 16; they finish in rounds sh .. sh + cnt - 1
        uint32_t livemask = 0;
        if (!FILTER) {
          const uint32_t first = wbase + lane;
          const uint32_t cnt = first < clen ? min(16u, (clen - first + 31u) >> 5) : 0u;
          livemask = ((1u << cnt) - 1u) << sh;
        }
        const uint4* up = reinterpret_cast<const uint4*>(sp + (size_t)((c0 >> 9) + warp) * SKEW_SLAB_BYTES) + lane;
        float A = 0.0f, B = 0.0f;
        uint4 cur = c0 == 0 ? first_unit : __ldg(up);
#pragma unroll
        for (int r = 0; r < SKEW_ROUNDS; ++r) {
          uint4 nxt = cur;
          if (r + 1 < SKEW_ROUNDS) nxt = __ldg(up + (r + 1) * 32);
          const uint32_t w[4] = {cur.x, cur.y, cur.z, cur.w};
#pragma unroll
          for (int t = 0; t < 16; ++t) {
            // shared address = 0x10000 | code << 8 | bank bits: one byte permute (bytes 0, 2, 3 <- lp, byte 1 <- code)
            const float v = lds_f32(__byte_perm(w[t >> 2], lp[t], 0x7604u | ((uint32_t)(t & 3) << 4)));
            A = __fmaf_rn(v, wA[t], A);
            B = __fmaf_rn(v, wB[t], B);
          }
          float dist = A;
          A = B;
          B = 0.0f;
          if (METRIC == METRIC_DOT) dist = __fsub_rn(dist, dot_fix);  // pq/storage.rs:957-958
          const int32_t kv = total_order_key(dist);
          bool live;
          if (FILTER) {
            const int ri = r - sh;
            const uint32_t j = wbase + lane + 32 * ri;
            live = ri >= 0 && ri < 16 && j < clen && row_allowed(allow, off + c0 + j) && key_in_range(a.flt, kv);
          } else {
            live = ((livemask >> r) & 1u) != 0;
          }
          key[r] = live ? kv : MAXKEY;
          mk = min(mk, key[r]);
          cur = nxt;
        }
      } else {
#pragma unroll
        for (int r = 0; r < SKEW_ROUNDS; ++r) key[r] = MAXKEY;
      }
      // ---- selection.  With two teams per SM nothing hides the dependent shuffle steps of sorting networks, and
      // instruction issue is what bounds the kernel, so: (1) per warp, Tw = kk-th smallest lane minimum = the
      // largest lane minimum with fewer than kk smaller ones (32 broadcast reads + one warp reduction);
      wmin[warp * 32 + lane] = mk;
      __syncwarp();
      {
        int lt = 0;
#pragma unroll
        for (int j = 0; j < 32; ++j) lt += wmin[warp * 32 + j] < mk ? 1 : 0;
        const int32_t twv = __reduce_max_sync(0xffffffffu, lt < kk ? mk : (int32_t)0x80000000);
        if (lane == 0) s_tw[warp] = twv;
      }
      team_sync<TT>(team);
      // (2) T = the smallest warp threshold: at least kk rows of the team have key <= T; every row with key <= T
      // goes to the team list (typically kk + a few rows; ballots that come back empty cost three instructions);
      int32_t T = s_tw[0];
#pragma unroll
      for (int w = 1; w < TW; ++w) T = min(T, s_tw[w]);
      T = min(T, MAXKEY - 1);
      if (__any_sync(0xffffffffu, mk <= T)) {
#pragma unroll
        for (int u = 0; u < SKEW_ROUNDS; ++u) {
          const bool take = key[u] <= T;
          const unsigned bal = __ballot_sync(0xffffffffu, take);
          if (bal) {
            uint32_t base = 0;
            if (lane == 0) base = atomicAdd(s_cnt, (uint32_t)__popc(bal));
            base = __shfl_sync(0xffffffffu, base, 0) + __popc(bal & ((1u << lane) - 1));
            if (take && base < (uint32_t)LIST) tl[base] = pack_cand(key[u], c0 + wbase + lane + 32 * (u - sh));
          }
        }
      }
      team_sync<TT>(team);
      // (3) the kk smallest of list + carried winners by RANK (packed (key, position) words are unique): thread i
      // counts the entries smaller than its own and stores it at that rank.
      const uint32_t cnt = *s_cnt;
      if (cnt > (uint32_t)LIST) {  // a flood of equal keys: the exact replay takes the slot
        replay = true;
      } else {
        const uint32_t tot = cnt + nw;
        const uint64_t* cold = car + par * SCAN_KFAST;
        uint64_t* cnew = car + (par ^ 1) * SCAN_KFAST;
        for (uint32_t i = ttid; i < tot; i += TT) {
          const uint64_t v = i < cnt ? tl[i] : cold[i - cnt];
          int rank = 0;
          for (uint32_t j = 0; j < cnt; ++j) rank += tl[j] < v ? 1 : 0;
          for (uint32_t j = 0; j < nw; ++j) rank += cold[j] < v ? 1 : 0;
          if (rank < kk) cnew[rank] = v;
        }
        nw = min((uint32_t)kk, tot);
        par ^= 1;
      }
      team_sync<TT>(team);
    }
    fast_slot_epilogue(a, slot, off, car + par * SCAN_KFAST, nw, replay, ttid, TT, rlist, rcount);
  }
}

// ------------------------------------------------------------------------------------------------
// IVF_FLAT: exact distances of the query to every row of a probed partition
// (FlatDistanceCal::distance_all, lance-index/src/vector/flat/storage.rs:397-403) + top-k.
// 16 lanes per row: lane l owns the reference's lane-accumulator l (elements 16c + l), so the L2 /
// dot results are bit-identical to l2.rs:57-91 / dot.rs:30-58; cosine follows cosine.rs:143-174 in
// structure (f32 FMA lanes) and is checked to the reference's own tolerance.
// ------------------------------------------------------------------------------------------------
// element of a stored / raw vector as f32 (l2.rs:100-106,156: f16 / bf16 elements are converted one by one)
template <class T> __device__ __forceinline__ float ldf(const T* p, int e);
template <> __device__ __forceinline__ float ldf<float>(const float* p, int e) { return p[e]; }
template <> __device__ __forceinline__ float ldf<__half>(const __half* p, int e) { return __half2float(p[e]); }
template <> __device__ __forceinline__ float ldf<__nv_bfloat16>(const __nv_bfloat16* p, int e) { return __bfloat162float(p[e]); }
template <> __device__ __forceinline__ float ldf<uint8_t>(const uint8_t* p, int e) { return (float)p[e]; }

template <int METRIC, class T = float>
__device__ __forceinline__ float flat_row_distance(const float* __restrict__ q, const T* __restrict__ v,
                                                   int d, int l, unsigned mask, float q_norm) {
  const int n16 = d & ~15;
  if (METRIC == METRIC_COSINE) {
    float xy = 0.0f, yy = 0.0f;
    for (int e = l; e < d; e += 16) {
      const float y = ldf<T>(v, e);
      xy = fmaf(q[e], y, xy);
      yy = fmaf(y, y, yy);
    }
#pragma unroll
    for (int off = 8; off >= 1; off >>= 1) {
      xy += __shfl_xor_sync(mask, xy, off, 16);
      yy += __shfl_xor_sync(mask, yy, off, 16);
    }
    return 1.0f - xy / q_norm / sqrtf(yy);
  }
  float acc = 0.0f;
  for (int e = l; e < n16; e += 16) acc = f_add(acc, term<METRIC>(q[e], ldf<T>(v, e)));
  float s = 0.0f;  // sequential tail, every lane redundantly (l2.rs:69-79)
  for (int e = n16; e < d; ++e) s = f_add(s, term<METRIC>(q[e], ldf<T>(v, e)));
  float t = 0.0f;
#pragma unroll
  for (int qq = 0; qq < 16; ++qq) t = f_add(t, __shfl_sync(mask, acc, qq, 16));
  return finish<METRIC>(f_add(s, t));
}

template <int METRIC, class T>
__global__ void __launch_bounds__(256)
ivfflat_scan_kernel(const float* __restrict__ queries, int d, const uint32_t* __restrict__ probe_ids,
                    int np, const uint64_t* __restrict__ part_offsets,
                    const T* __restrict__ vectors, const uint64_t* __restrict__ row_ids, int k,
                    float* __restrict__ cand_d, uint64_t* __restrict__ cand_id,
                    uint32_t* __restrict__ cand_cnt, const ScanFilter flt) {
  extern __shared__ float smem[];
  float* qs = smem;                          // [d]
  const SlotSmem s(qs + d, k + 1);
  __shared__ float s_qnorm;
  const int tid = threadIdx.x, l = tid & 15;
  const unsigned hmask = 0xffffu << (16 * ((tid >> 4) & 1));
  const int pi = blockIdx.x;
  const size_t qi = blockIdx.y;
  const uint32_t p = probe_ids[qi * np + pi];
  const uint64_t off = part_offsets[p];
  const uint32_t n_p = (uint32_t)(part_offsets[p + 1] - off);
  const size_t slot = qi * np + pi;
  if (n_p == 0) {
    if (tid == 0) cand_cnt[slot] = 0;
    return;
  }
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
  const uint32_t cnt = slot_topk(s, n_p, k, flt, off, false, fill);
  write_slot(s, cnt, slot, k, off, row_ids, cand_d, cand_id, cand_cnt);
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
template <int METRIC>
__device__ __forceinline__ uint32_t sq_word(uint32_t x, uint32_t q, uint32_t acc) {
  if (METRIC == METRIC_DOT) return __dp4a(x, q, acc);
  const uint32_t df = __vabsdiffu4(x, q);
  return __dp4a(df, df, acc);
}

template <int METRIC, bool VEC4>
__global__ void __maxnreg__(128)  // 256 threads; under __launch_bounds__(256) ptxas spills the selection's state
ivfsq_scan_kernel(const uint8_t* __restrict__ qcodes, int d, float r2, const uint32_t* __restrict__ probe_ids, int np,
                  const uint64_t* __restrict__ part_offsets, const uint8_t* __restrict__ codes,
                  const uint64_t* __restrict__ row_ids, int k, float* __restrict__ cand_d, uint64_t* __restrict__ cand_id,
                  uint32_t* __restrict__ cand_cnt, const ScanFilter flt) {
  extern __shared__ uint4 sq_smem[];
  const int nw = d >> 2;                                   // 4-byte words per row
  uint32_t* qw = reinterpret_cast<uint32_t*>(sq_smem);     // the query's codes, [nw] words (16-byte aligned)
  const SlotSmem s(qw + ((nw + 3) & ~3), k + 1);
  const int tid = threadIdx.x, l = tid & 7;
  const unsigned gmask = 0xffu << (8 * ((tid >> 3) & 3));  // the row's 8 lanes
  const int pi = blockIdx.x;
  const size_t qi = blockIdx.y;
  const uint32_t p = probe_ids[qi * np + pi];
  const uint64_t off = part_offsets[p];
  const uint32_t n_p = (uint32_t)(part_offsets[p + 1] - off);
  const size_t slot = qi * np + pi;
  if (n_p == 0) {
    if (tid == 0) cand_cnt[slot] = 0;
    return;
  }
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
        float f = __uint2float_rn(acc);
        if (METRIC == METRIC_DOT) f = __fsub_rn(1.0f, f);
        const float dist = __fdiv_rn(__fmul_rn(f, r2), 65025.0f);
        s.ukey[j] = (uint32_t)total_order_key(dist) ^ 0x80000000u;
      }
    }
  };
  const uint32_t cnt = slot_topk(s, n_p, k, flt, off, false, fill);
  write_slot(s, cnt, slot, k, off, row_ids, cand_d, cand_id, cand_cnt);
}

// ------------------------------------------------------------------------------------------------
// IVF_RQ: RabitDistCalculator (lance-index/src/vector/bq/storage.rs:160-445) + top-k, one CTA per (probe, query).
// rq = the slot's rotated residual query (dot(R[i, :d], q - c_p), storage.rs:130-156).  In shared memory:
//   - the code_dim / 4 sub-tables of 16 entries by the lowbit chain t[j] = t[j - lowbit(j)] + rq[4s + ctz(j)]
//     (storage.rs:210-245), which fixes the rounding order;
//   - sum_q = the sequential f32 sum of rq from -0.0 (Rust's float Sum);
//   - the table quantised to u8 with qmin / qmax over the whole table in total_cmp order (storage.rs:249-267).
// distance_all (storage.rs:319-369): the rows before the partition's last n_p % 32 sum u8 entries in 16-bit lanes
// that wrap mod 2^16, as the x86 kernels do (dist_table.rs:96-160, dist_table.c) -- an exact u32 sum & 0xffff --
// and are dequantised as q * ((qmax - qmin) / 255) + (code_dim / 4) * qmin; the last n_p % 32 rows take the exact
// f32 sum of the pairs t_lo[lo] + t_hi[hi] from 0.0.  With a prefilter every row takes DistCalculator::distance
// (storage.rs:297-316), the same pair sums from -0.0; no table entry is -0.0 (t[0] = +0.0 and x + y is -0.0 only
// when both are), so the start does not matter.  Then ((2 dist - sum_q) / sqrt_d) * scale + add + q_factor, each
// operation rounded on its own.  Codes are row-major [n][code_dim / 8]; the 32-row rule uses the partition-local row.
// ------------------------------------------------------------------------------------------------
static size_t rq_scan_smem_bytes(int code_dim, int k) {
  return (size_t)code_dim * 4 * (sizeof(float) + 1) + slot_smem_bytes(k);
}

__global__ void __launch_bounds__(256)
ivfrq_scan_kernel(const float* __restrict__ rq, int code_dim, float sqrt_d, int q_minus_one,
                  const uint32_t* __restrict__ probe_ids, const float* __restrict__ probe_dists, int np,
                  const uint64_t* __restrict__ part_offsets, const uint8_t* __restrict__ codes,
                  const float* __restrict__ add, const float* __restrict__ scale, const uint64_t* __restrict__ row_ids,
                  int k, float* __restrict__ cand_d, uint64_t* __restrict__ cand_id, uint32_t* __restrict__ cand_cnt,
                  const ScanFilter flt) {
  extern __shared__ float rq_smem[];
  const int nt = code_dim >> 2;  // sub-tables of 16 entries
  float* tab = rq_smem;                                      // [nt * 16] f32
  uint8_t* qt = reinterpret_cast<uint8_t*>(tab + nt * 16);  // [nt * 16] u8 (code_dim % 8 == 0: 4-byte aligned end)
  const SlotSmem s(qt + nt * 16, k + 1);
  __shared__ int32_t s_mn, s_mx;
  __shared__ float s_sum_q;
  const int tid = threadIdx.x;
  const int pi = blockIdx.x;
  const size_t qi = blockIdx.y;
  const size_t slot = qi * np + pi;
  const uint32_t p = probe_ids[slot];
  const uint64_t off = part_offsets[p];
  const uint32_t n_p = (uint32_t)(part_offsets[p + 1] - off);
  if (n_p == 0) {
    if (tid == 0) cand_cnt[slot] = 0;
    return;
  }
  const float* r = rq + slot * (size_t)code_dim;
  if (tid == 0) { s_mn = 0x7fffffff; s_mx = (int32_t)0x80000000; }
  for (int st = tid; st < nt; st += 256) {
    float t[16];
    t[0] = 0.0f;
#pragma unroll
    for (int j = 1; j < 16; ++j) {
      const int ctz = (j & 1) ? 0 : (j & 2) ? 1 : (j & 4) ? 2 : 3;
      t[j] = __fadd_rn(t[j - (j & -j)], r[4 * st + ctz]);
    }
#pragma unroll
    for (int j = 0; j < 16; ++j) tab[st * 16 + j] = t[j];
  }
  __syncthreads();
  int32_t mn = 0x7fffffff, mx = (int32_t)0x80000000;
  for (int i = tid; i < nt * 16; i += 256) {
    const int32_t kv = total_order_key(tab[i]);
    mn = min(mn, kv);
    mx = max(mx, kv);
  }
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) {
    mn = min(mn, __shfl_xor_sync(0xffffffffu, mn, o));
    mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  }
  if ((tid & 31) == 0) { atomicMin(&s_mn, mn); atomicMax(&s_mx, mx); }
  if (tid == 0) {
    float sq = -0.0f;
    for (int i = 0; i < code_dim; ++i) sq = __fadd_rn(sq, r[i]);
    s_sum_q = sq;
  }
  __syncthreads();
  const float qmin = key_to_float(s_mn), qmax = key_to_float(s_mx);
  if (flt.allow == nullptr) {
    const bool flat = qmin == qmax;  // e.g. a zero residual query: all codes 0
    const float factor = flat ? 0.0f : __fdiv_rn(255.0f, __fsub_rn(qmax, qmin));
    for (int i = tid; i < nt * 16; i += 256) {
      const float v = flat ? 0.0f : roundf(__fmul_rn(__fsub_rn(tab[i], qmin), factor));  // f32::round
      qt[i] = (v != v) ? 0 : v <= 0.0f ? 0 : v >= 255.0f ? 255 : (uint8_t)v;           // `as u8`
    }
  }
  __syncthreads();
  const float range = __fdiv_rn(__fsub_rn(qmax, qmin), 255.0f), sum_min = __fmul_rn((float)nt, qmin);
  const float sum_q = s_sum_q, dqc = probe_dists[slot];
  const float q_factor = q_minus_one ? __fsub_rn(dqc, 1.0f) : dqc;  // storage.rs:427-434
  const int cb = code_dim >> 3;
  const uint8_t* pc = codes + off * cb;
  const uint32_t n_quant = flt.allow ? 0u : n_p - n_p % 32;
  auto fill = [&](uint32_t c0, uint32_t clen) {
    for (uint32_t j = tid; j < clen; j += 256) {
      const uint32_t row = c0 + j;
      const uint8_t* rp = pc + (size_t)row * cb;
      float dist;
      if (row < n_quant) {
        uint32_t qs = 0;
        for (int i = 0; i < cb; ++i) {
          const uint32_t c = __ldg(rp + i);
          qs += (uint32_t)qt[(2 * i) * 16 + (c & 15)] + (uint32_t)qt[(2 * i + 1) * 16 + (c >> 4)];
        }
        dist = __fadd_rn(__fmul_rn(__uint2float_rn(qs & 0xffffu), range), sum_min);
      } else {
        dist = 0.0f;
        for (int i = 0; i < cb; ++i) {
          const uint32_t c = __ldg(rp + i);
          dist = __fadd_rn(dist, __fadd_rn(tab[(2 * i) * 16 + (c & 15)], tab[(2 * i + 1) * 16 + (c >> 4)]));
        }
      }
      const float dvq = __fdiv_rn(__fsub_rn(__fmul_rn(2.0f, dist), sum_q), sqrt_d);
      float out = __fadd_rn(__fadd_rn(__fmul_rn(dvq, scale[off + row]), add[off + row]), q_factor);
      // x86's default NaN (0xFFC00000, ordered before every number): with finite rows a NaN only comes from invalid
      // operations, e.g. on a normalised zero query under cosine, and the reference runs on x86
      if (out != out) out = __int_as_float(0xffc00000);
      s.ukey[j] = (uint32_t)total_order_key(out) ^ 0x80000000u;
    }
  };
  const uint32_t cnt = slot_topk(s, n_p, k, flt, off, false, fill);
  write_slot(s, cnt, slot, k, off, row_ids, cand_d, cand_id, cand_cnt);
}

// residual queries of `nq` queries x np probes: out[(q np + pi) d + t] = queries[q d + t] - c_{probe}[t]
// (a probe id >= K is an empty slot of a search with minimum / maximum nprobes: its residual is 0)
__global__ void rq_query_residual_kernel(const float* __restrict__ queries, uint64_t nq, int np, int d,
                                         const float* __restrict__ centroids, int K,
                                         const uint32_t* __restrict__ probe_ids, float* __restrict__ out) {
  const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= nq * np * d) return;
  const uint64_t sl = g / d;
  const int t = (int)(g % d);
  const uint32_t p = probe_ids[sl];
  out[g] = p < (uint32_t)K ? __fsub_rn(queries[(sl / np) * d + t], centroids[(size_t)p * d + t]) : 0.0f;
}

// global merge per query: ascending (distance, row id), first k.  Candidate e of list pi of query qi sits
// at cand[pi * stride_p + qi * stride_q + e] (per-partition lists of one GPU: stride_p = k, stride_q = np * k;
// per-rank results gathered from a sharded index: stride_p = the rank stride, stride_q = k).
// Lists of up to MERGE_RANK_MAX candidates in total are merged by RANK COUNTING in shared memory: every candidate
// counts the candidates that precede it in (distance, row id) order -- the pairs are unique -- and the ones with rank
// < k are the output, already in place.  (The k-round argmin below re-reads all candidates from global memory per
// round: 3.6 ms for 10 000 queries x 10 lists x k = 100; it remains for larger totals.)
constexpr int MERGE_RANK_MAX = 2048;
__global__ void __launch_bounds__(256)
merge_rank_kernel(const float* __restrict__ cand_d, const uint64_t* __restrict__ cand_id,
                  const uint32_t* __restrict__ cand_cnt, int np, int k, size_t stride_p_d, size_t stride_p_id,
                  size_t stride_q, size_t cnt_stride_p, size_t cnt_stride_q, uint64_t* __restrict__ out_id,
                  float* __restrict__ out_d, uint32_t* __restrict__ out_cnt) {
  extern __shared__ __align__(16) unsigned char mr_smem[];
  const int total = np * k;
  uint64_t* s_id = reinterpret_cast<uint64_t*>(mr_smem);             // [total]
  int32_t* s_key = reinterpret_cast<int32_t*>(s_id + total);         // [total]; invalid entries: key = INT_MAX, id = ~0
  __shared__ uint32_t s_valid;
  const size_t qi = blockIdx.x;
  const int tid = threadIdx.x;
  if (tid == 0) s_valid = 0;
  __syncthreads();
  uint32_t myvalid = 0;
  for (int c = tid; c < total; c += 256) {
    const int pi = c / k, e = c % k;
    const bool ok = (uint32_t)e < cand_cnt[pi * cnt_stride_p + qi * cnt_stride_q];
    s_key[c] = ok ? total_order_key(cand_d[pi * stride_p_d + qi * stride_q + e]) : 0x7fffffff;
    s_id[c] = ok ? cand_id[pi * stride_p_id + qi * stride_q + e] : ~0ull;
    myvalid += ok ? 1u : 0u;
  }
  if (myvalid) atomicAdd(&s_valid, myvalid);
  __syncthreads();
  for (int c = tid; c < total; c += 256) {
    const uint64_t id = s_id[c];
    if (id == ~0ull && s_key[c] == 0x7fffffff) continue;
    const int32_t key = s_key[c];
    int rank = 0;
    for (int j = 0; j < total; ++j) {
      const int32_t kj = s_key[j];
      rank += (kj < key || (kj == key && s_id[j] < id)) ? 1 : 0;
    }
    if (rank < k) {
      out_id[qi * k + rank] = id;
      out_d[qi * k + rank] = key_to_float(key);
    }
  }
  const int r = min((uint32_t)k, s_valid);
  for (int e = r + tid; e < k; e += 256) {
    out_id[qi * k + e] = ~0ull;
    out_d[qi * k + e] = __int_as_float(0x7f800000);
  }
  if (tid == 0 && out_cnt) out_cnt[qi] = r;
}

__global__ void __launch_bounds__(128)
merge_kernel(const float* __restrict__ cand_d, const uint64_t* __restrict__ cand_id,
             const uint32_t* __restrict__ cand_cnt, int np, int k, size_t stride_p_d, size_t stride_p_id,
             size_t stride_q, size_t cnt_stride_p, size_t cnt_stride_q, uint64_t* __restrict__ out_id,
             float* __restrict__ out_d, uint32_t* __restrict__ out_cnt) {
  const size_t qi = blockIdx.x;
  const int tid = threadIdx.x;
  const int r = (int)emit_ascending<128>(
      k, np * k,
      [&](uint32_t c, int32_t& key, uint64_t& id) {
        const int pi = c / k, e = c % k;
        if ((uint32_t)e >= cand_cnt[pi * cnt_stride_p + qi * cnt_stride_q]) return false;
        key = total_order_key(cand_d[pi * stride_p_d + qi * stride_q + e]);
        id = cand_id[pi * stride_p_id + qi * stride_q + e];
        return true;
      },
      [&](uint32_t r, uint32_t c, int32_t, uint64_t id) {
        out_id[qi * k + r] = id;
        out_d[qi * k + r] = cand_d[(c / k) * stride_p_d + qi * stride_q + (c % k)];
      });
  for (int e = r + tid; e < k; e += 128) {
    out_id[qi * k + e] = ~0ull;
    out_d[qi * k + e] = __int_as_float(0x7f800000);
  }
  if (tid == 0 && out_cnt) out_cnt[qi] = r;
}

// ------------------------------------------------------------------------------------------------
// primitives exported one-to-one (used by the trait-level shim and by the parity tests)
// ------------------------------------------------------------------------------------------------
template <int METRIC>
__global__ void build_lut_kernel(const float* __restrict__ codebook, int M, int ncode, int ds,
                                 const float* __restrict__ query, float* __restrict__ lut) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= M * ncode) return;
  const int m = idx / ncode;
  lut[idx] = dist_exact_thread<METRIC>(query + m * ds, codebook + (size_t)idx * ds, ds);
}

__global__ void pq_scan_transposed_kernel(const float* __restrict__ lut, int M,
                                          const uint8_t* __restrict__ codes_t, uint64_t n,
                                          int is_dot, float* __restrict__ out) {
  extern __shared__ float s_lut[];
  for (int i = threadIdx.x; i < M * 256; i += blockDim.x) s_lut[i] = lut[i];
  __syncthreads();
  const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  float dist = 0.0f;
  for (int m = 0; m < M; ++m) dist = f_add(dist, s_lut[m * 256 + codes_t[(size_t)m * n + j]]);
  if (is_dot) dist = __fsub_rn(dist, (float)M - 1.0f);
  out[j] = dist;
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

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
// the shared memory a launch of `kernel` with `dyn` dynamic bytes takes: its static shared memory counts against the
// same per-block opt-in limit, and cudaFuncSetAttribute refuses a dynamic size that leaves no room for it
template <class Kern>
static size_t smem_with_static(Kern kernel, size_t dyn) {
  cudaFuncAttributes fa;
  LB2_CUDA(cudaFuncGetAttributes(&fa, kernel));
  return dyn + fa.sharedSizeBytes;
}

void find_partitions_f32(const float* centroids, int K, int d, int metric, const float* queries,
                         uint64_t nq, int nprobes, uint32_t* ids, float* dists) {
  if (nq == 0) return;
  DevBuf<float> all((size_t)nq * K);
  assign_f32(queries, nq, d, centroids, K, metric, nullptr, nullptr, nullptr, nullptr, all.p);
  LB2_LAUNCH("select_probes", select_probes_kernel, (unsigned)nq, 128, 0, all.p, K, nprobes, ids, dists);
}

// which fast kernel serves an 8-bit scan: LB2_SCAN=classic|skew overrides the size rule (tests run both)
static int scan_mode_env() {
  const char* e = getenv("LB2_SCAN");
  return !e ? 0 : (!strcmp(e, "classic") ? 1 : (!strcmp(e, "skew") ? 2 : 0));
}

template <int METRIC>
static void scan_launch(int nbits, dim3 grid, size_t smem, const ScanArgs& a, uint32_t* rlist, uint32_t* rcount,
                        const uint64_t* slab_off, const uint8_t* skew) {
  const bool filtering = a.flt.allow != nullptr || a.flt.range;
  if (nbits == 8 && a.k + 1 <= SCAN_KFAST) {
    const size_t smem_fast = sizeof(float) * ((size_t)a.M * 256 + a.d);
    LB2_CUDA(cudaMemsetAsync(rcount, 0, sizeof(uint32_t), ctx().stream));
    const uint64_t nslots = (uint64_t)grid.x * grid.y;
    const bool skew_ok = skew && a.M == 16 && a.ds == 8 && (reinterpret_cast<uintptr_t>(a.queries) & 15) == 0 &&
                         (size_t)SKEW_SMEM_BYTES <= ctx().smem_optin;
    // The persistent kernel wins at every batch size measured (profiles/scan_variants_r02.json: 19 vs 33 us for one
    // query, 3.9 vs 5.9 ms for 10 000 x 10 probes); LB2_SCAN=classic|skew and LB2_SCAN_TEAMS=2|4 override for tests.
    const bool use_skew = skew_ok && scan_mode_env() != 1;
    if (use_skew) {
      const char* te = getenv("LB2_SCAN_TEAMS");
      // four single-copy teams per SM once every SM has several slots per team; two double-copy teams below that
      const int nteam = te && atoi(te) == 2 ? 2 : (te && atoi(te) == 4 ? 4 : (nslots >= 16ull * ctx().num_sms ? 4 : 2));
      const unsigned g = (unsigned)std::min<uint64_t>((nslots + nteam - 1) / nteam, (uint64_t)ctx().num_sms);
      auto go = [&](auto kern) {
        set_smem(kern, SKEW_SMEM_BYTES);
        LB2_LAUNCH("pq_scan_skew", kern, g, 512, SKEW_SMEM_BYTES, a, slab_off, skew, (uint32_t)nslots, rlist, rcount);
      };
      if (filtering) {
        if (nteam == 2) go(ivfpq_scan_skew_kernel<METRIC, true, 2>); else go(ivfpq_scan_skew_kernel<METRIC, true, 4>);
      } else {
        if (nteam == 2) go(ivfpq_scan_skew_kernel<METRIC, false, 2>); else go(ivfpq_scan_skew_kernel<METRIC, false, 4>);
      }
    } else if (filtering) {  // filtered rows never enter the candidate lists
      set_smem(ivfpq_scan_kernel<METRIC, true>, smem_fast);
      LB2_LAUNCH("pq_scan", (ivfpq_scan_kernel<METRIC, true>), grid, 256, smem_fast, a, rlist, rcount);
    } else {
      set_smem(ivfpq_scan_kernel<METRIC, false>, smem_fast);
      LB2_LAUNCH("pq_scan", (ivfpq_scan_kernel<METRIC, false>), grid, 256, smem_fast, a, rlist, rcount);
    }
    // slots with ties beyond the k-th place (rare): the reference's heap loop, restated
    set_smem((ivfpq_scan_radix_kernel<METRIC, 8>), smem);
    const unsigned rgrid = (unsigned)std::min<uint64_t>((uint64_t)grid.x * grid.y, 4 * (uint64_t)ctx().num_sms);
    LB2_LAUNCH("pq_scan_tie_replay", (ivfpq_scan_radix_kernel<METRIC, 8>), rgrid, 256, smem, a,
               (const uint32_t*)rlist, (const uint32_t*)rcount);
    return;
  }
  if (nbits == 4) {
    set_smem((ivfpq_scan_radix_kernel<METRIC, 4>), smem);
    LB2_LAUNCH("pq_scan", (ivfpq_scan_radix_kernel<METRIC, 4>), grid, 256, smem, a, (const uint32_t*)nullptr,
               (const uint32_t*)nullptr);
    return;
  }
  set_smem((ivfpq_scan_radix_kernel<METRIC, 8>), smem);
  LB2_LAUNCH("pq_scan", (ivfpq_scan_radix_kernel<METRIC, 8>), grid, 256, smem, a, (const uint32_t*)nullptr,
             (const uint32_t*)nullptr);
}

// np lists of <= k candidates per query -> the k smallest by (distance, row id)
static void merge_lists(const char* name, uint64_t nq, const float* cand_d, const uint64_t* cand_id, const uint32_t* cand_cnt,
                        int np, int k, size_t stride_p_d, size_t stride_p_id, size_t stride_q, size_t cnt_stride_p,
                        size_t cnt_stride_q, uint64_t* out_ids, float* out_dists, uint32_t* out_counts) {
  if (nq == 0) return;
  const size_t total = (size_t)np * k;
  if (total <= (size_t)MERGE_RANK_MAX) {
    LB2_LAUNCH(name, merge_rank_kernel, (unsigned)nq, 256, total * 12, cand_d, cand_id, cand_cnt, np, k, stride_p_d, stride_p_id,
               stride_q, cnt_stride_p, cnt_stride_q, out_ids, out_dists, out_counts);
  } else {
    LB2_LAUNCH(name, merge_kernel, (unsigned)nq, 128, 0, cand_d, cand_id, cand_cnt, np, k, stride_p_d, stride_p_id, stride_q,
               cnt_stride_p, cnt_stride_q, out_ids, out_dists, out_counts);
  }
}

// The IVF query skeleton: the nprobes nearest partitions of every query, one candidate list of <= k per (query,
// probe) slot, the lists merged per query.  scan(q0, qn, np, offsets, probe_ids, probe_dists, cand_d, cand_id,
// cand_cnt) fills the lists of queries [q0, q0 + qn) (at most 32768 of them: the grid.y limit), np slots per query; probe_dists are
// find_partitions' distances of the probed centroids (dist_q_c).
constexpr uint64_t SEARCH_SLAB = 32768;
template <class Scan>
static void ivf_search(const float* centroids, int K, int d, int metric, const float* queries, uint64_t nq, int k,
                       int np, const uint64_t* part_offsets, uint64_t* out_ids, float* out_dists, uint32_t* out_counts,
                       Scan scan) {
  // partitions are found with L2 on the (normalised) vectors for cosine (ivf.rs:149-185)
  const int cmetric = metric == METRIC_DOT ? METRIC_DOT : METRIC_L2;
  DevBuf<uint32_t> pids((size_t)nq * np), cand_cnt((size_t)nq * np);
  DevBuf<float> pd((size_t)nq * np), cand_d((size_t)nq * np * k);
  DevBuf<uint64_t> cand_id((size_t)nq * np * k);
  find_partitions_f32(centroids, K, d, cmetric, queries, nq, np, pids.p, pd.p);
  for (uint64_t q0 = 0; q0 < nq; q0 += SEARCH_SLAB)
    scan(q0, std::min<uint64_t>(SEARCH_SLAB, nq - q0), np, part_offsets, pids.p + q0 * np, pd.p + q0 * np, cand_d.p + q0 * np * k,
         cand_id.p + q0 * np * k, cand_cnt.p + q0 * np);
  merge_lists("merge_topk", nq, cand_d.p, cand_id.p, cand_cnt.p, np, k, (size_t)k, (size_t)k, (size_t)np * k, (size_t)1,
              (size_t)np, out_ids, out_dists, out_counts);
}

// The same skeleton with a per-query probe count (probe.cu): per slab of queries every centroid distance is ranked
// (P = the first L = min(maximum_nprobes or K, K)), the cutoff fixes how many of P each query searches, and the scan
// runs over a grid as wide as the slab's largest count.  A query's slots past its own count hold the partition id K,
// which `ext_offsets` (part_offsets with one more empty partition) makes an empty partition for every scan kernel.
// With a mask the query may answer from (`pr.mask_ids`), every query gets one more slot: the shortcut list.
// With a range bound c_p depends on the distances: all L partitions are scanned, the cutoff reads the scan's list
// counts and empties the lists past it.  Candidate memory is bounded by sub-slabs of about 256 MB.
template <class Scan>
static void ivf_search_probed(const float* centroids, int K, int d, int metric, const float* queries, uint64_t nq,
                              int kc, const uint64_t* part_offsets, const ScanFilter& flt, const ProbeRule& pr,
                              uint64_t* out_ids, float* out_dists, uint32_t* out_counts, Scan scan) {
  if (nq == 0) return;
  const int cmetric = metric == METRIC_DOT ? METRIC_DOT : METRIC_L2;
  const int L = pr.max_np ? (int)std::min<uint32_t>(pr.max_np, (uint32_t)K) : K;
  const bool by_scan = flt.range != 0;
  const int extra = pr.mask_ids ? 1 : 0;
  DevBuf<uint64_t> ext_offsets((size_t)K + 2);
  d2d(ext_offsets.p, part_offsets, (size_t)K + 1);
  d2d(ext_offsets.p + K + 1, part_offsets + K, 1);
  DevBuf<uint32_t> cpart;
  if (!by_scan) {
    cpart.alloc(K);
    partition_counts(part_offsets, K, flt.allow, (uint32_t)kc, cpart.p);
  }
  // the ranking's buffers: distances, and two runs of packed words above one tile
  const uint64_t rank_bytes = (uint64_t)K * (K > RANK_TILE ? 20 : 4) + (uint64_t)L * 8;
  const uint64_t qs = std::max<uint64_t>(1, std::min<uint64_t>(SEARCH_SLAB, (256ull << 20) / rank_bytes));
  DevBuf<float> all(std::min(qs, nq) * K), pd(std::min(qs, nq) * L);
  DevBuf<uint32_t> pids(std::min(qs, nq) * L), nsearch(std::min(qs, nq)), shortcut(std::min(qs, nq)), nmax(1);
  for (uint64_t q0 = 0; q0 < nq; q0 += qs) {
    const uint64_t qn = std::min(qs, nq - q0);
    assign_f32(queries + q0 * d, qn, d, centroids, K, cmetric, nullptr, nullptr, nullptr, nullptr, all.p);
    rank_probes(all.p, qn, K, L, pids.p, pd.p);
    uint32_t* nprobes_out = pr.nprobes_out ? pr.nprobes_out + q0 : nullptr;
    int np = L;
    if (!by_scan) {
      nmax.zero();
      probe_cutoff(pr, qn, L, pids.p, pd.p, cpart.p, nullptr, 0, nsearch.p, shortcut.p, nmax.p, nprobes_out);
      uint32_t h = 0;
      d2h(&h, nmax.p, 1);
      sync_stream();
      np = (int)h;
    }
    const int nl = np + extra;  // slots per query
    DevBuf<uint32_t> sp((size_t)qn * nl);
    DevBuf<float> spd((size_t)qn * nl);
    gather_probes(qn, L, pids.p, pd.p, by_scan ? nullptr : nsearch.p, nl, (uint32_t)K, sp.p, spd.p);
    const uint64_t per_q = (uint64_t)nl * kc * 12 + 4 * (uint64_t)nl;
    const uint64_t sub = std::max<uint64_t>(1, std::min<uint64_t>(qn, (256ull << 20) / per_q));
    DevBuf<float> cd(sub * nl * kc);
    DevBuf<uint64_t> cid(sub * nl * kc);
    DevBuf<uint32_t> ccnt(sub * nl);
    for (uint64_t a = 0; a < qn; a += sub) {
      const uint64_t b = std::min(sub, qn - a);
      scan(q0 + a, b, nl, ext_offsets.p, sp.p + a * nl, spd.p + a * nl, cd.p, cid.p, ccnt.p);
      if (by_scan)
        probe_cutoff(pr, b, L, pids.p + a * L, pd.p + a * L, nullptr, ccnt.p, nl, nsearch.p + a, shortcut.p + a,
                     nmax.p, nprobes_out ? nprobes_out + a : nullptr);
      if (extra) shortcut_lists(b, shortcut.p + a, pr.mask_ids, pr.num_mask_ids, nl, kc, cd.p, cid.p, ccnt.p);
      merge_lists("merge_topk", b, cd.p, cid.p, ccnt.p, nl, kc, (size_t)kc, (size_t)kc, (size_t)nl * kc, (size_t)1,
                  (size_t)nl, out_ids + (q0 + a) * kc, out_dists + (q0 + a) * kc, out_counts ? out_counts + q0 + a : nullptr);
    }
  }
}

// the fixed-nprobes skeleton, or with a probe rule the per-query one
template <class Scan>
static void run_ivf_search(const float* centroids, int K, int d, int metric, const float* queries, uint64_t nq, int k,
                           int nprobes, const uint64_t* part_offsets, const ScanFilter& flt, const ProbeRule* pr,
                           uint64_t* out_ids, float* out_dists, uint32_t* out_counts, Scan scan) {
  if (pr)
    ivf_search_probed(centroids, K, d, metric, queries, nq, k, part_offsets, flt, *pr, out_ids, out_dists, out_counts,
                      scan);
  else
    ivf_search(centroids, K, d, metric, queries, nq, k, nprobes < K ? nprobes : K, part_offsets, out_ids, out_dists,
               out_counts, scan);
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

// the skewed copy of an index's codes (see ivfpq_scan_skew_kernel); sizes: slab_off u64[K + 1],
// skew (n / 512 + K) slabs of 8704 bytes at most
bool skew_layout_applies(int M, int d, int nbits) { return nbits == 8 && M == 16 && d == 128; }
size_t skew_bytes_bound(uint64_t n, int K) { return (size_t)(n / SKEW_SLAB_ROWS + (uint64_t)K) * SKEW_SLAB_BYTES; }
void build_skew_codes(const uint64_t* part_offsets, int K, const uint8_t* codes, uint64_t n, uint64_t* slab_off,
                      uint8_t* skew) {
  LB2_LAUNCH("skew_offsets", skew_offsets_kernel, 1, 1024, 0, part_offsets, K, slab_off);
  const unsigned g = (unsigned)std::min<uint64_t>(cdiv(n / SKEW_SLAB_ROWS + (uint64_t)K, 8), 8ull * ctx().num_sms);
  if (n) LB2_LAUNCH("skew_fill", skew_fill_kernel, std::max(1u, g), 256, 0, part_offsets, K, (const uint64_t*)slab_off, codes, skew);
}

void ivfpq_search_f32(const float* centroids, int K, int d, int metric, const float* codebook, int M,
                      int nbits, const uint64_t* part_offsets, const uint8_t* codes,
                      const uint64_t* row_ids, const float* queries, uint64_t nq, int k, int nprobes,
                      uint64_t* out_ids, float* out_dists, uint32_t* out_counts, const ScanFilter& flt,
                      const uint64_t* slab_off, const uint8_t* skew, const ProbeRule* pr) {
  if (nq == 0 || k == 0) return;
  if (nbits != 8 && nbits != 4) fail(LB2_INVALID_ARG, "PQ: num_bits must be 4 or 8, got %d", nbits);
  if (nbits == 4 && (M % 2 != 0 || M > 256)) fail(LB2_UNSUPPORTED, "4-bit PQ needs an even num_sub_vectors <= 256");
  if (k > 1024) fail(LB2_UNSUPPORTED, "k (incl. refine factor) > 1024 is not implemented");
  const int np = nprobes < K ? nprobes : K;
  const size_t smem = sizeof(float) * ((size_t)M * (nbits == 4 ? 16 : 256) + d) + slot_smem_bytes(k);
  // every kernel the scan may launch must fit: the radix kernel (the scan itself, or the tie replay of the fast
  // 8-bit kernels) and, for k + 1 <= SCAN_KFAST, the classic fast kernel with its LUT and larger static lists
  size_t need = 0;
  auto need_of = [&](auto m) {
    constexpr int METRIC = decltype(m)::value;
    need = nbits == 4 ? smem_with_static(ivfpq_scan_radix_kernel<METRIC, 4>, smem)
                      : smem_with_static(ivfpq_scan_radix_kernel<METRIC, 8>, smem);
    if (nbits == 8 && k + 1 <= SCAN_KFAST) {
      const size_t fast = sizeof(float) * ((size_t)M * 256 + d);
      const bool filtering = flt.allow != nullptr || flt.range;
      need = std::max(need, filtering ? smem_with_static(ivfpq_scan_kernel<METRIC, true>, fast)
                                      : smem_with_static(ivfpq_scan_kernel<METRIC, false>, fast));
    }
  };
  if (metric == METRIC_DOT) need_of(std::integral_constant<int, METRIC_DOT>{});
  else need_of(std::integral_constant<int, METRIC_L2>{});
  if (need > ctx().smem_optin) fail(LB2_UNSUPPORTED, "LUT and top-k scratch of %zu bytes exceed shared memory", need);
  DevBuf<uint32_t> rlist((size_t)std::min<uint64_t>(nq, SEARCH_SLAB) * np), rcount(1);
  run_ivf_search(centroids, K, d, metric, queries, nq, k, np, part_offsets, flt, pr, out_ids, out_dists, out_counts,
             [&](uint64_t q0, uint64_t qn, int np, const uint64_t* offs, const uint32_t* pids, const float*, float* cd,
                 uint64_t* cid, uint32_t* ccnt) {
               if (rlist.n < qn * np) rlist.alloc(qn * np);
               const ScanArgs a{queries + q0 * d, d, centroids, codebook, M, d / M, pids, np, offs, codes,
                                row_ids, k, cd, cid, ccnt, flt};
               const dim3 g(np, (unsigned)qn);
               if (metric == METRIC_DOT)
                 scan_launch<METRIC_DOT>(nbits, g, smem, a, rlist.p, rcount.p, slab_off, skew);
               else
                 scan_launch<METRIC_L2>(nbits, g, smem, a, rlist.p, rcount.p, slab_off, skew);
             });
}

// Row-sharded index (SURVEY 8e search (ii)): every rank has searched its own shard; the per-rank top-k lists
// are exchanged in ONE collective and merged on every rank by (_distance, _rowid), the order of the
// reference's final SortExec (rust/lance/src/dataset/scanner.rs:3450-3466).  ids / dists / counts: this
// rank's [nq][k] / [nq] results on the device; outputs likewise.
void merge_sharded_topk(const uint64_t* ids, const float* dists, const uint32_t* counts, uint64_t nq, int k,
                        uint64_t* out_ids, float* out_dists, uint32_t* out_counts) {
  Comm* c = current_comm();
  const int nr = c ? c->nranks : 1;
  const size_t id_bytes = (size_t)nq * k * 8, d_bytes = ((size_t)nq * k * 4 + 7) / 8 * 8, c_bytes = ((size_t)nq * 4 + 7) / 8 * 8;
  const size_t S = id_bytes + d_bytes + c_bytes;
  DevBuf<uint8_t> blob(S), gathered(S * nr);
  LB2_CUDA(cudaMemcpyAsync(blob.p, ids, (size_t)nq * k * 8, cudaMemcpyDeviceToDevice, ctx().stream));
  LB2_CUDA(cudaMemcpyAsync(blob.p + id_bytes, dists, (size_t)nq * k * 4, cudaMemcpyDeviceToDevice, ctx().stream));
  LB2_CUDA(cudaMemcpyAsync(blob.p + id_bytes + d_bytes, counts, (size_t)nq * 4, cudaMemcpyDeviceToDevice, ctx().stream));
  comm_allgather_bytes(blob.p, gathered.p, S);
  merge_lists("merge_sharded_topk", nq, reinterpret_cast<const float*>(gathered.p + id_bytes),
              reinterpret_cast<const uint64_t*>(gathered.p), reinterpret_cast<const uint32_t*>(gathered.p + id_bytes + d_bytes),
              nr, k, S / 4, S / 8, (size_t)k, S / 4, (size_t)1, out_ids, out_dists, out_counts);
  sync_stream();  // the exchange buffers are freed on return
}

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
void row_mask_f32(const uint64_t* row_ids, uint64_t n, const uint64_t* allow, uint64_t n_allow, bool has_allow,
                  const uint64_t* block, uint64_t n_block, bool has_block, uint64_t* bitmap) {
  const uint64_t padded = (n + 63) / 64 * 64;
  if (padded == 0) return;
  LB2_LAUNCH("row_mask", row_mask_kernel, cdiv(padded, 256), 256, 0, row_ids, n, allow, n_allow,
             has_allow ? 1 : 0, block, n_block, has_block ? 1 : 0, reinterpret_cast<uint32_t*>(bitmap));
}

void ivfflat_search_f32(const float* centroids, int K, int d, int metric, const uint64_t* part_offsets,
                        const void* vectors, int vdt, const uint64_t* row_ids, const float* queries, uint64_t nq,
                        int k, int nprobes, uint64_t* out_ids, float* out_dists, uint32_t* out_counts,
                        const ScanFilter& flt, const ProbeRule* pr) {
  if (nq == 0 || k == 0) return;
  if (k > 1024) fail(LB2_UNSUPPORTED, "k (incl. refine factor) > 1024 is not implemented");
  const size_t smem = sizeof(float) * (size_t)d + slot_smem_bytes(k);
  size_t need = 0;
  dispatch_metric_elem<false>(metric, vdt, [&](auto m, auto e) {
    need = smem_with_static(ivfflat_scan_kernel<decltype(m)::value, typename decltype(e)::type>, smem);
  });
  if (need > ctx().smem_optin) fail(LB2_UNSUPPORTED, "dimension %d too large for the flat scan", d);
  run_ivf_search(centroids, K, d, metric, queries, nq, k, nprobes, part_offsets, flt, pr, out_ids, out_dists, out_counts,
             [&](uint64_t q0, uint64_t qn, int np, const uint64_t* offs, const uint32_t* pids, const float*, float* cd,
                 uint64_t* cid, uint32_t* ccnt) {
               dispatch_metric_elem<false>(metric, vdt, [&](auto m, auto e) {
                 using T = typename decltype(e)::type;
                 auto kern = ivfflat_scan_kernel<decltype(m)::value, T>;
                 set_smem(kern, smem);
                 LB2_LAUNCH("flat_scan", kern, dim3(np, (unsigned)qn), 256, smem, queries + q0 * d, d, pids, np,
                            offs, reinterpret_cast<const T*>(vectors), row_ids, k, cd, cid, ccnt, flt);
               });
             });
}

void ivfsq_search_f32(const float* centroids, int K, int d, int metric, const uint64_t* part_offsets,
                      const uint8_t* codes, const uint64_t* row_ids, float r2, const float* queries,
                      const uint8_t* qcodes, uint64_t nq, int k, int nprobes, uint64_t* out_ids, float* out_dists,
                      uint32_t* out_counts, const ScanFilter& flt, const ProbeRule* pr) {
  if (nq == 0 || k == 0) return;
  if (k > 1024) fail(LB2_UNSUPPORTED, "k (incl. refine factor) > 1024 is not implemented");
  const size_t smem = (size_t)(d + 15) / 16 * 16 + slot_smem_bytes(k);
  auto with_kernel = [&](auto f) {
    const bool vec4 = d % 16 == 0;
    if (metric == METRIC_DOT) {
      if (vec4) f(ivfsq_scan_kernel<METRIC_DOT, true>); else f(ivfsq_scan_kernel<METRIC_DOT, false>);
    } else {  // cosine: L2 on the normalised vectors' codes (sq/storage.rs:436-440)
      if (vec4) f(ivfsq_scan_kernel<METRIC_L2, true>); else f(ivfsq_scan_kernel<METRIC_L2, false>);
    }
  };
  size_t need = 0;
  with_kernel([&](auto kern) { need = smem_with_static(kern, smem); });
  if (need > ctx().smem_optin) fail(LB2_UNSUPPORTED, "dimension %d too large for the SQ scan", d);
  run_ivf_search(centroids, K, d, metric, queries, nq, k, nprobes, part_offsets, flt, pr, out_ids, out_dists, out_counts,
             [&](uint64_t q0, uint64_t qn, int np, const uint64_t* offs, const uint32_t* pids, const float*, float* cd,
                 uint64_t* cid, uint32_t* ccnt) {
               with_kernel([&](auto kern) {
                 set_smem(kern, smem);
                 LB2_LAUNCH("sq_scan", kern, dim3(np, (unsigned)qn), 256, smem, qcodes + q0 * d, d, r2, pids, np,
                            offs, codes, row_ids, k, cd, cid, ccnt, flt);
               });
             });
}

bool rq_scan_fits(int code_dim, int k) {
  return smem_with_static(ivfrq_scan_kernel, rq_scan_smem_bytes(code_dim, k)) <= ctx().smem_optin;
}

void ivfrq_search_f32(const float* centroids, int K, int d, int metric, const float* rotation, int code_dim,
                      const uint64_t* part_offsets, const uint8_t* codes, const float* add, const float* scale,
                      const uint64_t* row_ids, const float* queries, uint64_t nq, int k, int nprobes,
                      uint64_t* out_ids, float* out_dists, uint32_t* out_counts, const ScanFilter& flt,
                      const ProbeRule* pr) {
  if (nq == 0 || k == 0) return;
  if (k > 1024) fail(LB2_UNSUPPORTED, "k (incl. refine factor) > 1024 is not implemented");
  if (!rq_scan_fits(code_dim, k))
    fail(LB2_UNSUPPORTED, "IVF_RQ: the tables of code_dim %d do not fit the scan's shared memory", code_dim);
  const size_t smem = rq_scan_smem_bytes(code_dim, k);
  const float sqrt_d = sqrtf((float)code_dim);  // (dim as f32 * num_bits as f32).sqrt(): the product is exact
  const int q_minus_one = metric != METRIC_L2;    // the storage's metric: cosine / dot -> dist_q_c - 1.0
  run_ivf_search(centroids, K, d, metric, queries, nq, k, nprobes, part_offsets, flt, pr, out_ids, out_dists, out_counts,
             [&](uint64_t q0, uint64_t qn, int np, const uint64_t* offs, const uint32_t* pids, const float* pdists,
                 float* cd, uint64_t* cid, uint32_t* ccnt) {
               // the (query, probe) residuals are rotated in groups of queries that keep both buffers near 256 MB
               const uint64_t per_q = (uint64_t)np * (d + code_dim) * sizeof(float);
               const uint64_t qc = std::max<uint64_t>(1, std::min<uint64_t>(qn, (256ull << 20) / per_q));
               DevBuf<float> res(qc * np * d), rot(qc * np * code_dim);
               set_smem(ivfrq_scan_kernel, smem);
               for (uint64_t a = 0; a < qn; a += qc) {
                 const uint64_t b = std::min(qc, qn - a);
                 LB2_LAUNCH("rq_query_residual", rq_query_residual_kernel, cdiv(b * np * d, 256), 256, 0,
                            queries + (q0 + a) * d, b, np, d, centroids, K, pids + a * np, res.p);
                 rq_rotate_f32(rotation, code_dim, d, res.p, b * np, rot.p);
                 LB2_LAUNCH("rq_scan", ivfrq_scan_kernel, dim3(np, (unsigned)b), 256, smem, rot.p, code_dim, sqrt_d,
                            q_minus_one, pids + a * np, pdists + a * np, np, offs, codes, add, scale, row_ids,
                            k, cd + a * np * k, cid + a * np * k, ccnt + a * np, flt);
               }
             });
}

// ------------------------------------------------------------------------------------------------
// refine: exact distances of k' = k * refine_factor candidates from the raw vectors, then the k
// best by (distance, row id)  (scanner.rs:2884-2905, flat.rs:95-148)
// ------------------------------------------------------------------------------------------------
// The refine plan takes the distance function of the column's own element type (flat.rs:94-150), unlike the
// IVF_FLAT scan, whose storage is f32 (flat/storage.rs:352-365):
//  * f16 dot: dot_scalar::<f16, f32, 32> (dot.rs:30-58,133): lane l owns the accumulators l and l + 16, the d % 32
//    tail comes first, the 32 sums are folded 0..31;
//  * u8 L2 / dot: exact integer sums, one conversion to f32 (l2.rs:44-49, dot.rs:152-161); the query came in as
//    u8 too, so its f32 view holds integers;
//  * everything else (f16 L2, bf16, cosine) as flat_row_distance.
template <int METRIC, class T>
__device__ __forceinline__ float refine_row_distance(const float* __restrict__ q, const T* __restrict__ v, int d,
                                                     int l, unsigned mask, float q_norm) {
  if constexpr (std::is_same<T, uint8_t>::value && METRIC != METRIC_COSINE) {
    uint32_t acc = 0;
    for (int e = l; e < d; e += 16) {
      const int x = __float2int_rn(q[e]), y = v[e];
      acc += METRIC == METRIC_DOT ? (uint32_t)(x * y) : (uint32_t)((x - y) * (x - y));
    }
#pragma unroll
    for (int off = 8; off >= 1; off >>= 1) acc += __shfl_xor_sync(mask, acc, off, 16);
    return finish<METRIC>(__uint2float_rn(acc));
  } else if constexpr (std::is_same<T, __half>::value && METRIC == METRIC_DOT) {
    const int n32 = d & ~31;
    float a0 = 0.0f, a1 = 0.0f;
    for (int e = l; e < n32; e += 32) {
      a0 = f_add(a0, __fmul_rn(q[e], ldf<T>(v, e)));
      a1 = f_add(a1, __fmul_rn(q[e + 16], ldf<T>(v, e + 16)));
    }
    float s = 0.0f;  // sequential tail, every lane redundantly
    for (int e = n32; e < d; ++e) s = f_add(s, __fmul_rn(q[e], ldf<T>(v, e)));
    float t = 0.0f;
#pragma unroll
    for (int qq = 0; qq < 16; ++qq) t = f_add(t, __shfl_sync(mask, a0, qq, 16));
#pragma unroll
    for (int qq = 0; qq < 16; ++qq) t = f_add(t, __shfl_sync(mask, a1, qq, 16));
    return finish<METRIC>(f_add(s, t));
  } else {
    return flat_row_distance<METRIC, T>(q, v, d, l, mask, q_norm);
  }
}

template <int METRIC, class T>
__global__ void __launch_bounds__(256)
refine_kernel(const float* __restrict__ queries, int d, const T* __restrict__ vectors,
              uint64_t num_vectors, const uint64_t* __restrict__ cand_id, const uint32_t* __restrict__ cand_cnt,
              int kc, int k, uint64_t* __restrict__ out_id, float* __restrict__ out_d,
              uint32_t* __restrict__ out_cnt, int has_lower, float lower, int has_upper, float upper) {
  extern __shared__ float smem[];
  float* qs = smem;       // [d]
  float* cd = qs + d;     // [kc]
  __shared__ float s_qnorm;
  const size_t qi = blockIdx.x;
  const int tid = threadIdx.x, l = tid & 15;
  const unsigned hmask = 0xffffu << (16 * ((tid >> 4) & 1));
  const uint32_t cnt = min(cand_cnt[qi], (uint32_t)kc);
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
  const uint64_t* ids = cand_id + qi * kc;
  for (uint32_t c = tid >> 4; c < cnt; c += 16) {
    const uint64_t id = ids[c];
    float dist = __int_as_float(0x7fc00000);
    if (id < num_vectors) dist = refine_row_distance<METRIC, T>(qs, vectors + id * (uint64_t)d, d, l, hmask, qn);
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
        out_id[qi * k + r] = id;
        out_d[qi * k + r] = cd[c];
      });
  for (uint32_t e = r + tid; e < (uint32_t)k; e += 256) {
    out_id[qi * k + e] = ~0ull;
    out_d[qi * k + e] = __int_as_float(0x7f800000);
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
    auto kern = refine_kernel<decltype(m)::value, T>;
    set_smem(kern, smem);
    LB2_LAUNCH("refine", kern, (unsigned)nq, 256, smem, queries, d, reinterpret_cast<const T*>(vectors), num_vectors,
               cand_id, cand_cnt, kc, k, out_id, out_d, out_cnt, has_lower, lower, has_upper, upper);
  });
}

void build_lut_f32(const float* codebook, int M, int nbits, int d, int metric, const float* query,
                   float* lut) {
  const int ncode = 1 << nbits, ds = d / M;
  if (metric == METRIC_DOT)
    LB2_LAUNCH("build_lut", build_lut_kernel<METRIC_DOT>, cdiv((uint64_t)M * ncode, 128), 128, 0,
               codebook, M, ncode, ds, query, lut);
  else
    LB2_LAUNCH("build_lut", build_lut_kernel<METRIC_L2>, cdiv((uint64_t)M * ncode, 128), 128, 0,
               codebook, M, ncode, ds, query, lut);
}

void pq_scan_transposed_f32(const float* lut, int M, int metric, const uint8_t* codes_t, uint64_t n,
                            float* out) {
  if (n == 0) return;
  const size_t smem = sizeof(float) * (size_t)M * 256;
  if (smem > ctx().smem_optin) fail(LB2_UNSUPPORTED, "LUT of %zu bytes exceeds shared memory", smem);
  set_smem(pq_scan_transposed_kernel, smem);
  LB2_LAUNCH("pq_scan_transposed", pq_scan_transposed_kernel, cdiv(n, 256), 256, smem, lut, M,
             codes_t, n, metric == METRIC_DOT ? 1 : 0, out);
}

// ------------------------------------------------------------------------------------------------
// a19  4-bit PQ scan: compute_pq_distance_4bit (pq/distance.rs:147-242).  lut = M x 16 f32, codes_t =
// transposed packed codes [M/2][n] (low nibble = sub-vector 2i, high nibble = 2i+1).
//   rows [0, flat_num) and the last n % 16 rows: exact f32, two adds per byte in byte order;
//   the others: saturating u8 sum of the table quantised with qmin = min(table), qmax = max of the
//   flat rows (total order), then q * ((qmax - qmin) / 255) + qmin.
// ------------------------------------------------------------------------------------------------
__global__ void pq4_flat_kernel(const float* __restrict__ lut, int nb, const uint8_t* __restrict__ codes_t,
                                uint64_t n, uint64_t off, uint64_t len, float* __restrict__ out) {
  const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= len) return;
  const uint64_t j = off + t;
  float dist = 0.0f;
  for (int i = 0; i < nb; ++i) {
    const uint8_t c = codes_t[(size_t)i * n + j];
    dist = f_add(dist, lut[(2 * i) * 16 + (c & 0xF)]);
    dist = f_add(dist, lut[(2 * i + 1) * 16 + (c >> 4)]);
  }
  out[j] = dist;
}
// one block: qmax over the flat rows (total order), qmin over the table (f32::min ignores NaN), the u8 table
__global__ void pq4_quantize_kernel(const float* __restrict__ lut, int M, const float* __restrict__ flat,
                                    uint64_t flat_num, uint8_t* __restrict__ qt, float* __restrict__ params) {
  __shared__ int32_t s_max[256];
  __shared__ float s_min[256];
  pq4_quantize(lut, M, flat_num, [&](uint64_t j) { return flat[j]; }, qt, params, s_max, s_min);
}
__global__ void pq4_quant_scan_kernel(const uint8_t* __restrict__ qt, int nb, const uint8_t* __restrict__ codes_t,
                                      uint64_t n, uint64_t begin, uint64_t end,
                                      const float* __restrict__ params, float* __restrict__ out) {
  extern __shared__ uint8_t s_qt[];
  for (int i = threadIdx.x; i < nb * 32; i += blockDim.x) s_qt[i] = qt[i];
  __syncthreads();
  const uint64_t j = begin + (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= end) return;
  uint32_t q = 0;  // saturating u8 adds of non-negative terms == min(255, sum)
  for (int i = 0; i < nb; ++i) {
    const uint8_t c = codes_t[(size_t)i * n + j];
    q += s_qt[(2 * i) * 16 + (c & 0xF)];
    q += s_qt[(2 * i + 1) * 16 + (c >> 4)];
  }
  q = min(q, 255u);
  out[j] = pq4_dequantize(q, params);
}
__global__ void sub_scalar_kernel(float* __restrict__ v, uint64_t n, float s) {
  const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j < n && v[j] == v[j]) v[j] = __fsub_rn(v[j], s);  // a NaN passes through (see x86_nan)
}
void pq_scan_4bit_f32(const float* lut, int M, int metric, const uint8_t* codes_t, uint64_t n, uint64_t k_hint,
                      float* out) {
  if (n == 0) return;
  const int nb = M / 2;
  k_hint = std::min<uint64_t>(k_hint, n);
  const uint64_t flat_num = std::min<uint64_t>(std::max<uint64_t>(200, k_hint), n);  // FLAT_NUM_4BIT_PQ = 200
  const uint64_t rem = n % 16;
  LB2_LAUNCH("pq4_flat", pq4_flat_kernel, cdiv(flat_num, 256), 256, 0, lut, nb, codes_t, n, (uint64_t)0, flat_num, out);
  DevBuf<uint8_t> qt((size_t)M * 16);
  DevBuf<float> params(2);
  LB2_LAUNCH("pq4_quantize", pq4_quantize_kernel, 1, 256, 0, lut, M, (const float*)out, flat_num, qt.p, params.p);
  if (n - rem > flat_num)
    LB2_LAUNCH("pq4_scan", pq4_quant_scan_kernel, cdiv(n - rem - flat_num, 256), 256, (size_t)M * 16, qt.p, nb,
               codes_t, n, flat_num, n - rem, params.p, out);
  if (rem > 0) {
    const uint64_t off = std::max(n - rem, flat_num);
    if (n > off) LB2_LAUNCH("pq4_flat", pq4_flat_kernel, cdiv(n - off, 256), 256, 0, lut, nb, codes_t, n, off, n - off, out);
  }
  if (metric == METRIC_DOT)
    LB2_LAUNCH("pq4_dot_fix", sub_scalar_kernel, cdiv(n, 256), 256, 0, out, n, (float)M - 1.0f);
  sync_stream();  // qt / params are freed on return
}

// two 4-bit codes per byte: (v[1] << 4) | v[0]  (pq.rs:168-173)
__global__ void pack_nibbles_kernel(const uint8_t* __restrict__ codes, uint64_t total_bytes, uint8_t* __restrict__ out) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < total_bytes) out[i] = (uint8_t)((codes[2 * i + 1] << 4) | (codes[2 * i] & 0xF));
}
void pack_nibbles(const uint8_t* codes, uint64_t n, int M, uint8_t* out) {
  const uint64_t total = n * (uint64_t)(M / 2);
  if (total) LB2_LAUNCH("pack_nibbles", pack_nibbles_kernel, cdiv(total, 256), 256, 0, codes, total, out);
}

void flat_topk_f32(const float* dists, const uint64_t* row_ids, uint64_t n, int k, const ScanFilter& flt,
                   uint64_t* out_id, float* out_d, uint32_t* out_cnt) {
  if (k > 1024) fail(LB2_UNSUPPORTED, "k > 1024 is not implemented");
  LB2_LAUNCH("flat_topk", flat_topk_kernel, 1, 256, slot_smem_bytes(k), dists, row_ids, n, k, flt, out_id, out_d, out_cnt);
}

}  // namespace lb2
