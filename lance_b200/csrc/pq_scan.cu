// pq_scan.cu -- the IVF_PQ query path: lookup tables, the three partition scans (radix, classic, skew), the skewed
// code layout, and the stand-alone PQ primitives.
//
// Replaces  IVFIndex::preprocess_query           rust/lance/src/index/vector/ivf/v2.rs:316-332
//           build_distance_table_l2/_dot         lance-index/src/vector/pq/distance.rs:24-92
//           compute_pq_distance (+ Dot fix-up)   pq/distance.rs:109-144, pq/storage.rs:921-962
//
// One CTA per (query, probed partition): the residual query and its M x 256 f32 lookup table are
// built in shared memory (never written to HBM), the partition's codes are streamed once with
// 128-bit loads, each row's distance is the reference's m-ascending f32 sum (bit-exact), and
// warp-level sorting networks (k <= 16) or a block radix select produce the k smallest (distance,
// position) pairs.
#include <algorithm>
#include <type_traits>
#include <vector>

#include "common.cuh"
#include "exact.cuh"
#include "ivf_search.cuh"
#include "pq_lut.cuh"
#include "scan.cuh"
#include "topk.cuh"

namespace lb2 {

// ------------------------------------------------------------------------------------------------
// the fused (residual query -> LUT -> code scan -> top-k) kernels: one CTA per (query, probed
// partition).  Partitions are processed in chunks of <= SCAN_CHUNK rows, the winners of a chunk
// joining the next chunk's candidate pool.
// ------------------------------------------------------------------------------------------------

// arguments shared by the fused scan kernels (one slot = one (query, probed partition) pair)
struct ScanArgs {
  const float* queries; int d; const float* centroids; const float* codebook; int M, ds;
  const uint32_t* probe_ids; int np; const uint64_t* part_offsets; const uint8_t* codes;
  const uint64_t* row_ids; int k; float* cand_d; uint64_t* cand_id; uint32_t* cand_cnt;
  ScanFilter flt;
  const QueryParam* qp;  // per-query k' and filter of the slab's queries (k is then the lists' stride), or null
  // the (slab-relative) queries a launch covers, one route's group of a batch: grid row / slot group g is query
  // qlist[g]; null: every query of the slab
  const uint32_t* qlist = nullptr;
};

// the residual query of partition p (v2.rs:316-332) and its LUT, in shared memory (256 threads)
template <int METRIC, int NBITS>
__device__ __forceinline__ void stage_query_lut(float* lut, float* qr, const ScanArgs& a, size_t qi, uint32_t p) {
  const float* q = a.queries + qi * a.d;
  for (int t = threadIdx.x; t < a.d; t += 256)
    qr[t] = METRIC == METRIC_DOT ? q[t] : __fsub_rn(q[t], a.centroids[(size_t)p * a.d + t]);
  __syncthreads();
  build_lut<METRIC, NBITS>(lut, qr, a.codebook, a.M, a.ds, threadIdx.x);
  __syncthreads();
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

// BATCH: the slot's query's k' and filter come from a.qp; the single-parameter scan is compiled without the lookup
template <int METRIC, int NBITS, bool BATCH>
__device__ void radix_slot(const ScanArgs& a, size_t slot, bool replay) {
  extern __shared__ float smem[];
  const int M = a.M, d = a.d, np = a.np;
  float* lut = smem;                         // [M*16] (4-bit) or [M*256] (8-bit)
  float* qr = lut + M * (NBITS == 4 ? 16 : 256);  // [d]
  const int tid = threadIdx.x;
  const int pi = (int)(slot % np);
  const size_t qi = slot / np;
  const int k = BATCH ? a.qp[qi].k : a.k;  // a.k: the lists' stride
  const ScanFilter& flt = BATCH ? a.qp[qi].flt : a.flt;
  const SlotSmem s(qr + d, k + 1);
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
  if (NBITS == 4 && flt.allow == nullptr)  // the selection's (still unused) key buffer is the scratch
    pq4_quantize(lut, M, flat_num, exact4, qt, s_q, reinterpret_cast<int32_t*>(s.ukey),
                 reinterpret_cast<float*>(s.ukey + 256));
  auto fill = [&](uint32_t c0, uint32_t clen) {
    for (uint32_t j = tid; j < clen; j += 256) {
      const uint32_t row = c0 + j;
      float dist;
      if constexpr (NBITS == 4) {
        if (flt.allow != nullptr || row < flat_num || row >= n_p - rem16) {
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
  const uint32_t cnt = slot_topk(s, n_p, k, flt, off, replay, fill);
  write_slot(s, cnt, slot, a.k, off, a.row_ids, a.cand_d, a.cand_id, a.cand_cnt);
}

// grid (np, nq): one CTA per slot; or, with a replay list (slots the fast kernel could not settle because of
// ties at the k-th distance), a small persistent grid that replays the listed slots
template <int METRIC, int NBITS, bool BATCH = false>
__global__ void __launch_bounds__(256)
ivfpq_scan_radix_kernel(const ScanArgs a, const uint32_t* __restrict__ rlist, const uint32_t* __restrict__ rcount) {
  if (rlist) {
    const uint32_t cnt = *rcount;
    for (uint32_t i = blockIdx.x; i < cnt; i += gridDim.x) {
      radix_slot<METRIC, NBITS, BATCH>(a, rlist[i], true);
      __syncthreads();
    }
    return;
  }
  radix_slot<METRIC, NBITS, BATCH>(a, (size_t)(a.qlist ? a.qlist[blockIdx.y] : blockIdx.y) * a.np + blockIdx.x, false);
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
// k: the slot's query's k' (the lists' stride is a.k)
__device__ __forceinline__ void fast_slot_epilogue(const ScanArgs& a, int k, uint32_t slot, uint64_t off,
                                                   const uint64_t* win, uint32_t nw, bool replay, int t, int nt,
                                                   uint32_t* rlist, uint32_t* rcount) {
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
    a.cand_d[(size_t)slot * a.k + i] = key_to_float(cand_key(win[i]));
    a.cand_id[(size_t)slot * a.k + i] = a.row_ids[off + cand_pos(win[i])];
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
  const int M = a.M, np = a.np;
  float* lut = smem;          // [M*256]
  float* qr = lut + M * 256;  // [d]
  __shared__ uint64_t wl[8][SCAN_WLIST];                 // per-warp compacted candidates
  __shared__ uint64_t fin[8 * SCAN_KFAST + SCAN_KFAST];  // 8 x kk warp winners, then the carried winners
  __shared__ uint64_t car[SCAN_KFAST];
  __shared__ uint32_t s_nw;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  size_t qi, slot;
  uint32_t p, n_p;
  uint64_t off;
  if (!slot_partition(a.probe_ids, np, a.part_offsets, a.cand_cnt, qi, slot, p, off, n_p, a.qlist)) return;
  const int k = query_k(a.qp, qi, a.k);  // a.k: the lists' stride
  const int kk = k + 1;  // <= SCAN_KFAST: one more than asked for, to expose ties that overflow the k-th place
  const ScanFilter flt = query_filter(a.qp, qi, a.flt);
  const uint64_t* __restrict__ allow = flt.allow;
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
        if (!FILTER || key_in_range(flt, kv)) {
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
  fast_slot_epilogue(a, k, (uint32_t)slot, off, car, s_nw, false, tid, 256, rlist, rcount);
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
  const int d = a.d, np = a.np;
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
      const uint32_t rs = a.qlist ? a.qlist[slot / np] * np + slot % np : slot;
      rlist[atomicAdd(rcount, 1u)] = rs;
      a.cand_cnt[rs] = 0;
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
  // slot v of the launch is slot real(v) of the slab (a group's queries: qlist)
  auto real = [&](uint32_t v) -> uint32_t { return a.qlist ? a.qlist[v / np] * np + v % np : v; };
  uint32_t slot = blockIdx.x * NTEAM + team;
  uint32_t p_n = slot < nslots ? a.probe_ids[real(slot)] : 0u;
  uint64_t off_n = a.part_offsets[p_n], end_n = a.part_offsets[p_n + 1], so_n = slab_off[p_n];
  for (; slot < nslots; slot += stride) {
    const uint32_t rs = real(slot);
    const size_t qi = rs / np;
    const int k = query_k(a.qp, qi, a.k);  // a.k: the lists' stride
    const int kk = k + 1;  // one more than asked for, to expose ties that overflow the k-th place
    const ScanFilter flt = query_filter(a.qp, qi, a.flt);
    const uint64_t* __restrict__ allow = flt.allow;
    const uint32_t p = p_n;
    const uint64_t off = off_n;
    const uint32_t n_p = (uint32_t)(end_n - off_n);
    const uint8_t* sp = skew + so_n * SKEW_SLAB_BYTES;
    p_n = slot + stride < nslots ? a.probe_ids[real(slot + stride)] : 0u;
    if (n_p == 0) {
      off_n = a.part_offsets[p_n]; end_n = a.part_offsets[p_n + 1]; so_n = slab_off[p_n];
      if (ttid == 0) a.cand_cnt[rs] = 0;
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
            live = ri >= 0 && ri < 16 && j < clen && row_allowed(allow, off + c0 + j) && key_in_range(flt, kv);
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
    fast_slot_epilogue(a, k, rs, off, car + par * SCAN_KFAST, nw, replay, ttid, TT, rlist, rcount);
  }
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

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
// which fast kernel serves an 8-bit scan: LB2_SCAN=classic|skew overrides the size rule (tests run both)
static int scan_mode_env() {
  const char* e = getenv("LB2_SCAN");
  return !e ? 0 : (!strcmp(e, "classic") ? 1 : (!strcmp(e, "skew") ? 2 : 0));
}

// the radix kernel, with per-query values when the search has them
template <int METRIC, int NBITS>
static void radix_launch(const char* name, dim3 grid, size_t smem, const ScanArgs& a, const uint32_t* rlist,
                         const uint32_t* rcount) {
  auto go = [&](auto kern) {
    set_smem(kern, smem);
    LB2_LAUNCH(name, kern, grid, 256, smem, a, rlist, rcount);
  };
  if (a.qp) go(ivfpq_scan_radix_kernel<METRIC, NBITS, true>);
  else go(ivfpq_scan_radix_kernel<METRIC, NBITS, false>);
}

// one launch of the fast 8-bit scan (k' + 1 <= SCAN_KFAST) over grid (probes, queries); ties go to rlist
template <int METRIC>
static void fast_launch(dim3 grid, const ScanArgs& a, bool filtering, uint32_t* rlist, uint32_t* rcount,
                        const uint64_t* slab_off, const uint8_t* skew) {
  {
    const size_t smem_fast = sizeof(float) * ((size_t)a.M * 256 + a.d);
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
  }
}

// slots with ties beyond the k-th place (rare): the reference's heap loop, restated, over the listed slots
template <int METRIC>
static void tie_replay(uint64_t nslots, size_t smem, ScanArgs a, const uint32_t* rlist, const uint32_t* rcount) {
  a.qlist = nullptr;  // the list holds slots of the slab
  const unsigned rgrid = (unsigned)std::min<uint64_t>(nslots, 4 * (uint64_t)ctx().num_sms);
  radix_launch<METRIC, 8>("pq_scan_tie_replay", rgrid, smem, a, rlist, rcount);
}

template <int METRIC>
static void scan_launch(int nbits, dim3 grid, size_t smem, const ScanArgs& a, bool filtering, uint32_t* rlist,
                        uint32_t* rcount, const uint64_t* slab_off, const uint8_t* skew) {
  if (nbits == 8 && a.k + 1 <= SCAN_KFAST) {
    LB2_CUDA(cudaMemsetAsync(rcount, 0, sizeof(uint32_t), ctx().stream));
    fast_launch<METRIC>(grid, a, filtering, rlist, rcount, slab_off, skew);
    tie_replay<METRIC>((uint64_t)grid.x * grid.y, smem, a, rlist, rcount);
    return;
  }
  if (nbits == 4)
    radix_launch<METRIC, 4>("pq_scan", grid, smem, a, nullptr, nullptr);
  else
    radix_launch<METRIC, 8>("pq_scan", grid, smem, a, nullptr, nullptr);
}

// A batch's slab (queries with their own k' and filter): its queries in route groups -- the fast kernel without and
// with the filter test (k' + 1 <= SCAN_KFAST, 8-bit), the radix kernel for the others -- and one launch per group
// present, each over its own queries (qlist), then one tie replay for both fast groups.  groups[r] lists route r's
// slab-relative queries on the host, glist holds them on the device in that order.
template <int METRIC>
static void scan_launch_groups(int np, size_t smem, ScanArgs a, const std::vector<uint32_t>* groups,
                               const uint32_t* glist, uint32_t* rlist, uint32_t* rcount, const uint64_t* slab_off,
                               const uint8_t* skew) {
  const size_t nfast = groups[0].size() + groups[1].size();
  if (nfast) LB2_CUDA(cudaMemsetAsync(rcount, 0, sizeof(uint32_t), ctx().stream));
  size_t at = 0;
  for (int r = 0; r < 3; ++r) {
    const size_t n = groups[r].size();
    if (!n) continue;
    a.qlist = glist + at;
    at += n;
    const dim3 g((unsigned)np, (unsigned)n);
    if (r < 2) fast_launch<METRIC>(g, a, r == 1, rlist, rcount, slab_off, skew);
    else radix_launch<METRIC, 8>("pq_scan", g, smem, a, nullptr, nullptr);
  }
  if (nfast) tie_replay<METRIC>((uint64_t)nfast * np, smem, a, rlist, rcount);
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

void ivfpq_search(const IvfSearch& s, const float* codebook, int M, int nbits, const uint8_t* codes,
                  const uint64_t* slab_off, const uint8_t* skew) {
  if (s.nq == 0 || s.k == 0) return;  // an empty search refuses nothing, a shape included
  if (nbits != 8 && nbits != 4) fail(LB2_INVALID_ARG, "PQ: num_bits must be 4 or 8, got %d", nbits);
  if (nbits == 4 && (M % 2 != 0 || M > 256)) fail(LB2_UNSUPPORTED, "4-bit PQ needs an even num_sub_vectors <= 256");
  const int d = s.d, k = s.k, metric = s.metric;
  const int np = s.nprobes < s.K ? s.nprobes : s.K;
  const size_t smem = sizeof(float) * ((size_t)M * (nbits == 4 ? 16 : 256) + d) + slot_smem_bytes(k);
  // every kernel the scan may launch must fit: the radix kernel (the scan itself, or the tie replay of the fast
  // 8-bit kernels) and, for k + 1 <= SCAN_KFAST (a batch: any query's k'), the classic fast kernel with its LUT and
  // larger static lists
  bool any_fast = k + 1 <= SCAN_KFAST;
  for (uint64_t q = 0; s.qp_host && q < s.nq && !any_fast; ++q) any_fast = s.qp_host[q].k + 1 <= SCAN_KFAST;
  size_t need = 0;
  auto need_of = [&](auto m) {
    constexpr int METRIC = decltype(m)::value;
    need = nbits == 4 ? smem_with_static(ivfpq_scan_radix_kernel<METRIC, 4>, smem)
                      : smem_with_static(ivfpq_scan_radix_kernel<METRIC, 8>, smem);
    if (nbits == 8 && any_fast) {
      const size_t fast = sizeof(float) * ((size_t)M * 256 + d);
      const bool filtering = s.filtering();
      need = std::max(need, filtering ? smem_with_static(ivfpq_scan_kernel<METRIC, true>, fast)
                                      : smem_with_static(ivfpq_scan_kernel<METRIC, false>, fast));
    }
  };
  if (metric == METRIC_DOT) need_of(std::integral_constant<int, METRIC_DOT>{});
  else need_of(std::integral_constant<int, METRIC_L2>{});
  if (!ivf_search_begin(s, need, "LUT and top-k scratch of %zu bytes exceed shared memory", need)) return;
  DevBuf<uint32_t> rlist((size_t)std::min<uint64_t>(s.nq, SEARCH_SLAB) * np), rcount(1), glist;
  run_ivf_search(s, [&](const ScanSlots& sl) {
    if (rlist.n < sl.qn * sl.np) rlist.alloc(sl.qn * sl.np);
    const ScanArgs a{s.queries + sl.q0 * d, d, s.centroids, codebook, M, d / M, sl.probe_ids, sl.np, sl.offsets, codes,
                     s.row_ids, k, sl.cand_d, sl.cand_id, sl.cand_cnt, s.flt, s.qp_at(sl.q0)};
    if (s.qp_host && nbits == 8) {  // a batch: route groups (fast unfiltered, fast filtered, radix), one launch each
      std::vector<uint32_t> groups[3];
      for (uint32_t q = 0; q < (uint32_t)sl.qn; ++q) {
        const QueryParam& p = s.qp_host[sl.q0 + q];
        groups[p.k + 1 > SCAN_KFAST ? 2 : (p.flt.allow || p.flt.range ? 1 : 0)].push_back(q);
      }
      std::vector<uint32_t> all(groups[0]);
      all.insert(all.end(), groups[1].begin(), groups[1].end());
      all.insert(all.end(), groups[2].begin(), groups[2].end());
      if (glist.n < all.size()) glist.alloc(all.size());
      h2d(glist.p, all.data(), all.size());
      if (metric == METRIC_DOT)
        scan_launch_groups<METRIC_DOT>(sl.np, smem, a, groups, glist.p, rlist.p, rcount.p, slab_off, skew);
      else
        scan_launch_groups<METRIC_L2>(sl.np, smem, a, groups, glist.p, rlist.p, rcount.p, slab_off, skew);
      return;
    }
    const dim3 g(sl.np, (unsigned)sl.qn);
    if (metric == METRIC_DOT)
      scan_launch<METRIC_DOT>(nbits, g, smem, a, s.filtering(), rlist.p, rcount.p, slab_off, skew);
    else
      scan_launch<METRIC_L2>(nbits, g, smem, a, s.filtering(), rlist.p, rcount.p, slab_off, skew);
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

}  // namespace lb2
