// tc_pq.cu -- tensor-core FILTER + in-epilogue exact re-rank for PQ code assignment (8-wide
// sub-vectors, 256 codewords), sm_90a: wgmma tf32 + TMA + mbarrier.
//
// Replaces the inner loop of  ProductQuantizer::transform_impl  (lance-index/src/vector/pq.rs:116-191:
// per row, per sub-vector, argmin over the codebook via compute_partition kmeans.rs:1350-1369) and of
// the PQ training membership step (pq/builder.rs:89-157 -> kmeans.rs:317-369), bit for bit:
//
//   * B operand: the codebook as one K-major matrix Bm[c][m*8+t] = cb[m][c][t] (256 x d f32), resident
//     in shared memory for the whole kernel (TMA, SWIZZLE_128B).
//   * A operand: 64-row tiles of the (residual) vectors, TMA-streamed in 32-float chunks (= 4 sub-spaces).
//   * two wgmmas (M64 N128 K8, tf32: one per half of the codebook) per (tile, sub-space) into register
//     accumulators, consumer warpgroups taking the work items in turns (see Pipe); the epilogue keeps the
//     top-3 of  r.c - |c|^2/2  over the 128 codeword PAIRS (c, c ^ 1) of the row (tc_common.cuh: column units) and
//     classifies the row against tau = 3*2^-10 (|r_m|^2 + max|c_m|^2) (with the norm floor of cert_tau) like
//     tc_assign.cu: flag 0 certifies the two codewords of the best pair, flag 1 the four of the two best;
//   * the top 3 of each (row, sub-space) are parked in shared memory, and once an item's sub-spaces have been
//     through the tournament, one converged DECISION PASS per warp classifies its 16 rows x 4 sub-spaces (all
//     32 lanes, two pairs per lane): each certified codeword of a flag 0/1 pair gets the reference-order f32
//     distance from the operands still in shared memory (sequential 8-term sum, l2.rs:69-79; strict-< / lowest
//     index), as four independent chains; the item's stage is released after that pass;
//   * flag 2 (row, sub-space) pairs are appended to a list and finished by pq_fallback_kernel
//     (half-warp per pair, exact scan of all 256 codewords).
#include "assign.cuh"
#include "common.cuh"
#include "exact.cuh"
#include "tc_common.cuh"
#include "tc_pq.cuh"

namespace lb2 {
namespace tcpq {

using namespace tc;

constexpr int DS = 8;
constexpr int UNIT = 2;  // the tournament's entrants are column pairs (tc_common.cuh); decide() ranks their columns
constexpr int MAX_M_RESIDENT = 16;  // d <= 128: the whole codebook matrix stays in shared memory
constexpr int MAX_M = 256;          // d <= 2048: codebook chunk + its -|c|^2/2 slice streamed per work item
constexpr int CNH_CHUNK_BYTES = 4 * TN * 4;                                       // 4 sub-spaces
constexpr int STREAM_STAGE_BYTES = A_STAGE_BYTES + B_CHUNK_BYTES + CNH_CHUNK_BYTES;  // 44 KB

// One TMA producer warpgroup and CONSUMERS warpgroups that take the work items in turns.  The epilogue is bound by
// the ALU pipe (per 128 scores of a lane 64 pair maxima, 64 packs and about 210 min/max of the pair tournament,
// against 128 adds on the FMA pipe), and a consumer warp stalls often (wgmma waits, barrier waits, the shuffles of
// top3_finish); the resident variant runs four consumers (4 warps per scheduler) so that the others fill those
// stalls.  The decisions of an item run as one converged pass after its tournaments, with no MMA in flight: run
// under the next item's first MMA instead, the pass holds a second stage per consumer, and the ring's slack lost
// that way cost more than the overlap won (65 536-row training calls on an H100).  The streamed ring (44 KB per stage) has no room for more than four stages, so the streamed variant keeps two
// consumers.
// ACC_SETS: 64-register accumulator sets of a consumer.  With two, the tournament of one 128-codeword half runs
// while the MMA of the next is in flight; they do not fit the 112 registers of four consumers without spills,
// so there one half is computed at a time and the other warpgroups fill the MMA latency.
template <bool STREAM>
struct Pipe {
  static constexpr int CONSUMERS = STREAM ? 2 : 4;
  static constexpr int STAGES = STREAM ? 4 : 8;
  static constexpr int ACC_SETS = STREAM ? 2 : 1;
  static constexpr int THREADS = 128 * (1 + CONSUMERS);
  static constexpr int PRODUCER_REGS = STREAM ? 40 : 24;
  static constexpr int CONSUMER_REGS = STREAM ? 232 : 112;
  // every stage always serves the same warpgroup, so a stage is refilled only after its own consumer released it
  static_assert(STAGES % CONSUMERS == 0, "stages are dealt to the consumer warpgroups in turns");
  // setmaxnreg only moves registers between the warps of the CTA: the consumers can gain what the producer gives
  // up of the launch allocation (THREADS x the per-thread count that __launch_bounds__ leaves, a multiple of 8)
  static_assert(128 * (PRODUCER_REGS + CONSUMERS * CONSUMER_REGS) <= THREADS * ((65536 / THREADS) & ~7),
                "register file");
};

// The parked tournament results of one consumer warp: the top 3 of its 16 rows for the item's 4 sub-spaces, as
// [sub-space j][rank][row] (row-minor: the decision pass's half-warps read sub-spaces j and j + 2, 48 words apart,
// so that their 16 rows fall on distinct banks)
constexpr int PARK_WARP_FLOATS = 4 * 3 * 16;  // 768 B
constexpr uint32_t SMEM_OPTIN = 227 * 1024;   // H100: the opt-in dynamic shared memory of one block

// RESIDENT: [B: nkc x 32 KB][A ring: STAGES x 8 KB][cnh: M x 1 KB][bars][cbm][misc][park: 4 CONSUMERS x 768 B]
// STREAM:   [ring: STAGES x (A 8 KB | B chunk 32 KB | cnh slice 4 KB)][bars][cbm][misc][park]
struct Layout {
  uint32_t b_off, a_off, cnh_off, bar_off, cbm_off, misc_off, park_off, total;
  uint32_t stage_bytes;  // distance between two A stages
};
__host__ __device__ constexpr Layout layout(int nkc, int M, bool stream) {
  Layout L{};
  if (stream) {
    L.b_off = A_STAGE_BYTES;                  // + s * stage_bytes
    L.a_off = 0;                              // + s * stage_bytes
    L.cnh_off = A_STAGE_BYTES + B_CHUNK_BYTES;  // + s * stage_bytes
    L.stage_bytes = STREAM_STAGE_BYTES;
    L.bar_off = Pipe<true>::STAGES * STREAM_STAGE_BYTES;
  } else {
    L.b_off = 0;
    L.a_off = nkc * B_CHUNK_BYTES;
    L.cnh_off = L.a_off + Pipe<false>::STAGES * A_STAGE_BYTES;
    L.stage_bytes = A_STAGE_BYTES;
    L.bar_off = L.cnh_off + M * TN * 4;
  }
  static_assert((2 * Pipe<false>::STAGES + 1) * 8 <= 256 && (2 * Pipe<true>::STAGES + 1) * 8 <= 256, "barriers");
  L.cbm_off = L.bar_off + 256;              // max_c |c|^2 per sub-space
  L.misc_off = L.cbm_off + MAX_M * 4;
  L.park_off = L.misc_off + MAX_M;  // after one "active" byte per sub-space
  L.total = L.park_off + (stream ? Pipe<true>::CONSUMERS : Pipe<false>::CONSUMERS) * 4 * PARK_WARP_FLOATS * 4;
  return L;
}
// the largest shape of each variant, with the 1 KB that aligning the base to 1024 may take (tc_pq_assign)
static_assert(layout(MAX_M_RESIDENT / 4, MAX_M_RESIDENT, false).total + 1024 <= SMEM_OPTIN, "resident layout");
static_assert(layout(MAX_M / 4, MAX_M, true).total + 1024 <= SMEM_OPTIN, "streamed layout");

// 1-D bulk copy global -> shared with mbarrier completion (the streamed -|c|^2/2 slice)
__device__ __forceinline__ void bulk_load_1d(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}

// physical address of the 16-byte unit `u` (0..7) of row `r` inside a [rows x 128 B] SWIZZLE_128B tile
__device__ __forceinline__ const float4* swz(const uint8_t* tile, int r, int u) {
  return reinterpret_cast<const float4*>(tile + (r >> 3) * 1024 + (r & 7) * 128 + ((u ^ (r & 7)) << 4));
}

// Work items = (64-row tile, 32-float chunk = 4 sub-spaces), finer than whole tiles so that the persistent CTAs
// (one per SM) stay balanced on short inputs (65 536-row training calls: 1024 tiles).  The consumer warpgroups
// take the items with an active sub-space in turns (see Pipe).
template <bool TRAIN, bool STREAM>
__global__ void __launch_bounds__(Pipe<STREAM>::THREADS, 1)
tc_pq_kernel(const __grid_constant__ CUtensorMap map_r, const __grid_constant__ CUtensorMap map_b,
             uint64_t n, int M, const float* __restrict__ cnh_g, const float* __restrict__ cbmax2,
             const float* __restrict__ rn2, const uint8_t* __restrict__ row_valid,
             uint8_t* __restrict__ codes, uint32_t* __restrict__ ids, float* __restrict__ dists,
             uint8_t* __restrict__ valid, uint32_t* __restrict__ fb_pairs,
             uint32_t* __restrict__ fb_count, const uint8_t* __restrict__ active) {
  using P = Pipe<STREAM>;
  constexpr int STAGES = P::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_align1024(smem_raw);
  const int nkc = M / 4;
  const Layout L = layout(nkc, M, STREAM);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L.bar_off);
  uint8_t* act_s = smem + L.misc_off;  // [M] 0/1 (M % 4 == 0: read as one word per chunk)
  float* cbm_s = reinterpret_cast<float*>(smem + L.cbm_off);  // [M]
  const uint32_t sb = smem_u32(smem);
  auto full_bar = [&](int s) { return smem_u32(&bars[s]); };
  auto empty_bar = [&](int s) { return smem_u32(&bars[STAGES + s]); };
  const uint32_t b_full = smem_u32(&bars[2 * STAGES]);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint64_t num_tiles = (n + TM - 1) / TM;

  if (!STREAM) {
    float* cnh = reinterpret_cast<float*>(smem + L.cnh_off);
    for (int i = threadIdx.x; i < M * TN; i += P::THREADS) cnh[i] = cnh_g[i];
  }
  int any_active = 0;
  for (int m = threadIdx.x; m < M; m += P::THREADS) {
    const uint8_t a = (!active || active[m]) ? 1 : 0;
    act_s[m] = a;
    cbm_s[m] = cbmax2[m];
    any_active |= a;
  }
  if (threadIdx.x == 32) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 4);  // the 4 warps of the consumer (they re-read the operands after the MMAs)
    }
    mbar_init(b_full, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  any_active = __syncthreads_or(any_active);
  if (!any_active) return;  // uniform
  // bit j of chunk_mask(kc) = sub-space 4*kc + j still active
  auto chunk_mask = [&](int kc) -> uint32_t {
    const uint32_t w = reinterpret_cast<const uint32_t*>(act_s)[kc];
    return (w | (w >> 7) | (w >> 14) | (w >> 21)) & 0xFu;
  };

  if (warp < 4) {
    // ===== TMA producer =====
    setmaxnreg_dec<P::PRODUCER_REGS>();
    if (threadIdx.x == 0) {
      if (!STREAM) {
        mbar_expect_tx(b_full, (uint32_t)nkc * B_CHUNK_BYTES);
        for (int kc = 0; kc < nkc; ++kc)
          tma_load_2d(sb + L.b_off + kc * B_CHUNK_BYTES, &map_b, b_full, kc * KC, 0);
      }
      int s = 0;
      uint32_t ph = 0;
      for (uint64_t item = blockIdx.x; item < num_tiles * nkc; item += gridDim.x) {
        const uint64_t tile = item / nkc;
        const int kc = (int)(item % nkc);
        if (chunk_mask(kc) == 0) continue;  // chunk with no active sub-space
        mbar_wait_relaxed(empty_bar(s), ph ^ 1);
        mbar_expect_tx(full_bar(s), STREAM ? STREAM_STAGE_BYTES : A_STAGE_BYTES);
        tma_load_2d(sb + L.a_off + s * L.stage_bytes, &map_r, full_bar(s), kc * KC, (int)(tile * TM));
        if (STREAM) {
          tma_load_2d(sb + L.b_off + s * L.stage_bytes, &map_b, full_bar(s), kc * KC, 0);
          bulk_load_1d(sb + L.cnh_off + s * L.stage_bytes, cnh_g + (size_t)kc * 4 * TN, CNH_CHUNK_BYTES,
                       full_bar(s));
        }
        if (++s == STAGES) { s = 0; ph ^= 1; }
      }
    }
  } else {
    // ===== consumers: per active sub-space two wgmmas (K = 8, one per 128-codeword half) and the top-3
    // tournament; per item one converged decision pass (every lane works, fixed trip counts) =====
    // Each half is its own wgmma group.
    setmaxnreg_inc<P::CONSUMER_REGS>();
    const uint32_t w = (threadIdx.x >> 7) - 1;
    if (!STREAM) mbar_wait(b_full, 0);
    const int h = lane & 1;      // lanes 0 / 1 of the quad finish rows r0 / r0 + 8
    const int wrow = 16 * (warp & 3);  // the warp's 16 rows inside the tile
    float* park = reinterpret_cast<float*>(smem + L.park_off) + (warp - 4) * PARK_WARP_FLOATS;
    // decision pass: lane l decides row wrow + (l & 15) for sub-spaces dj + 2 d, d = 0, 1
    const int drow = lane & 15, dj = lane >> 4;
    // The flags, exact re-ranks and outputs of the item (tile, kc) in stage s for the warp's 16 rows and the item's
    // active sub-spaces, from the parked top 3; rn = |r_m|^2 of the lane's two pairs.  Releases the stage.
    auto decide_item = [&](uint32_t tile, int kc, int s, const float (&rn)[2]) {
      __syncwarp();  // the parked results of the other lanes
      const uint32_t cm = chunk_mask(kc);
      const uint8_t* atile = smem + L.a_off + s * L.stage_bytes;
      const uint8_t* bt = smem + L.b_off + (STREAM ? s * L.stage_bytes : kc * B_CHUNK_BYTES);
      const uint32_t row = tile * TM + wrow + drow;  // n < 2^32 (n * M < 2^32)
      const bool in = row < n;
      uint32_t code2 = 0;  // encode: the lane's two codes at their byte positions of the row's 4-code word
#pragma unroll
      for (int d = 0; d < 2; ++d) {
        const int j = dj + 2 * d, m = kc * 4 + j;
        const float* pk = park + j * 48 + drow;
        const float m1 = pk[0], m2 = pk[16], m3 = pk[32];
        const float tau = cert_tau(0.0029296875f, rn[d] + cbm_s[m]);
        // flag 0 certifies pair 1, flag 1 pairs 1 and 2; two pairs with the same score bits are duplicated
        // codewords: such rows keep their route through pq_fallback_kernel, which handles any multiplicity
        // (tests/test_assignment_routes.py pins the routes)
        const bool f0 = m1 - m2 > tau;
        const bool f1 = !f0 && m1 - m3 > tau && ((__float_as_uint(m1) ^ __float_as_uint(m2)) >> 8) != 0;
        const bool live = in && ((cm >> j) & 1u);
        // the low byte is a PAIR of columns (2p, 2p + 1), p < 128
        const uint32_t p1 = __float_as_uint(m1) & 0x7Fu, p2 = __float_as_uint(m2) & 0x7Fu;
        const uint32_t plo = f0 ? p1 : min(p1, p2), phi = max(p1, p2);
        // exact, reference-order distances of four columns as independent chains; in ascending column order the
        // certified ones (two under flag 0, four under flag 1) are ranked by strict < (the lowest index wins a tie)
        const float4 r0 = *swz(atile, wrow + drow, j * 2), r1 = *swz(atile, wrow + drow, j * 2 + 1);
        const float rv[8] = {r0.x, r0.y, r0.z, r0.w, r1.x, r1.y, r1.z, r1.w};
        float v[4];
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const int ci = (int)(2 * (c < 2 ? plo : phi) + (c & 1));
          const float4 c0v = *swz(bt, ci, j * 2), c1v = *swz(bt, ci, j * 2 + 1);
          const float cv[8] = {c0v.x, c0v.y, c0v.z, c0v.w, c1v.x, c1v.y, c1v.z, c1v.w};
          float sacc = 0.0f;
#pragma unroll
          for (int t = 0; t < 8; ++t) sacc = f_add(sacc, sq_diff(rv[t], cv[t]));
          v[c] = f_add(sacc, 0.0f);
        }
        float bv = __int_as_float(0x7f800000);
        uint32_t bi = 0xffffffffu;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const bool better_c = (c < 2 || !f0) && v[c] < bv;
          bv = better_c ? v[c] : bv;
          bi = better_c ? 2 * (c < 2 ? plo : phi) + (c & 1) : bi;
        }
        const bool ok = bi != 0xffffffffu, decided = live && (f0 || f1);
        if (TRAIN) {
          if (decided) {  // consecutive lanes: consecutive rows of one sub-space
            ids[(uint64_t)m * n + row] = ok ? bi : 0u;
            dists[(uint64_t)m * n + row] = ok ? bv : __int_as_float(0x7fc00000);
            valid[(uint64_t)m * n + row] = ok ? 1 : 0;
          }
        } else {
          // an undecided pair's byte is rewritten by pq_fallback_kernel
          code2 |= (ok ? bi & 0xFFu : 0u) << (8 * j);
        }
        // undecided pairs join sub-space m's list: one atomic per half-warp (= sub-space), ranks by popc.  Their
        // order inside the list is free: pq_fallback_kernel decides every listed pair on its own
        const uint32_t und = (__ballot_sync(0xffffffffu, live && !f0 && !f1) >> (16 * dj)) & 0xFFFFu;
        const int lead = und ? __ffs(und) - 1 : 0;
        uint32_t base = 0;
        if (und && drow == lead) base = atomicAdd(fb_count + m, (uint32_t)__popc(und));
        base = __shfl_sync(0xffffffffu, base, 16 * dj + lead);
        if ((und >> drow) & 1u) fb_pairs[(size_t)m * n + base + __popc(und & ((1u << drow) - 1))] = row;
      }
      if (!TRAIN) {
        // the row's four codes as one aligned word (codes is [n][M], M % 4 == 0); encode has every sub-space active
        const uint32_t word = code2 | __shfl_xor_sync(0xffffffffu, code2, 16);
        const bool rv_ok = in && (row_valid ? row_valid[row] != 0 : true);
        if (in && dj == 0) *reinterpret_cast<uint32_t*>(codes + row * (uint64_t)M + 4 * kc) = rv_ok ? word : 0u;
      }
      // this warp's pass has read the stage and the parked results
      __syncwarp();
      if (lane == 0) mbar_arrive(empty_bar(s));
    };
    float acc[P::ACC_SETS][64];
    uint32_t k = 0;  // ring index of the items with an active sub-space
    for (uint64_t item = blockIdx.x; item < num_tiles * nkc; item += gridDim.x) {
      const uint64_t tile = item / nkc;
      const int kc = (int)(item % nkc);
      const uint32_t cm = chunk_mask(kc);
      if (cm == 0) continue;
      const bool mine = k % P::CONSUMERS == w;
      const int s = (int)(k % STAGES);
      const uint32_t ph = (k / STAGES) & 1;
      ++k;
      if (!mine) continue;
      // |r_m|^2 of the lane's two decision pairs, fetched before the MMAs
      float rn[2] = {0.0f, 0.0f};
      {
        const uint64_t row = tile * TM + wrow + drow;
        if (row < n) {
          rn[0] = rn2[row * M + 4 * kc + dj];
          rn[1] = rn2[row * M + 4 * kc + dj + 2];
        }
      }
      mbar_wait(full_bar(s), ph);
      const uint8_t* bt = smem + L.b_off + (STREAM ? s * L.stage_bytes : kc * B_CHUNK_BYTES);
      const float* cn4 = reinterpret_cast<const float*>(smem + L.cnh_off + (STREAM ? s * L.stage_bytes : kc * CNH_CHUNK_BYTES));
      const uint32_t a_addr = smem_u32(smem + L.a_off + s * L.stage_bytes), b_addr = smem_u32(bt);
      // half `hf` of sub-space j into d: codewords 128 hf .. 128 hf + 127 are B rows 128 hf.. (128 B each)
      auto issue = [&](float* d, int j, int hf) {
        __syncwarp();  // wgmma is warp-aligned: reconverge after the barrier polls
        acc_fence<64>(d);
        wgmma_fence();
        wgmma_tf32_n128(d, make_desc(a_addr + j * 32), make_desc(b_addr + hf * (TN / 2) * 128 + j * 32), 0u);
        wgmma_commit();
      };
      uint32_t rest = cm;
      int j = __ffs(rest) - 1;
      rest &= rest - 1;
      issue(acc[0], j, 0);
      if constexpr (P::ACC_SETS == 2) issue(acc[1], j, 1);
      // the finished top 3 of sub-space j, row r0 + 8 (lane & 1): every lane of the quad holds it, and both lanes of
      // a row store it (the same value; no divergent code while the next sub-space's MMA is in flight)
      auto park_top3 = [&](int j, const float (&mm)[3]) {
        float* pk = park + j * 48 + (lane >> 2) + 8 * h;
        pk[0] = mm[0];
        pk[16] = mm[1];
        pk[32] = mm[2];
      };
      if constexpr (P::ACC_SETS == 2) {
        // the tournament of half 0 runs while half 1 is in flight, and that of half 1 while the next sub-space's
        // half 0, issued into the registers just read, is
        for (;;) {
          const int jn = rest ? __ffs(rest) - 1 : -1;  // next active sub-space of the item
          Tour tour;
          wgmma_wait<1>();
          acc_fence<64>(acc[0]);
          top3_half<0, UNIT>(acc[0], cn4 + j * TN, tour);
          if (jn >= 0) {
            issue(acc[0], jn, 0);
            wgmma_wait<1>();
          } else {
            wgmma_wait<0>();
          }
          acc_fence<64>(acc[1]);
          top3_half<1, UNIT>(acc[1], cn4 + j * TN, tour);
          float mm[3];
          top3_finish<UNIT>(tour, mm);
          wgmma_wait<0>();
          park_top3(j, mm);
          if (jn < 0) break;
          issue(acc[1], jn, 1);
          j = jn;
          rest &= rest - 1;
        }
      } else {
        // one half at a time, into the same registers
        for (;;) {
          Tour tour;
          wgmma_wait<0>();
          acc_fence<64>(acc[0]);
          top3_half<0, UNIT>(acc[0], cn4 + j * TN, tour);
          issue(acc[0], j, 1);
          wgmma_wait<0>();
          acc_fence<64>(acc[0]);
          top3_half<1, UNIT>(acc[0], cn4 + j * TN, tour);
          float mm[3];
          top3_finish<UNIT>(tour, mm);
          park_top3(j, mm);
          if (!rest) break;
          j = __ffs(rest) - 1;
          rest &= rest - 1;
          issue(acc[0], j, 0);
        }
      }
      // every MMA of the item has completed
      decide_item((uint32_t)tile, kc, s, rn);
    }
  }
}

// Bm[c][m*8+t] = cb[m][c][t];  cnh[m][c] = -|cb[m][c]|^2 / 2;  cbmax2[m] = max_c |cb[m][c]|^2
__global__ void __launch_bounds__(256)
prep_codebook_kernel(const float* __restrict__ cb, TcPqPrepArgs a) {
  __shared__ float s_n2[TN];
  const int m = blockIdx.x;  // grid M, block 256
  if (threadIdx.x == 0) a.fb_count[m] = 0;  // one undecided-row list per sub-space
  tc_pq_prep_block(cb + (size_t)m * TN * DS, m, a, s_n2);
}

// (optional residual) + per-sub-space squared norms: one thread per (row, m)
__global__ void residual_norms_kernel(const float* x, const float* __restrict__ cent,
                                      const uint32_t* __restrict__ part, uint64_t n, int M,
                                      float* r_out, float* __restrict__ rn2) {
  const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n * M) return;
  const uint64_t row = g / M;
  const int m = g % M;
  const int d = M * DS;
  const float4* xp = reinterpret_cast<const float4*>(x + row * d + m * DS);
  float4 a = xp[0], b = xp[1];
  if (cent) {
    const float4* cp = reinterpret_cast<const float4*>(cent + (size_t)part[row] * d + m * DS);
    const float4 ca = cp[0], cbv = cp[1];
    a.x = __fsub_rn(a.x, ca.x); a.y = __fsub_rn(a.y, ca.y); a.z = __fsub_rn(a.z, ca.z); a.w = __fsub_rn(a.w, ca.w);
    b.x = __fsub_rn(b.x, cbv.x); b.y = __fsub_rn(b.y, cbv.y); b.z = __fsub_rn(b.z, cbv.z); b.w = __fsub_rn(b.w, cbv.w);
  }
  if (r_out) {
    float4* rp = reinterpret_cast<float4*>(r_out + row * d + m * DS);
    rp[0] = a;
    rp[1] = b;
  }
  rn2[g] = a.x * a.x + a.y * a.y + a.z * a.z + a.w * a.w + b.x * b.x + b.y * b.y + b.z * b.z + b.w * b.w;
}

// The (row, sub-space) pairs the filter could not decide.  The filter appends the rows to one list per sub-space,
// so a CTA stages that sub-space's codebook (8 KB) and -|c|^2/2 in shared memory once and serves its share of the
// list from there, TWO pairs per half-warp at a time (each codeword fetched from shared memory serves two rows:
// the kernel is bound by that traffic otherwise), lane l owning codewords l, l+16, ...:
//   1. pre-screen with fused multiply-adds: s'(c) = r.c - |c|^2/2, 8 FFMA per codeword instead of 24 separately
//      rounded operations.  s' is within 2^-21 (|r|^2 + |c|^2) of the true score (8 fused steps, one rounding
//      each, plus the rounded |c|^2), and the reference's own f32 distances are within 2^-20 (|r|^2 + |c|^2) of
//      the true ones, so the reference's argmin has s'(c) >= max s' - 2^-18 (|r|^2 + max|c|^2) (twice the sum;
//      the norm term has the floor of cert_tau: below the normal range both roundings are absolute, <= 2^-149 each);
//   2. only those few codewords get the reference-order distance (sequential 8-term sum, l2.rs:69-79), with the
//      reference's strict-< / lowest-index rule among them.
// A NaN anywhere makes the threshold or the scores NaN: `!(s' < thr)` then keeps the codeword and the exact
// arithmetic decides as a full scan would.
constexpr int FB_P = 2;
// reference-order distance of one candidate codeword (kept out of line: the 32 unrolled call sites would otherwise
// be if-converted with all their shared-memory loads hoisted -- 250 registers)
static __device__ __noinline__ void fb_exact_candidate(const float* rvq, const float* cp, int c, float& bv, uint32_t& bi) {
  float sacc = 0.0f;
#pragma unroll
  for (int t = 0; t < DS; ++t) sacc = f_add(sacc, sq_diff(rvq[t], cp[t]));
  const float v = f_add(sacc, 0.0f);
  if (v < bv) { bv = v; bi = (uint32_t)c; }
}
template <bool TRAIN>
__global__ void __launch_bounds__(256, 2)
pq_fallback_kernel(const float* __restrict__ r, uint64_t n, int M, const float* __restrict__ cb,
                   const uint32_t* __restrict__ pairs, const uint32_t* __restrict__ count,
                   const uint8_t* __restrict__ row_valid, uint8_t* __restrict__ codes,
                   uint32_t* __restrict__ ids, float* __restrict__ dists, uint8_t* __restrict__ valid) {
  __shared__ __align__(16) float cbs[TN * DS];
  __shared__ float cnh_s[TN];
  __shared__ float s_cmax;
  const int m = blockIdx.x;
  const uint32_t total = count[m];
  if (blockIdx.y * (16u * FB_P) >= total) return;  // uniform
  {
    const float4* src = reinterpret_cast<const float4*>(cb + (size_t)m * TN * DS);
    float4* dst = reinterpret_cast<float4*>(cbs);
    for (int i = threadIdx.x; i < TN * DS / 4; i += 256) dst[i] = src[i];
  }
  __syncthreads();
  {
    const int c = threadIdx.x;  // 256 threads == 256 codewords
    float n2 = 0.0f;
#pragma unroll
    for (int t = 0; t < DS; ++t) n2 = fmaf(cbs[c * DS + t], cbs[c * DS + t], n2);
    cnh_s[c] = -0.5f * n2;
    float mx = n2;
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if (c == 0) s_cmax = 0.0f;
    __syncthreads();
    if ((c & 31) == 0) atomicMax(reinterpret_cast<int*>(&s_cmax), __float_as_int(mx));  // n2 >= 0: int order == float order
    __syncthreads();
  }
  const float cmax = s_cmax;  // NaN codewords: mx is NaN -> as an int it is larger than every number: thr turns NaN
  const int l = threadIdx.x & 15;
  const unsigned mask = 0xffffu << (16 * ((threadIdx.x >> 4) & 1));
  const uint32_t* list = pairs + (size_t)m * n;
  for (uint32_t p0 = (blockIdx.y * 16u + (threadIdx.x >> 4)) * FB_P; p0 < total; p0 += gridDim.y * 16u * FB_P) {
    float rv[FB_P][DS], rn[FB_P];
    uint64_t rows[FB_P];
#pragma unroll
    for (int q = 0; q < FB_P; ++q) {
      rows[q] = list[min(p0 + q, total - 1)];  // the tail repeats the last pair (same result written twice)
      const float* rp = r + rows[q] * (uint64_t)(M * DS) + m * DS;
      const float4 r0 = reinterpret_cast<const float4*>(rp)[0], r1 = reinterpret_cast<const float4*>(rp)[1];
      rv[q][0] = r0.x; rv[q][1] = r0.y; rv[q][2] = r0.z; rv[q][3] = r0.w;
      rv[q][4] = r1.x; rv[q][5] = r1.y; rv[q][6] = r1.z; rv[q][7] = r1.w;
      rn[q] = 0.0f;
#pragma unroll
      for (int t = 0; t < DS; ++t) rn[q] = fmaf(rv[q][t], rv[q][t], rn[q]);
    }
    float sc[FB_P][TN / 16], smax[FB_P];
#pragma unroll
    for (int q = 0; q < FB_P; ++q) smax[q] = __int_as_float(0xff800000);
#pragma unroll
    for (int i = 0; i < TN / 16; ++i) {
      const int c = l + 16 * i;
      const float4 c0 = reinterpret_cast<const float4*>(cbs + c * DS)[0];
      const float4 c1 = reinterpret_cast<const float4*>(cbs + c * DS)[1];
      const float cv[DS] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
      const float ch = cnh_s[c];
#pragma unroll
      for (int q = 0; q < FB_P; ++q) {
        float dot = ch;
#pragma unroll
        for (int t = 0; t < DS; ++t) dot = fmaf(rv[q][t], cv[t], dot);
        sc[q][i] = dot;
        smax[q] = fmaxf(smax[q], dot);
      }
      // (keeps the compiler from hoisting all 16 codeword loads to the top: 144 live registers otherwise)
      if ((i & 3) == 3) asm volatile("" ::: "memory");
    }
#pragma unroll
    for (int q = 0; q < FB_P; ++q) {
#pragma unroll
      for (int off = 8; off >= 1; off >>= 1) smax[q] = fmaxf(smax[q], __shfl_xor_sync(mask, smax[q], off, 16));
      const float thr = smax[q] - cert_tau(3.814697265625e-6f, rn[q] + cmax);  // 2^-18
      float bv = __int_as_float(0x7f800000);
      uint32_t bi = 0xffffffffu;
#pragma unroll
      for (int i = 0; i < TN / 16; ++i) {
        if (!(sc[q][i] < thr)) fb_exact_candidate(rv[q], cbs + (l + 16 * i) * DS, l + 16 * i, bv, bi);
      }
#pragma unroll
      for (int off = 8; off >= 1; off >>= 1) {
        const float ov = __shfl_xor_sync(mask, bv, off, 16);
        const uint32_t oi = __shfl_xor_sync(mask, bi, off, 16);
        if (better(ov, oi, bv, bi)) { bv = ov; bi = oi; }
      }
      if (l == 0) {
        const uint64_t row = rows[q];
        const bool ok = bi != 0xffffffffu;
        if (TRAIN) {
          ids[(uint64_t)m * n + row] = ok ? bi : 0u;
          dists[(uint64_t)m * n + row] = ok ? bv : __int_as_float(0x7fc00000);
          valid[(uint64_t)m * n + row] = ok ? 1 : 0;
        } else {
          const bool rv_ok = row_valid ? row_valid[row] != 0 : true;
          codes[row * (uint64_t)M + m] = (ok && rv_ok) ? (uint8_t)bi : (uint8_t)0;
        }
      }
    }
  }
}

}  // namespace tcpq

bool tc_pq_supported(uint64_t n, int d, int M, int ds, int Kc, int metric, const float* x) {
  if (getenv("LB2_DISABLE_TC") && *getenv("LB2_DISABLE_TC")) return false;
  return metric == METRIC_L2 && ds == 8 && Kc == 256 && d == M * 8 && d % 32 == 0 && M <= tcpq::MAX_M &&
         n >= 256 && n * (uint64_t)M < (1ull << 32) && (reinterpret_cast<uintptr_t>(x) & 15) == 0;
}

TcPqPrepArgs tc_pq_prep_args(int M, int d, TcPqWorkspace* ws) {
  if (ws->bm.n < (size_t)tc::TN * d) ws->bm.alloc((size_t)tc::TN * d);
  if (ws->cnh.n < (size_t)M * tc::TN + M) ws->cnh.alloc((size_t)M * tc::TN + M);
  if (ws->fb_count.n < (size_t)M) ws->fb_count.alloc(M);
  TcPqPrepArgs a;
  a.bm = ws->bm.p;
  a.cnh = ws->cnh.p;
  a.cbmax2 = ws->cnh.p + (size_t)M * tc::TN;
  a.fb_count = ws->fb_count.p;
  a.d = d;
  return a;
}
void tc_pq_prepare(const float* codebook, int M, int d, TcPqWorkspace* ws) {
  using namespace tcpq;
  const TcPqPrepArgs a = tc_pq_prep_args(M, d, ws);
  LB2_LAUNCH("tc_pq_prep_codebook", prep_codebook_kernel, M, tc::TN, 0, codebook, a);
}

// r: residual (or raw) vectors [n][d] with their per-sub-space norms rn2 [n][M] already computed
void tc_pq_assign(const float* r, const float* rn2, uint64_t n, int d, int M, const float* codebook,
                  const uint8_t* row_valid, uint8_t* codes, uint32_t* ids, float* dists,
                  uint8_t* valid, const uint8_t* active, TcPqWorkspace* ws, bool prepared) {
  using namespace tcpq;
  const int nkc = M / 4;
  const bool stream = M > MAX_M_RESIDENT;
  const Layout L = layout(nkc, M, stream);
  const size_t smem = L.total + 1024;
  if (smem > ctx().smem_optin) fail(LB2_UNSUPPORTED, "tc_pq: shared memory");
  LB2_REQUIRE(!(codes && active), "tc_pq: encode decides every sub-space");
  if (!prepared) tc_pq_prepare(codebook, M, d, ws);  // also resets the undecided-row lists
  if (ws->fb_pairs.n < n * M) ws->fb_pairs.alloc(n * M);
  const CUtensorMap map_r = make_map_2d(r, n, d, tc::TM);
  const CUtensorMap map_b = make_map_2d(ws->bm.p, tc::TN, d, tc::TN);
  const uint64_t tiles = (n + tc::TM - 1) / tc::TM;
  const unsigned grid = (unsigned)std::min<uint64_t>(tiles * nkc, (uint64_t)ctx().num_sms);
  const float* cnh = ws->cnh.p;
  const float* cbmax2 = ws->cnh.p + (size_t)M * tc::TN;
  // per sub-space: enough CTAs (16 pairs per pass each) for the worst case, capped; idle ones exit at once
  const dim3 fb_grid((unsigned)M, (unsigned)std::min<uint64_t>(cdiv(n, 16 * tcpq::FB_P), std::max(1, 8 * ctx().num_sms / M)));
#define LB2_PQ_FILTER(TRAINV, STREAMV)                                                                      \
  do {                                                                                                      \
    set_smem(tc_pq_kernel<TRAINV, STREAMV>, smem);                                                          \
    LB2_LAUNCH("tc_pq_filter", (tc_pq_kernel<TRAINV, STREAMV>), grid, Pipe<STREAMV>::THREADS, smem, map_r,   \
               map_b, n, M, cnh, cbmax2, rn2, row_valid, codes, ids, dists, valid, ws->fb_pairs.p,          \
               ws->fb_count.p, active);                                                                     \
  } while (0)
  if (codes) {
    if (stream) LB2_PQ_FILTER(false, true); else LB2_PQ_FILTER(false, false);
    LB2_LAUNCH("tc_pq_fallback", pq_fallback_kernel<false>, fb_grid, 256, 0, r, n, M, codebook,
               ws->fb_pairs.p, ws->fb_count.p, row_valid, codes, ids, dists, valid);
  } else {
    if (stream) LB2_PQ_FILTER(true, true); else LB2_PQ_FILTER(true, false);
    LB2_LAUNCH("tc_pq_fallback", pq_fallback_kernel<true>, fb_grid, 256, 0, r, n, M, codebook,
               ws->fb_pairs.p, ws->fb_count.p, row_valid, codes, ids, dists, valid);
  }
#undef LB2_PQ_FILTER
  if (getenv("LB2_TC_STATS") && *getenv("LB2_TC_STATS")) {
    std::vector<uint32_t> cm(M);
    d2h(cm.data(), ws->fb_count.p, M);
    sync_stream();
    uint64_t c = 0;
    for (int m = 0; m < M; ++m) c += cm[m];
    fprintf(stderr, "[lb2 tc_pq] n=%llu M=%d: exact-fallback pairs %.2f%%\n", (unsigned long long)n, M,
            100.0 * c / ((double)n * M));
  }
}

void pq_encode_dev(const float* x, uint64_t n, int d, int M, int ds, const float* codebook, int metric,
                   const float* cent, const uint32_t* part, const uint8_t* row_valid, uint8_t* codes) {
  if (n == 0) return;
  // (the filter stores a row's four codes of a chunk as one word)
  if (!tc_pq_supported(n, d, M, ds, 256, metric, x) || (reinterpret_cast<uintptr_t>(codes) & 3) != 0) {
    pq_assign_f32(x, n, d, M, ds, codebook, 256, metric, cent, part, row_valid, codes, nullptr, nullptr, nullptr,
                  nullptr);
    return;
  }
  TcPqWorkspace ws;
  const uint64_t chunk = std::max<uint64_t>(1ull << 16, (1ull << 28) / (uint64_t)d);  // <= 1 GB of residuals
  DevBuf<float> r, rn2(std::min(n, chunk) * M);
  if (cent) r.alloc(std::min(n, chunk) * d);
  for (uint64_t r0 = 0; r0 < n; r0 += chunk) {
    const uint64_t rows = std::min(chunk, n - r0);
    const float* xs = x + r0 * d;
    tc_pq_residual_norms(xs, cent, part ? part + r0 : nullptr, rows, M, cent ? r.p : nullptr, rn2.p);
    tc_pq_assign(cent ? r.p : xs, rn2.p, rows, d, M, codebook, row_valid ? row_valid + r0 : nullptr,
                 codes + r0 * M, nullptr, nullptr, nullptr, nullptr, &ws);
  }
}

void tc_pq_residual_norms(const float* x, const float* cent, const uint32_t* part, uint64_t n, int M,
                          float* r_out, float* rn2) {
  LB2_LAUNCH("tc_pq_residual_norms", tcpq::residual_norms_kernel, cdiv(n * M, 256), 256, 0, x, cent,
             part, n, M, r_out, rn2);
}

}  // namespace lb2
