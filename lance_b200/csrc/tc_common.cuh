// tc_common.cuh -- PTX wrappers shared by the Hopper tensor-core kernels (tc_assign.cu, tc_pq.cu):
// mbarrier, TMA (cp.async.bulk.tensor), wgmma shared-memory descriptors, wgmma.mma_async, and the
// reductions of the epilogues over the wgmma accumulator fragment.
// Descriptor and fragment layouts follow the PTX ISA ("Asynchronous Warpgroup Level Matrix Multiply").
#pragma once
#include <cuda.h>
#include <cudaTypedefs.h>
#include <stdint.h>
#include <stdio.h>

#include "common.cuh"

namespace lb2 {
namespace tc {

constexpr int TM = 64;                   // rows per tile (wgmma M: one consumer warpgroup)
constexpr int TN = 256;                  // centroids per tile (wgmma N)
constexpr int KC = 32;                   // f32 per 128-byte swizzle row
constexpr int A_STAGE_BYTES = TM * 128;  // 8 KB
constexpr int B_CHUNK_BYTES = TN * 128;  // 32 KB
constexpr int MAX_STAGES = 6;
constexpr int NUM_THREADS = 384;  // warpgroup 0: TMA producer (one thread); warpgroups 1 and 2: consumers taking
                                  // alternate tiles, so that one warpgroup's epilogue overlaps the other's MMAs
constexpr int PRODUCER_REGS = 40, CONSUMER_REGS = 232;  // 128 * 40 + 256 * 232 <= 64 K registers

// The certificate of every filter: tau = tau_scale * max(|x|^2 + max|c|^2, NORM_FLOOR) (DESIGN.md section 5).
// The relative bounds hold while operands, products and sums are normal f32 numbers.  Below that range roundings are
// absolute (<= 2^-149 each; a product flushed to zero loses < 2^-126; the packed column index moves a subnormal score
// by < 2^-141) while tau_scale * (|x|^2 + max|c|^2) underflows to 0.  With the floor tau >= 2^-13 * 2^-90 = 2^-103,
// twice the worst absolute error of a score (d * 2^-126 + 2^-141 <= 2^-114 at d <= 4096): rows below the floor become
// undecided and take the exact path, tau of every other row is unchanged.  `s < F ? F : s` keeps NaN / Inf norms.
constexpr float NORM_FLOOR = 0x1p-90f;
__device__ __forceinline__ float cert_tau(float tau_scale, float norm2) {
  return tau_scale * (norm2 < NORM_FLOOR ? NORM_FLOOR : norm2);
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// Watchdog: a wait that spins for more than ~4 s of SM clocks is a protocol bug, never a slow kernel.
// It traps: the launch fails with an error instead of hanging the GPU.  The path makes no function call
// (no printf): a call inside the consumer warpgroups would serialize their wgmma pipeline and void their
// register budget (setmaxnreg).
__device__ __forceinline__ bool mbar_try(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
// slow path of a wait: taken every few thousand failed polls; the first time records the start time, later
// times compare against it
__device__ __forceinline__ void mbar_watchdog_tick(long long* t0) {
  const long long now = clock64();
  if (*t0 == 0) *t0 = now;
  else if (now - *t0 > 8000000000ll) __trap();
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  long long t0 = 0;
  for (uint32_t spins = 1;; ++spins) {
    if (mbar_try(bar, parity)) return;
    if ((spins & 0x3FFFu) == 0) mbar_watchdog_tick(&t0);
  }
}
// same, for the single-thread producer: back off between polls so that the spin loop does not steal
// issue slots from the consumer warps sharing the scheduler
__device__ __forceinline__ void mbar_wait_relaxed(uint32_t bar, uint32_t parity) {
  long long t0 = 0;
  for (uint32_t spins = 1;; ++spins) {
    if (mbar_try(bar, parity)) return;
    __nanosleep(40);
    if ((spins & 0x3FFu) == 0) mbar_watchdog_tick(&t0);
  }
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar,
                                            int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
// K-major, SWIZZLE_128B shared-memory matrix descriptor of wgmma: start>>4 [0,14), LBO>>4 [16,30) (unused for
// swizzled K-major, 1), SBO>>4 [32,46) = 1024 B (8 rows of 128 B), base offset [49,52) = 0 (every tile starts
// 1024-aligned), layout type [62,64) = 1 (SWIZZLE_128B).  A K step inside the 128-byte row advances the start.
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr) {
  return (uint64_t)((saddr & 0x3FFFF) >> 4) | (1ull << 16) | (64ull << 32) | (1ull << 62);
}

// ---- wgmma (M64 N256, f32 accumulators in 128 registers per thread) ----------------------------------------
// d = A (64 x K, shared) * B^T (256 x K, shared) (+ d when scale_d != 0); TF32: K = 8, f16 / bf16: K = 16
// (32 bytes of a 128-byte swizzled row either way)
__device__ __forceinline__ void wgmma_tf32(float* d, uint64_t a_desc, uint64_t b_desc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
      "%128, %129, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(a_desc), "l"(b_desc), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_f16(float* d, uint64_t a_desc, uint64_t b_desc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
      "%128, %129, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(a_desc), "l"(b_desc), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_bf16(float* d, uint64_t a_desc, uint64_t b_desc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
      "%128, %129, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(a_desc), "l"(b_desc), "r"(scale_d));
}
// M64 N128 (TF32), 64 registers per thread: half of the columns of the N256 tile, same fragment layout with j < 16
__device__ __forceinline__ void wgmma_tf32_n128(float* d, uint64_t a_desc, uint64_t b_desc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a_desc), "l"(b_desc), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// wait until at most N committed wgmma groups of this warpgroup are still in flight
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { wgmma_wait<0>(); }
// ties the accumulator registers to this point: no access to them moves across an asynchronous MMA or its wait
template <int N = 128>
__device__ __forceinline__ void acc_fence(float* d) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// The 1024-aligned base of the dynamic shared memory (SWIZZLE_128B tiles).  Derived from `raw` by pointer
// arithmetic, not through an integer, so that the compiler keeps the shared state space of every access through
// it (LDS, not generic loads).
__device__ __forceinline__ uint8_t* smem_align1024(uint8_t* raw) {
  return raw + ((1024u - (smem_u32(raw) & 1023u)) & 1023u);
}
// OPK: 0 = f32 operands as TF32, 1 = f16, 2 = bf16
template <int OPK>
__device__ __forceinline__ void wgmma_op(float* d, uint64_t a_desc, uint64_t b_desc, uint32_t scale_d) {
  if (OPK == 0) wgmma_tf32(d, a_desc, b_desc, scale_d);
  else if (OPK == 1) wgmma_f16(d, a_desc, b_desc, scale_d);
  else wgmma_bf16(d, a_desc, b_desc, scale_d);
}
// The MMAs of one unit (a 64-row tile against a 256-centroid tile), chunk by chunk: the four K steps of a 128-byte
// chunk of A (64 rows) and B (256 rows) are issued as one wgmma group; the unit's first step overwrites d.
// One group stays in flight: chunk kc is issued before the wait for chunk kc - 1, after which
// release(stage of kc - 1) hands that stage back to the producer.  stage(kc, a, b) waits for the chunk's operands,
// sets their shared-memory addresses and returns the stage.  d is final when this returns.
template <int OPK, class Stage, class Release>
__device__ __forceinline__ void mma_unit(float* d, int nkc, Stage&& stage, Release&& release) {
  acc_fence(d);
  int prev = -1;
  for (int kc = 0; kc < nkc; ++kc) {
    uint32_t a_addr, b_addr;
    const int s = stage(kc, a_addr, b_addr);
    __syncwarp();  // wgmma is warp-aligned: reconverge after the divergent barrier polls
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k)
      wgmma_op<OPK>(d, make_desc(a_addr + k * 32), make_desc(b_addr + k * 32), (kc != 0 || k != 0) ? 1u : 0u);
    wgmma_commit();
    if (prev >= 0) {
      wgmma_wait<1>();
      release(prev);
    }
    prev = s;
  }
  wgmma_wait_all();
  acc_fence(d);
  release(prev);
}
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }

// ---- the accumulator fragment ---------------------------------------------------------------------------------
// Thread t of a warpgroup holds rows r0 = 16 (t / 32) + (t % 32) / 4 and r0 + 8 of the 64-row tile:
// d[4j + 2h + e] = (row r0 + 8h, column 8j + 2 (t % 4) + e), j < 32.  A row's 256 columns are spread over the
// four lanes of a quad.
__device__ __forceinline__ int frag_row(int h) { return 16 * ((threadIdx.x >> 5) & 3) + ((threadIdx.x & 31) >> 2) + 8 * h; }

// ---- top-3 of a 256-column accumulator row by TOURNAMENT ------------------------------------------
// The epilogue is bound by min/max instructions per column.  Pair the values: the winners (max) go on, and
// of the losers (min) only the LARGEST can be among the row's top 3 -- a loser is beaten by its own partner,
// so two losers in the top 3 would need four distinct values ahead of the smaller one.  (All values are
// distinct: each carries its column index in the low mantissa byte.)  Applying this at every level,
//     top3(row) = { champion }  U  top2( largest loser of each level ),
// i.e. per level one running maximum over the losers.  The 256 columns come as two 128-column halves (an
// M64 N128 wgmma each, or the two halves of an N256 fragment); a lane holds 32 values of each half and row:
// levels 0..4 pair those, level 5 pairs the winners of the two halves.
constexpr int TOUR_LEVELS = 6;
// COLUMN UNITS.  With UNIT = 2 the entrants are the 128 column PAIRS (c, c ^ 1) of the row, which are the two
// columns of a lane's j: level 0 is one max of the two raw scores, packed once with the PAIR id (col >> 1), and
// has no loser.  The top 3 are then the three best pair maxima, all distinct by their ids, and the same argument
// holds between pairs: m1 - m2 > tau proves every column outside pair 1 below m1 - tau, m1 - m3 > tau every column
// outside pairs 1 and 2.  The caller ranks the columns of the certified pair(s) exactly (tc_pq.cu).  Per score:
// half a max and half a pack at level 0 instead of a pack, a max, a min and a running max.
constexpr int tour_first_level(int unit) { return unit == 2 ? 1 : 0; }  // levels below it have no losers

struct Tour {
  float top[2];              // winner so far of fragment row h
  float L[2][TOUR_LEVELS];   // largest level-lvl loser so far
};

// score with its column (or unit) in the low mantissa byte: byte b of the id word cw (one PRMT, b a constant)
__device__ __forceinline__ float pack_col(float f, uint32_t cw, int b) {
  return __uint_as_float(__byte_perm(__float_as_uint(f), cw, 0x3214 + b));
}

// Folds one 128-column half of both fragment rows into the tournament (half 0 starts it, half 1 completes it):
// score acc + cn[col], packed with its column (UNIT = 1) or the maximum of a column pair packed with the pair id
// (UNIT = 2).  a: the half's 64 accumulators, a[4j + 2h + e] = (row r0 + 8h,
// column 128 HALF + 8j + 2 (t % 4) + e), j < 16; cn: the 256 values of -|c|^2/2 (shared or global memory).
template <int HALF, int UNIT = 1>
__device__ __forceinline__ void top3_half(const float* a, const float* cn, Tour& st) {
  static_assert(UNIT == 1 || UNIT == 2, "columns or column pairs");
  const uint32_t q = threadIdx.x & 3, q2 = 2 * q;
  // cw[e][i], byte b: the column of j = 4i + b, 128 HALF + 32i + 8b + q2 + e (< 256: no carry between bytes);
  // for pairs one word per i: the pair of j = 4i + b, 64 HALF + 16i + 4b + q
  uint32_t cw[2][4];
#pragma unroll
  for (int e = 0; e < 2; ++e)
#pragma unroll
    for (int i = 0; i < 4; ++i)
      cw[e][i] = UNIT == 2 ? (HALF ? 0x4C484440u : 0x0C080400u) + 0x10101010u * i + 0x01010101u * q
                           : (HALF ? 0x98908880u : 0x18100800u) + 0x20202020u * i + 0x01010101u * (q2 + e);
  float w[2][16];
#pragma unroll
  for (int j = 0; j < 16; ++j) {  // level 0: the two columns of a j
    const float2 cv = *reinterpret_cast<const float2*>(cn + 128 * HALF + 8 * j + q2);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (UNIT == 2) {
        w[h][j] = pack_col(fmaxf(a[4 * j + 2 * h] + cv.x, a[4 * j + 2 * h + 1] + cv.y), cw[0][j >> 2], j & 3);
      } else {
        const float x = pack_col(a[4 * j + 2 * h] + cv.x, cw[0][j >> 2], j & 3);
        const float y = pack_col(a[4 * j + 2 * h + 1] + cv.y, cw[1][j >> 2], j & 3);
        w[h][j] = fmaxf(x, y);
        const float lo = fminf(x, y);
        st.L[h][0] = (HALF == 0 && j == 0) ? lo : fmaxf(st.L[h][0], lo);
      }
    }
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
#pragma unroll
    for (int lvl = 1, cnt = 16; lvl < 5; ++lvl, cnt >>= 1) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        if (i < cnt / 2) {
          const float x = w[h][2 * i], y = w[h][2 * i + 1];
          w[h][i] = fmaxf(x, y);
          const float lo = fminf(x, y);
          st.L[h][lvl] = (HALF == 0 && i == 0) ? lo : fmaxf(st.L[h][lvl], lo);
        }
      }
    }
    if (HALF == 0) {
      st.top[h] = w[h][0];
    } else {  // level 5
      st.L[h][5] = fminf(st.top[h], w[h][0]);
      st.top[h] = fmaxf(st.top[h], w[h][0]);
    }
  }
}

// top-3 of the union of two sorted triples (a[0] >= a[1] >= a[2]), into a
__device__ __forceinline__ void top3_merge(float (&a)[3], const float (&b)[3]) {
  const float x = fminf(a[0], b[0]), y = fmaxf(a[1], b[1]), z = fmaxf(a[2], b[2]);
  a[0] = fmaxf(a[0], b[0]);
  a[1] = fmaxf(x, y);
  a[2] = fmaxf(fminf(x, y), z);
}

// The finished tournament: m = the top-3 (sorted, column or pair id in the low mantissa byte) of all 256 columns
// (128 pairs) of the fragment row r0 + 8 (lane & 1), in every lane of the quad.
template <int UNIT = 1>
__device__ __forceinline__ void top3_finish(const Tour& st, float (&m)[3]) {
  constexpr int F = tour_first_level(UNIT);
  float t[2][3];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float a = fmaxf(st.L[h][F], st.L[h][F + 1]), b = fminf(st.L[h][F], st.L[h][F + 1]);
#pragma unroll
    for (int lvl = F + 2; lvl < TOUR_LEVELS; ++lvl) {
      b = fmaxf(b, fminf(a, st.L[h][lvl]));
      a = fmaxf(a, st.L[h][lvl]);
    }
    t[h][0] = st.top[h];
    t[h][1] = a;
    t[h][2] = b;
  }
  // lanes 0 / 2 of the quad keep row r0 and lanes 1 / 3 row r0 + 8; each hands the other row to its xor-1
  // neighbour, then the xor-2 neighbours (same row) merge
  const bool odd = threadIdx.x & 1;
  float o[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    m[i] = odd ? t[1][i] : t[0][i];
    o[i] = __shfl_xor_sync(0xffffffffu, odd ? t[0][i] : t[1][i], 1);
  }
  top3_merge(m, o);
#pragma unroll
  for (int i = 0; i < 3; ++i) o[i] = __shfl_xor_sync(0xffffffffu, m[i], 2);
  top3_merge(m, o);
}

// top-3 of acc + cn[col] over a whole N256 fragment (see top3_finish)
__device__ __forceinline__ void top3_frag(const float* acc, const float* cn, float (&m)[3]) {
  Tour st;
  top3_half<0>(acc, cn, st);
  top3_half<1>(acc + 64, cn, st);
  top3_finish(st, m);
}

// ---- candidate pass: every column of the fragment's rows whose score reaches thr[h] ---------------------------
// (rows that the top-3 passes could not settle; hits are rare, so the common path is one add and one compare per
// column; the hits of a row are collected as a bit mask and appended afterwards)
constexpr int CAND_SLOTS = 16;
__device__ __forceinline__ void cand_frag(const float* acc, const float* cn, const float (&thr)[2], uint32_t col_base,
                                          uint32_t* const (&cnt)[2], uint32_t* const (&cand)[2]) {
  const uint32_t q2 = 2 * (threadIdx.x & 3);
  uint64_t hit[2] = {0, 0};  // bit 2j + e: column 8j + q2 + e
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const float2 cv = *reinterpret_cast<const float2*>(cn + 8 * j + q2);
#pragma unroll
    for (int h = 0; h < 2; ++h) {  // thr = +inf for rows beyond the list; NaN never compares true
      if (acc[4 * j + 2 * h] + cv.x >= thr[h]) hit[h] |= 1ull << (2 * j);
      if (acc[4 * j + 2 * h + 1] + cv.y >= thr[h]) hit[h] |= 1ull << (2 * j + 1);
    }
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    for (uint64_t m = hit[h]; m; m &= m - 1) {
      const uint32_t b = (uint32_t)(__ffsll((long long)m) - 1);
      const uint32_t slot = atomicAdd(cnt[h], 1u);
      if (slot < (uint32_t)CAND_SLOTS) cand[h][slot] = col_base + 8 * (b >> 1) + q2 + (b & 1);
    }
  }
}

// ---- work order of the filter kernels ----------------------------------------------------------------------
// A unit is one 64-row tile against one 256-centroid tile.  The CTA's row tiles are taken in pairs (one per
// consumer warpgroup) and, per centroid tile, the two warpgroups take turns: their MMA phases alternate
// (named barriers 1 and 2), so one warpgroup's epilogue runs while the other's MMAs do.  The turns also keep
// every stage of the shared TMA ring within one phase of the warpgroup waiting on it: a unit's MMAs start only
// after every earlier chunk of the ring has been consumed.
// f(tile, nt) for every unit, in ring order (the producer).
template <class F>
__device__ __forceinline__ void for_units_producer(uint64_t num_tiles, int ntiles, F&& f) {
  for (uint64_t t0 = blockIdx.x; t0 < num_tiles; t0 += 2 * (uint64_t)gridDim.x) {
    const uint64_t t1 = t0 + gridDim.x;
    for (int nt = 0; nt < ntiles; ++nt) {
      f(t0, nt);
      if (t1 < num_tiles) f(t1, nt);
    }
  }
}
// f(tile, nt, k, pass_turn) for the units of consumer warpgroup w; k = ring index of the unit's first chunk.
// The turn is already held when f runs; f passes it on (pass_turn()) once its MMAs are done.
template <class F>
__device__ __forceinline__ void for_units_consumer(uint64_t num_tiles, int ntiles, int nkc, int w, F&& f) {
  uint64_t k = 0;
  for (uint64_t t0 = blockIdx.x; t0 < num_tiles; t0 += 2 * (uint64_t)gridDim.x) {
    const uint64_t t1 = t0 + gridDim.x;
    const bool has1 = t1 < num_tiles;
    const bool more = t0 + 2 * (uint64_t)gridDim.x < num_tiles;
    for (int nt = 0; nt < ntiles; ++nt) {
      for (int o = 0; o < 2; ++o) {
        if (o == 1 && !has1) continue;
        if (o == w) {
          if (o == 1 || (nt > 0 ? has1 : t0 != blockIdx.x)) asm volatile("bar.sync %0, 256;" ::"r"(1 + w) : "memory");
          const bool pass = o == 0 ? has1 : (nt + 1 < ntiles || more);
          f(o ? t1 : t0, nt, k, [&] {
            if (pass) asm volatile("bar.arrive %0, 256;" ::"r"(2 - w) : "memory");
          });
        }
        k += (uint64_t)nkc;
      }
    }
  }
}

}  // namespace tc

// host: 2-D f32 tensor map, box = [32 floats (128 B, SWIZZLE_128B)] x box_rows
CUtensorMap make_map_2d(const float* base, uint64_t rows, uint64_t cols, uint32_t box_rows);
// same for f16 / bf16 rows: box = [64 elements (128 B)] x box_rows
CUtensorMap make_map_2d_16(const void* base, bool bf16, uint64_t rows, uint64_t cols, uint32_t box_rows);

}  // namespace lb2
