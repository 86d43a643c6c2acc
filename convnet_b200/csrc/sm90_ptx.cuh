// sm90_ptx.cuh — thin inline-PTX wrappers for the Hopper (sm_90a) features the conv kernels use: mbarrier, TMA tiled
// loads, wgmma (bf16, operands in shared memory, accumulators in registers) and mma.sync (tf32).
// Hand-written from the PTX ISA; descriptor fields as in the PTX "matrix descriptor" section.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace cnb {
namespace ptx {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---- mbarrier ---------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P1;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, P1;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Wait with a watchdog: a protocol bug must trap, not hang the GPU.  The budget is WALL-CLOCK time (%globaltimer, 20 s):
// a healthy wait that is merely descheduled (time slicing with another process) cannot reach it.
// -DCNB_NO_MBAR_WATCHDOG removes it.
__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t;
}
__device__ __forceinline__ void mbar_wait_slow(uint64_t* bar, uint32_t parity) {
#ifdef CNB_NO_MBAR_WATCHDOG
  while (!mbar_try_wait(bar, parity)) {}
#else
  unsigned long long t0 = 0;
  unsigned spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if ((++spins & 0x3FFu) != 0) continue;                 // look at the clock every 1024 failed polls only
    const unsigned long long now = globaltimer_ns();
    if (t0 == 0) t0 = now;
    else if (now - t0 > 20000000000ULL) {
      __trap();                                            // no printf: a call here would serialise the wgmma pipeline
    }
  }
#endif
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (!mbar_try_wait(bar, parity)) mbar_wait_slow(bar, parity);
}

// ---- TMA tiled loads (global -> shared, completes on an mbarrier) ------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const void* desc) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(desc)) : "memory");
}
__device__ __forceinline__ void tma_load_3d(const void* desc, uint64_t* bar, void* dst, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(desc)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(const void* desc, uint64_t* bar, void* dst, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(desc)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_load_5d(const void* desc, uint64_t* bar, void* dst, int c0, int c1, int c2, int c3,
                                            int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(desc)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2),
      "r"(c3), "r"(c4)
      : "memory");
}

// Programmatic dependent launch (griddepcontrol): a kernel launched with cudaLaunchAttributeProgrammaticStreamSerialization
// may become resident while its predecessor in the stream is still draining; pdl_wait() blocks until every prerequisite
// grid has completed and its memory is visible.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// ---- shared-memory loads the compiler must not hoist above an mbarrier wait ---------------------
__device__ __forceinline__ uint32_t lds32(uint32_t addr) {
  uint32_t v; asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory"); return v;
}

// ---- mma.sync (tf32): D[16x8] += A[16x8] * B[8x8], fp32 bit patterns in, the tensor core reads their tf32 part ---------
__device__ __forceinline__ void mma_tf32_16x8x8(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                                uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
               "{%0, %1, %2, %3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

// ---- wgmma ---------------------------------------------------------------------------------------
// Shared-memory matrix descriptor: start>>4 [0,14), LBO>>4 [16,30), SBO>>4 [32,46), layout [62,64) (1 = SWIZZLE_128B).
//   K-major SWIZZLE_128B : rows of 128 B, SBO = 8 rows = 1 KiB between 8-row groups, LBO unused (16);
//                          the K step of 16 bf16 is +32 B inside the swizzle atom.
//   MN-major SWIZZLE_128B: [64-element MN chunk][K rows][128 B], LBO = MN-chunk stride, SBO = 1 KiB between 8-K-row
//                          groups; the K step of 16 is +2 KiB.
__device__ __forceinline__ uint64_t gmma_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  return (uint64_t)((smem_addr >> 4) & 0x3FFF) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16) |
         ((uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32) | (1ULL << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from touching accumulator registers across wgmma issue / wait
__device__ __forceinline__ void wgmma_fence_operands(float (&d)[16][4]) {
#pragma unroll
  for (int j = 0; j < 16; j++)
#pragma unroll
    for (int e = 0; e < 4; e++) asm volatile("" : "+f"(d[j][e])::"memory");
}

#define CNB_ACC4(j) "+f"(d[j][0]), "+f"(d[j][1]), "+f"(d[j][2]), "+f"(d[j][3])
// D[64 x 128] (fp32, registers of one warpgroup) += A[64 x 16] * B[16 x 128], bf16 in shared memory.
// TA / TB = 1: that operand is MN-major (transposed).  Accumulator j*4+e of a thread: n8-tile j, as in mma.sync m16n8.
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n128k16_bf16(float (&d)[16][4], uint64_t desc_a, uint64_t desc_b) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %68, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1, %66, %67;\n\t}"
      : CNB_ACC4(0), CNB_ACC4(1), CNB_ACC4(2), CNB_ACC4(3), CNB_ACC4(4), CNB_ACC4(5), CNB_ACC4(6), CNB_ACC4(7),
        CNB_ACC4(8), CNB_ACC4(9), CNB_ACC4(10), CNB_ACC4(11), CNB_ACC4(12), CNB_ACC4(13), CNB_ACC4(14), CNB_ACC4(15)
      : "l"(desc_a), "l"(desc_b), "n"(TA), "n"(TB), "r"(1));
}
#undef CNB_ACC4

}  // namespace ptx
}  // namespace cnb
