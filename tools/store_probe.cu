// store_probe.cu — how fast one SM can drain 128-row fp32 output tiles to HBM, by the two write paths a conv epilogue
// has on sm_90a.  Built and driven by tools/store_probe.py; not part of the library.
//
// The buffer is `cols` channel planes of `plane` floats each (the conv output layout: a tile of 128 images x BN
// channels at one output position is BN runs of 512 bytes, `plane` floats apart).  One CTA per SM walks tiles
// t = blockIdx.x, blockIdx.x + gridDim.x, ..., as the conv kernel does, and writes each from shared memory:
//   mode 0 (st.global): `warps` warps, warp w takes columns w, w + warps, ...; lane l reads rows 4l..4l+3 of a column
//          with one ld.shared.v4 and writes them with one 16-byte st.global (512 bytes per warp instruction);
//   mode 1 (tensor store): the tile is one box {128 rows, BN columns} of a 2-D tensor map, unswizzled.  `slots`
//          staging tiles: the `warps` warps rewrite tile t's slot in place (one ld/st.shared.v4 per 16 bytes, standing in
//          for the epilogue arithmetic), fence it to the async proxy, and one lane issues the store and commits it.
//          Slot t % slots is reused once the group of tile t - slots has been read (cp.async.bulk.wait_group.read).
//   mode 2 (st.global behind a hand-off): mode 0 fed as the conv kernel feeds its store warps, without the MMAs.  Eight
//          more warps stand in for the consumers: per tile they wait until the store warps have read the one staging
//          tile (`epi_empty`), write it with 32-bit st.shared (BN / 2 values per thread, the accumulator count of a
//          consumer thread) and arrive on `epi_full`; the store warps wait on `epi_full` and release the tile after
//          their last ld.shared, before their last stores.
#include <cuda.h>
#include <cudaTypedefs.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

namespace {

constexpr int kRows = 128;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ float4 lds128(uint32_t a) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(a) : "memory");
  return v;
}
__device__ __forceinline__ void sts128(uint32_t a, float4 v) {
  asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(a), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ void bar_sync(int id, int threads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory"); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok = 0;
  while (!ok)
    asm volatile("{\n\t.reg .pred P1;\n\tmbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2;\n\tselp.b32 %0, 1, 0, P1;\n\t}"
                 : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
}
constexpr int kFillWarps = 8;

__global__ void __launch_bounds__(512, 1)
store_probe_kernel(const __grid_constant__ CUtensorMap map, float* out, long long plane, int tiles_per_col, int num_tiles,
                   int bn, int mode, int warps, int slots, float scale) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const uint32_t slot_bytes = (uint32_t)kRows * bn * 4;
  for (uint32_t i = threadIdx.x * 16; i < slot_bytes * slots; i += blockDim.x * 16)
    sts128(smem_u32(smem) + i, make_float4(1.f, 2.f, 3.f, 4.f));
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t base = smem_u32(smem);
  if (mode == 0) {
    for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
      const int pos = t % tiles_per_col, ct = t / tiles_per_col;
      float* const tile = out + (long long)pos * kRows + (long long)ct * bn * plane + 4 * lane;
      for (int c = warp; c < bn; c += warps) {
        const float4 v = lds128(base + c * (kRows * 4) + 16 * lane);
        *reinterpret_cast<float4*>(tile + plane * c) = make_float4(v.x * scale, v.y * scale, v.z * scale, v.w * scale);
      }
    }
    return;
  }
  if (mode == 2) {
    // the conv kernel's staging layout: column-major, the 16-byte unit row / 4 XORed with col & 7
    auto epi_off = [](int row, int col) {
      return (uint32_t)(col * (kRows * 4) + ((((row >> 2) ^ col) & 7) << 4) + (((row >> 2) & ~7) << 4) + ((row & 3) << 2));
    };
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + 2 * slot_bytes);   // [0] epi_full, [1] epi_empty
    if (threadIdx.x == 0) {
      mbar_init(&bars[0], kFillWarps);
      mbar_init(&bars[1], warps);
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    uint32_t phase = 0;
    if (warp < kFillWarps) {                   // the consumers' hand-off: rows 16 w + g (+8), columns 8 j + 2 q + e
      const int row0 = 16 * warp + (lane >> 2), q = lane & 3;
      for (int t = blockIdx.x; t < num_tiles; t += gridDim.x, phase ^= 1) {
        mbar_wait(&bars[1], phase ^ 1);
        for (int j = 0; j < bn / 8; j++)
#pragma unroll
          for (int e = 0; e < 4; e++) {
            const float v = scale * (float)(j + e);
            asm volatile("st.shared.f32 [%0], %1;" ::"r"(base + epi_off(row0 + 8 * (e >> 1), 8 * j + 2 * q + (e & 1))),
                         "f"(v) : "memory");
          }
        __syncwarp();
        if (lane == 0) mbar_arrive(&bars[0]);
      }
      return;
    }
    const int sw = warp - kFillWarps;
    for (int t = blockIdx.x; t < num_tiles; t += gridDim.x, phase ^= 1) {
      const int pos = t % tiles_per_col, ct = t / tiles_per_col;
      float* const tile = out + (long long)pos * kRows + (long long)ct * bn * plane + 4 * lane;
      mbar_wait(&bars[0], phase);
      for (int c0 = sw; c0 < bn; c0 += 4 * warps) {
        float4 v[4];
#pragma unroll
        for (int k = 0; k < 4; k++) {
          const int c = c0 + k * warps;
          if (c < bn) v[k] = lds128(base + epi_off(4 * lane, c));
        }
        if (c0 + 4 * warps >= bn) {            // the last read of the tile: the fill warps may rewrite it
          __syncwarp();
          if (lane == 0) mbar_arrive(&bars[1]);
        }
#pragma unroll
        for (int k = 0; k < 4; k++) {
          const int c = c0 + k * warps;
          if (c < bn) *reinterpret_cast<float4*>(tile + plane * c) = v[k];
        }
      }
    }
    return;
  }
  const int threads = 32 * warps;
  int n = 0;
  for (int t = blockIdx.x; t < num_tiles; t += gridDim.x, n++) {
    const int pos = t % tiles_per_col, ct = t / tiles_per_col;
    const uint32_t slot = base + (uint32_t)(n % slots) * slot_bytes;
    if (threadIdx.x == 0) {                    // the slot's previous store (tile n - slots) has read it
      if (slots == 1) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
      else asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
    }
    bar_sync(1, threads);
    for (uint32_t i = threadIdx.x * 16; i < slot_bytes; i += threads * 16) {
      const float4 v = lds128(slot + i);
      sts128(slot + i, make_float4(v.x * scale, v.y * scale, v.z * scale, v.w * scale));
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    bar_sync(1, threads);
    if (threadIdx.x == 0) {
      asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
                   ::"l"(reinterpret_cast<uint64_t>(&map)), "r"(slot), "r"(pos * kRows), "r"(ct * bn)
                   : "memory");
      asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    }
  }
  if (threadIdx.x == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

}  // namespace

// Writes `cols` planes of `plane` floats at `out` (plane a multiple of 128) once, on `stream`.  Returns 0, or a
// nonzero code when the tensor map or the launch is refused.
extern "C" int store_probe_run(float* out, long long plane, int cols, int bn, int mode, int warps, int slots,
                               void* stream) {
  static PFN_cuTensorMapEncodeTiled_v12000 encode = nullptr;
  static int sms = 0;
  if (!encode) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      return 1;
    encode = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(fn);
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    cudaFuncSetAttribute(store_probe_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
  }
  const int threads = 32 * (warps + (mode == 2 ? kFillWarps : 0));
  if (plane % kRows != 0 || cols % bn != 0 || bn % 8 != 0 || warps < 1 || threads > 512 || slots < 1 || slots > 2) return 2;
  CUtensorMap map;
  cuuint64_t gdim[2] = {(cuuint64_t)plane, (cuuint64_t)cols}, gstr[1] = {(cuuint64_t)plane * 4};
  cuuint32_t box[2] = {(cuuint32_t)kRows, (cuuint32_t)bn}, estr[2] = {1, 1};
  if (encode(&map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, out, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
             CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
    return 3;
  const int tiles_per_col = (int)(plane / kRows), num_tiles = tiles_per_col * (cols / bn);
  // 227 KiB whatever the slots need: one CTA per SM, as the conv kernel runs
  store_probe_kernel<<<sms, threads, 227 * 1024, (cudaStream_t)stream>>>(map, out, plane, tiles_per_col, num_tiles,
                                                                            bn, mode, warps, slots, 1.0f);
  return cudaGetLastError() == cudaSuccess ? 0 : 4;
}
