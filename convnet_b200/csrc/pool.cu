// pool.cu — max / average pooling forward and backward (2-D and 3-D), HBM-bound.
//
// Replaces kPool / kMaxPoolUndo / kAvgPoolUndo (cudamat_conv_gemm.cu:153-300) and
// kLocalPool* / kLocalMaxUndo / kLocalAvgUndo (cudamat_conv_others.cu:1667-1864,3114-3437).
// Layout (SURVEY.md Appendix A): images (N, W, H, C, T) with N fastest, so a thread
// owns VEC consecutive images of one (pixel, channel) and every load/store is a
// fully coalesced 16-byte access.  Backward passes are GATHERS over the windows that
// cover an input element: no atomics, deterministic (the reference scatters with
// atomicAdd + __syncthreads per tap).
#include <cuda_bf16.h>

#include <algorithm>
#include <type_traits>

#include "conv_kernels.h"

namespace cnb {

template <int VEC> struct Vec;
template <> struct Vec<4> { using T = float4; };
template <> struct Vec<1> { using T = float; };

template <int VEC> __device__ __forceinline__ void vload(const float* p, float (&v)[VEC]);
template <> __device__ __forceinline__ void vload<4>(const float* p, float (&v)[4]) {
  const float4 t = __ldg(reinterpret_cast<const float4*>(p)); v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
}
template <> __device__ __forceinline__ void vload<1>(const float* p, float (&v)[1]) { v[0] = __ldg(p); }
template <int VEC> __device__ __forceinline__ void vstore(float* p, const float (&v)[VEC]);
template <> __device__ __forceinline__ void vstore<4>(float* p, const float (&v)[4]) {
  *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
}
template <> __device__ __forceinline__ void vstore<1>(float* p, const float (&v)[1]) { *p = v[0]; }
// optional bf16 twin of a result (convnet_b200_emit_bf16_next); p16 is indexed like the fp32 target
template <int VEC> __device__ __forceinline__ void vemit(__nv_bfloat16* p16, const float (&v)[VEC]);
template <> __device__ __forceinline__ void vemit<4>(__nv_bfloat16* p16, const float (&v)[4]) {
  const __nv_bfloat162 lo = __floats2bfloat162_rn(v[0], v[1]), hi = __floats2bfloat162_rn(v[2], v[3]);
  uint2 o; o.x = *reinterpret_cast<const uint32_t*>(&lo); o.y = *reinterpret_cast<const uint32_t*>(&hi);
  *reinterpret_cast<uint2*>(p16) = o;
}
template <> __device__ __forceinline__ void vemit<1>(__nv_bfloat16* p16, const float (&v)[1]) { *p16 = __float2bfloat16_rn(v[0]); }

// the fused ReLU' step of PoolEpi (cnb_relu_deriv): acc is zeroed where the mask is not > 0.  The mask is read at p[i], or,
// where it is the pool input itself (a max pool right above its ReLU layer), taken from that input's values `in`
template <int VEC, typename I>
__device__ __forceinline__ void mask_step(float (&acc)[VEC], const float* p, I i, bool is_input, const float (&in)[VEC]) {
  float mk[VEC];
  if (is_input) {
#pragma unroll
    for (int v = 0; v < VEC; v++) mk[v] = in[v];
  } else vload<VEC>(p + i, mk);
#pragma unroll
  for (int v = 0; v < VEC; v++) acc[v] = mk[v] > 0.f ? acc[v] : 0.f;
}
// the colsum of PoolEpi: deterministic block sum of `total` -> rowsum[blockIdx.x][plane] (256 threads)
__device__ __forceinline__ void block_rowsum(float total, float* rowsum) {
  __shared__ float sh[8];
  for (int o = 16; o > 0; o >>= 1) total += __shfl_xor_sync(0xffffffffu, total, o);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = total;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int w = 0; w < 8; w++) s += sh[w];
    rowsum[(size_t)blockIdx.x * gridDim.y + blockIdx.y] = s;
  }
}

// ---- forward -------------------------------------------------------------------------
// the divisor of a 2-D average: the product of the CLIPPED extents, as the reference computes it (gemm.cu:185).  A window
// wholly in the padding has an extent <= 0 on some axis, so its average is 0 / region: NaN where an extent is 0, a signed
// zero where it is negative — not the count of elements the window holds (0, which would give NaN everywhere).
__device__ __forceinline__ int clipped_region(int X0, int Y0, const PoolGeom& g) {
  return (min(X0 + g.kx, g.W) - max(X0, 0)) * (min(Y0 + g.ky, g.H) - max(Y0, 0));
}

// K > 0: 2-D window with kx, ky <= K, fully unrolled with predicated loads so that all K*K 16-byte loads of a
// thread are in flight together (the generic K == 0 version walks the window with runtime loops, one load at a time).
template <int VEC, bool MAX, int K>
__global__ void __launch_bounds__(256) pool_fwd_kernel(PoolGeom g, const float* __restrict__ images,
                                                        float* __restrict__ targets, float so) {
  // blockIdx.y = (channel, output frame) plane; inside a plane all index arithmetic is 32-bit (the 64-bit
  // divisions of a flat index made these kernels instruction-bound, not HBM-bound)
  const unsigned NV = g.N / VEC;
  const unsigned plane = NV * g.modX * g.modY;                   // elements per plane
  const int c = blockIdx.y % g.C, mt = blockIdx.y / g.C;
  for (unsigned pidx = blockIdx.x * blockDim.x + threadIdx.x; pidx < plane; pidx += gridDim.x * blockDim.x) {
    const unsigned nv = pidx % NV, r = pidx / NV;
    const int mx = r % g.modX, my = r / g.modX;
    const long long idx = (long long)blockIdx.y * plane + pidx;
    float acc[VEC];
#pragma unroll
    for (int v = 0; v < VEC; v++) acc[v] = MAX ? -2e38f : 0.f;     // base value: gemm.cu:71
    int region = 0;
    if constexpr (K > 0) {
      const int X0 = mx * g.sx + g.px, Y0 = my * g.sy + g.py;
      region = clipped_region(X0, Y0, g);
      const float* base = images + (long long)g.N * ((long long)g.W * g.H * (c + (long long)g.C * mt)) + nv * VEC;
      float a[K * K][VEC];
      bool ok[K * K];
#pragma unroll
      for (int dy = 0; dy < K; dy++)
#pragma unroll
        for (int dx = 0; dx < K; dx++) {
          const int X = X0 + dx, Y = Y0 + dy;
          ok[dy * K + dx] = dy < g.ky && dx < g.kx && (unsigned)X < (unsigned)g.W && (unsigned)Y < (unsigned)g.H;
          if (ok[dy * K + dx]) vload<VEC>(base + (long long)g.N * (X + (long long)g.W * Y), a[dy * K + dx]);
        }
#pragma unroll
      for (int t = 0; t < K * K; t++)
        if (ok[t]) {
#pragma unroll
          for (int v = 0; v < VEC; v++) acc[v] = MAX ? fmaxf(acc[v], a[t][v]) : acc[v] + a[t][v];
        }
    } else {
      int sX = mx * g.sx + g.px, sY = my * g.sy + g.py, sT = mt * g.st + g.pt;
      const int eX = min(sX + g.kx, g.W), eY = min(sY + g.ky, g.H), eT = min(sT + g.kt, g.T);
      sX = max(sX, 0); sY = max(sY, 0); sT = max(sT, 0);
      for (int T = sT; T < eT; T++)
        for (int Y = sY; Y < eY; Y++) {
          const float* row = images + (long long)g.N * ((long long)g.W * (Y + (long long)g.H * (c + (long long)g.C * T))) + nv * VEC;
          for (int X = sX; X < eX; X++) {
            float a[VEC];
            vload<VEC>(row + (long long)g.N * X, a);
#pragma unroll
            for (int v = 0; v < VEC; v++) acc[v] = MAX ? fmaxf(acc[v], a[v]) : acc[v] + a[v];
          }
        }
      region = (eX - sX) * (eY - sY) * (eT - sT);                  // CLIPPED count: gemm.cu:185
    }
    if (!MAX) {
#pragma unroll
      for (int v = 0; v < VEC; v++) acc[v] = acc[v] / region;
    }
#pragma unroll
    for (int v = 0; v < VEC; v++) acc[v] = so * acc[v];
    vstore<VEC>(targets + idx * VEC, acc);
  }
}

// ---- backward (gather) -----------------------------------------------------------------
// windows covering input coordinate X: m*s + p <= X < m*s + p + k
__device__ __forceinline__ void cover(int X, int s, int p, int k, int mods, int& lo, int& hi) {
  const int a = X - p - k + 1;                 // m*s >= a
  lo = a <= 0 ? 0 : (a + s - 1) / s;
  const int b = X - p;                         // m*s <= b   (b >= 0 whenever a window can cover X)
  hi = b < 0 ? -1 : min(b / s, mods - 1);
}

// Q > 0: 2-D pooling where at most Q windows cover an element along each axis (kernel <= Q*stride): the Q*Q window
// visits are unrolled and predicated so their loads overlap; Q == 0 is the generic (3-D, any geometry) version.
template <int VEC, bool MAX, int Q>
__global__ void __launch_bounds__(256) pool_undo_kernel(PoolGeom g, const float* __restrict__ images,
                                                         const float* __restrict__ grads,
                                                         const float* __restrict__ acts, float* targets,
                                                         float st, float so, const float* __restrict__ relu_mask) {
  const unsigned NV = g.N / VEC;
  const unsigned plane = NV * g.W * g.H;
  const int c = blockIdx.y % g.C, T = blockIdx.y / g.C;
  for (unsigned pidx = blockIdx.x * blockDim.x + threadIdx.x; pidx < plane; pidx += gridDim.x * blockDim.x) {
    const unsigned nv = pidx % NV, r = pidx / NV;
    const int X = r % g.W, Y = r / g.W;
    const long long idx = (long long)blockIdx.y * plane + pidx;
    int x0, x1, y0, y1, t0, t1;
    cover(X, g.sx, g.px, g.kx, g.modX, x0, x1);
    cover(Y, g.sy, g.py, g.ky, g.modY, y0, y1);
    cover(T, g.st, g.pt, g.kt, g.modT, t0, t1);
    float img[VEC], acc[VEC], old[VEC];
#pragma unroll
    for (int v = 0; v < VEC; v++) { acc[v] = 0.f; old[v] = 0.f; img[v] = 0.f; }
    if (MAX) vload<VEC>(images + idx * VEC, img);
    if (st != 0.f) vload<VEC>(targets + idx * VEC, old);
    auto visit = [&](int mx, int my, int mt, const float (&gr)[VEC], const float (&a)[VEC]) {
      if (MAX) {
#pragma unroll
        for (int v = 0; v < VEC; v++) acc[v] += (img[v] == a[v]) ? so * gr[v] : 0.f;     // ties duplicate: gemm.cu:291
      } else {
        int sX = mx * g.sx + g.px, sY = my * g.sy + g.py, sT = mt * g.st + g.pt;
        const int eX = min(sX + g.kx, g.W), eY = min(sY + g.ky, g.H), eT = min(sT + g.kt, g.T);
        sX = max(sX, 0); sY = max(sY, 0); sT = max(sT, 0);
        const int region = (eX - sX) * (eY - sY) * (eT - sT);
#pragma unroll
        for (int v = 0; v < VEC; v++) acc[v] += so * gr[v] / region;                      // gemm.cu:237
      }
    };
    if constexpr (Q > 0) {
      float gr[Q * Q][VEC], a[Q * Q][VEC];
      bool ok[Q * Q];
#pragma unroll
      for (int j = 0; j < Q; j++)
#pragma unroll
        for (int i = 0; i < Q; i++) {
          const int mx = x0 + i, my = y0 + j;
          ok[j * Q + i] = mx <= x1 && my <= y1;
          if (ok[j * Q + i]) {
            const long long off = (long long)g.N * (mx + (long long)g.modX * (my + (long long)g.modY * (c + (long long)g.C * t0))) + nv * VEC;
            vload<VEC>(grads + off, gr[j * Q + i]);
            if (MAX) vload<VEC>(acts + off, a[j * Q + i]);
          }
        }
#pragma unroll
      for (int j = 0; j < Q; j++)
#pragma unroll
        for (int i = 0; i < Q; i++)
          if (ok[j * Q + i]) visit(x0 + i, y0 + j, t0, gr[j * Q + i], a[j * Q + i]);
    } else {
      for (int mt = t0; mt <= t1; mt++)
        for (int my = y0; my <= y1; my++)
          for (int mx = x0; mx <= x1; mx++) {
            const long long off = (long long)g.N * (mx + (long long)g.modX * (my + (long long)g.modY * (c + (long long)g.C * mt))) + nv * VEC;
            float gr[VEC], a[VEC];
            vload<VEC>(grads + off, gr);
            if (MAX) vload<VEC>(acts + off, a); else { for (int v = 0; v < VEC; v++) a[v] = 0.f; }
            visit(mx, my, mt, gr, a);
          }
    }
#pragma unroll
    for (int v = 0; v < VEC; v++) acc[v] += st * old[v];
    if (relu_mask) mask_step<VEC>(acc, relu_mask, idx * VEC, MAX && relu_mask == images, img);
    vstore<VEC>(targets + idx * VEC, acc);
  }
}


// ---- 2-D fast paths: one output ROW per block iteration ---------------------------------------------
// The flat-index kernels above spend ~300-400 instructions per 16-byte result on index arithmetic, which makes them
// issue-bound.  Here everything that depends on the row (window rows, row base pointers) is computed
// once per block iteration from blockIdx (uniform), the stride is a template constant (S = 0: run time), the image
// index is a shift when N/VEC is a power of two, and per-thread offsets are 32-bit.
template <int S> __device__ __forceinline__ int div_s(int a, int s) { return S > 0 ? a / S : a / s; }

// the steps of PoolEpi on VEC results whose first element has index `i` in the target tensor, in the order of the
// stand-alone passes they replace: cnb_relu, the dropout of cnb_dropout (mask-free, element index i), cnb_mult by a
// constant.  Each step is the pass's own single rounding, so the results are bit-identical to those passes.
template <int VEC>
__device__ __forceinline__ void epilogue(const PoolEpi& e, float (&acc)[VEC], long long i) {
#pragma unroll
  for (int v = 0; v < VEC; v++) {
    float x = acc[v];
    if (e.relu) x = fmaxf(x, 0.f);
    if (e.drop_scale != 0.f) x *= dropout_keep(e.drop_seed + (unsigned long long)(i + v), e.drop_prob, e.drop_scale);
    if (e.scale != 1.f) x *= e.scale;
    acc[v] = x;
  }
}
template <int S>
__device__ __forceinline__ void cover_s(int X, int s, int p, int k, int mods, int& lo, int& hi) {
  const int a = X - p - k + 1;
  lo = a <= 0 ? 0 : div_s<S>(a + (S > 0 ? S : s) - 1, s);
  const int b = X - p;
  hi = b < 0 ? -1 : min(div_s<S>(b, s), mods - 1);
}

// EPI: the steps, the mask and the colsum of PoolEpi after the scaled average (average pooling only).  Every instance
// writes the twin (epi.twin, passed as a __restrict__ parameter of its own); the max instances record the tie masks.
template <int VEC, bool MAX, int K, int S, bool EPI>
__global__ void __launch_bounds__(256) pool_fwd_rows_kernel(PoolGeom g, const float* __restrict__ images,
                                                             float* __restrict__ targets, float so, int nv_shift,
                                                             __nv_bfloat16* __restrict__ twin,
                                                             uint16_t* __restrict__ tie_masks, PoolEpi epi) {
  pdl_wait();
  pdl_trigger();
  const unsigned NV = g.N / VEC;
  const unsigned rowlen = NV * g.modX;
  const int sx = S > 0 ? S : g.sx, sy = S > 0 ? S : g.sy;
  const float* img = images + (long long)g.N * g.W * g.H * blockIdx.y;        // this channel's input plane
  float* out = targets + (long long)g.N * g.modX * g.modY * blockIdx.y;
  __nv_bfloat16* out16 = twin ? twin + (long long)g.N * g.modX * g.modY * blockIdx.y : nullptr;
  uint16_t* outm = (MAX && tie_masks) ? tie_masks + (long long)g.N * g.modX * g.modY * blockIdx.y : nullptr;
  const long long out_plane = (long long)g.N * g.modX * g.modY * blockIdx.y;
  const float* mk_p = EPI && epi.mask ? epi.mask + out_plane : nullptr;
  float total = 0.f;
  for (int my = blockIdx.x; my < g.modY; my += gridDim.x) {
    const int Y0 = my * sy + g.py;
    for (unsigned t = threadIdx.x; t < rowlen; t += blockDim.x) {
      const unsigned mx = nv_shift >= 0 ? (t >> nv_shift) : t / NV;
      const unsigned nv = t - mx * NV;
      const int X0 = (int)mx * sx + g.px;
      float acc[VEC];
#pragma unroll
      for (int v = 0; v < VEC; v++) acc[v] = MAX ? -2e38f : 0.f;             // base value: gemm.cu:71
      float a[K * K][VEC];
      bool ok[K * K];
#pragma unroll
      for (int dy = 0; dy < K; dy++)
#pragma unroll
        for (int dx = 0; dx < K; dx++) {
          const int X = X0 + dx, Y = Y0 + dy;
          ok[dy * K + dx] = dy < g.ky && dx < g.kx && (unsigned)X < (unsigned)g.W && (unsigned)Y < (unsigned)g.H;
          if (ok[dy * K + dx]) vload<VEC>(img + (unsigned)((Y * g.W + X) * g.N) + nv * VEC, a[dy * K + dx]);
        }
#pragma unroll
      for (int q = 0; q < K * K; q++)
        if (ok[q]) {
#pragma unroll
          for (int v = 0; v < VEC; v++) acc[v] = MAX ? fmaxf(acc[v], a[q][v]) : acc[v] + a[q][v];
        }
      if (!MAX) {
        const int region = clipped_region((int)X0, Y0, g);
#pragma unroll
        for (int v = 0; v < VEC; v++) acc[v] = acc[v] / region;
      }
      if (MAX && outm) {          // bit q = dx + K*dy: that window element equals the maximum; bit 15: the maximum is > 0
        uint16_t mk[VEC];
#pragma unroll
        for (int v = 0; v < VEC; v++) mk[v] = acc[v] > 0.f ? 0x8000 : 0;
#pragma unroll
        for (int q = 0; q < K * K; q++)
          if (ok[q]) {
#pragma unroll
            for (int v = 0; v < VEC; v++) mk[v] |= (a[q][v] == acc[v]) ? (uint16_t)(1u << q) : (uint16_t)0;
          }
        uint16_t* dstm = outm + (unsigned)(my * rowlen + t) * VEC;
        if (VEC == 4) *reinterpret_cast<uint2*>(dstm) = make_uint2((uint32_t)mk[0] | ((uint32_t)mk[1 % VEC] << 16), (uint32_t)mk[2 % VEC] | ((uint32_t)mk[3 % VEC] << 16));
        else dstm[0] = mk[0];
      }
#pragma unroll
      for (int v = 0; v < VEC; v++) acc[v] = so * acc[v];
      const unsigned o = (unsigned)(my * rowlen + t) * VEC;
      if constexpr (EPI) {
        epilogue<VEC>(epi, acc, out_plane + o);
        if (mk_p) mask_step<VEC>(acc, mk_p, o, false, acc);
        if (epi.colsum) {
#pragma unroll
          for (int v = 0; v < VEC; v++) total += acc[v];
        }
      }
      vstore<VEC>(out + o, acc);
      if (out16) vemit<VEC>(out16 + o, acc);
    }
  }
  if (EPI && epi.colsum) block_rowsum(total, epi.colsum);
}

// EPI: the steps of PoolEpi before its mask (average undo only).  Every instance applies the mask, the colsum and the
// twin, which it takes as __restrict__ parameters of their own (the `epi` pointers are not read).
template <int VEC, bool MAX, int Q, int S, bool EPI>
__global__ void __launch_bounds__(256) pool_undo_rows_kernel(PoolGeom g, const float* __restrict__ images,
                                                              const float* __restrict__ grads,
                                                              const float* __restrict__ acts, float* targets,
                                                              float st, float so, const float* __restrict__ relu_mask,
                                                              int nv_shift, __nv_bfloat16* __restrict__ targets16,
                                                              float* __restrict__ rowsum, PoolEpi epi) {
  pdl_wait();
  pdl_trigger();
  const unsigned NV = g.N / VEC;
  const unsigned rowlen = NV * g.W;
  const long long in_plane = (long long)g.N * g.W * g.H * blockIdx.y, out_plane = (long long)g.N * g.modX * g.modY * blockIdx.y;
  const float* img = MAX ? images + in_plane : nullptr;
  const float* gr_p = grads + out_plane;
  const float* ac_p = MAX ? acts + out_plane : nullptr;
  const float* mk_p = relu_mask ? relu_mask + in_plane : nullptr;
  const bool mask_is_input = MAX && relu_mask == images;     // max-pool right above the ReLU layer: mask == pool input
  float* out = targets + in_plane;
  __nv_bfloat16* out16 = targets16 ? targets16 + in_plane : nullptr;
  float total = 0.f;                            // rowsum: sum of everything this thread stores (bias gradient of the edge below)
  for (int Y = blockIdx.x; Y < g.H; Y += gridDim.x) {
    int y0, y1;
    cover_s<S>(Y, g.sy, g.py, g.ky, g.modY, y0, y1);
    for (unsigned t = threadIdx.x; t < rowlen; t += blockDim.x) {
      const unsigned X = nv_shift >= 0 ? (t >> nv_shift) : t / NV;
      const unsigned nv = t - X * NV;
      const unsigned idx = (unsigned)(Y * rowlen + t) * VEC;
      int x0, x1;
      cover_s<S>((int)X, g.sx, g.px, g.kx, g.modX, x0, x1);
      float im[VEC], acc[VEC], old[VEC];
#pragma unroll
      for (int v = 0; v < VEC; v++) { acc[v] = 0.f; old[v] = 0.f; im[v] = 0.f; }
      if (MAX) vload<VEC>(img + idx, im);
      if (st != 0.f) vload<VEC>(out + idx, old);
      float gr[Q * Q][VEC], a[Q * Q][VEC];
      bool ok[Q * Q];
#pragma unroll
      for (int j = 0; j < Q; j++)
#pragma unroll
        for (int i = 0; i < Q; i++) {
          const int mx = x0 + i, my = y0 + j;
          ok[j * Q + i] = mx <= x1 && my <= y1;
          if (ok[j * Q + i]) {
            const unsigned off = (unsigned)((my * g.modX + mx) * g.N) + nv * VEC;
            vload<VEC>(gr_p + off, gr[j * Q + i]);
            if (MAX) vload<VEC>(ac_p + off, a[j * Q + i]);
          }
        }
#pragma unroll
      for (int j = 0; j < Q; j++)
#pragma unroll
        for (int i = 0; i < Q; i++)
          if (ok[j * Q + i]) {
            if (MAX) {
#pragma unroll
              for (int v = 0; v < VEC; v++) acc[v] += (im[v] == a[j * Q + i][v]) ? so * gr[j * Q + i][v] : 0.f;   // ties duplicate: gemm.cu:291
            } else {
              int sX = (x0 + i) * g.sx + g.px, sY = (y0 + j) * g.sy + g.py;
              const int eX = min(sX + g.kx, g.W), eY = min(sY + g.ky, g.H);
              sX = max(sX, 0); sY = max(sY, 0);
              const int region = (eX - sX) * (eY - sY);
#pragma unroll
              for (int v = 0; v < VEC; v++) acc[v] += so * gr[j * Q + i][v] / region;                            // gemm.cu:237
            }
          }
#pragma unroll
      for (int v = 0; v < VEC; v++) acc[v] += st * old[v];
      if constexpr (EPI) epilogue<VEC>(epi, acc, in_plane + idx);
      if (relu_mask) mask_step<VEC>(acc, mk_p, idx, mask_is_input, im);
      vstore<VEC>(out + idx, acc);
      if (out16) vemit<VEC>(out16 + idx, acc);
      if (rowsum) {
#pragma unroll
        for (int v = 0; v < VEC; v++) total += acc[v];
      }
    }
  }
  if (rowsum) block_rowsum(total, rowsum);
}


// max-pool undo from the tie masks the forward kernel recorded (convnet_b200_pool_cache_next), stride 2, windows up to
// 3 x 3: every window covering an input element contributes its gradient iff the mask says this element equalled the
// window's maximum — the same sum as pool_undo_rows_kernel<MAX>, without loading the pool input or output.  positive_only:
// the fused ReLU' mask is the pool input itself and that input is a ReLU output (>= 0): an element passes the mask iff its
// value — the window maximum it equals — is > 0, which is bit 15.
// Organised by PATCHES: the 2 x 2 input elements whose offset from the padded origin is (2*mx + a, 2*my + b) are covered by
// the same 2 x 2 windows {mx-1, mx} x {my-1, my}, so one thread loads those four (gradient, mask) pairs once and writes
// four outputs.  The undo is bound by instruction issue; sharing the loads, unpacking and tests of the covering windows
// across a patch saves about a third of the instructions per element.  Sums run over the windows in the same ascending
// (y, x) order as the compare-based kernels: results are bit-identical to them.
template <int VEC>
__global__ void __launch_bounds__(256, 4) pool_undo_masked_patch_kernel(PoolGeom g, const float* __restrict__ grads,
                                                                     const uint16_t* __restrict__ tie_masks, float* targets,
                                                                     float st, float so, int positive_only, int nv_shift,
                                                                     __nv_bfloat16* __restrict__ targets16,
                                                                     float* __restrict__ rowsum, int PX, int PY) {
  pdl_wait();
  pdl_trigger();
  const unsigned NV = g.N / VEC;
  const unsigned rowlen = NV * PX;
  const long long in_plane = (long long)g.N * g.W * g.H * blockIdx.y, out_plane = (long long)g.N * g.modX * g.modY * blockIdx.y;
  const float* gr_p = grads + out_plane;
  const uint16_t* mk_p = tie_masks + out_plane;
  float* out = targets + in_plane;
  __nv_bfloat16* out16 = targets16 ? targets16 + in_plane : nullptr;
  float total = 0.f;
  for (int my = blockIdx.x; my < PY; my += gridDim.x) {       // patch row my: input rows 2*my + py + {0, 1} (py <= 0)
    for (unsigned t = threadIdx.x; t < rowlen; t += blockDim.x) {
      const unsigned mx = nv_shift >= 0 ? (t >> nv_shift) : t / NV;
      const unsigned nv = t - mx * NV;
      // per covering window and image: the gradient already scaled, and the tie mask as a 32-bit word that is 0 when the
      // window does not exist or (positive_only) its maximum is not > 0 — the tests below are then one AND each
      float gs[4][VEC];
      unsigned mk[4][VEC];
#pragma unroll
      for (int j = 0; j < 2; j++)
#pragma unroll
        for (int i = 0; i < 2; i++) {
          const int wx = (int)mx - 1 + i, wy = my - 1 + j;
          const int w = j * 2 + i;
#pragma unroll
          for (int v = 0; v < VEC; v++) { gs[w][v] = 0.f; mk[w][v] = 0u; }
          if ((unsigned)wx < (unsigned)g.modX && (unsigned)wy < (unsigned)g.modY) {
            const unsigned off = (unsigned)((wy * g.modX + wx) * g.N) + nv * VEC;
            float gr[VEC];
            vload<VEC>(gr_p + off, gr);
            if (VEC == 4) {
              const uint2 m = __ldg(reinterpret_cast<const uint2*>(mk_p + off));
              mk[w][0] = m.x & 0xFFFFu; mk[w][1 % VEC] = m.x >> 16; mk[w][2 % VEC] = m.y & 0xFFFFu; mk[w][3 % VEC] = m.y >> 16;
            } else mk[w][0] = __ldg(mk_p + off);
#pragma unroll
            for (int v = 0; v < VEC; v++) {
              gs[w][v] = so * gr[v];
              if (positive_only && !(mk[w][v] & 0x8000u)) mk[w][v] = 0u;
            }
          }
        }
#pragma unroll
      for (int b = 0; b < 2; b++) {
        const int Y = 2 * my + g.py + b;
        if ((unsigned)Y >= (unsigned)g.H) continue;
#pragma unroll
        for (int a = 0; a < 2; a++) {
          const int X = 2 * (int)mx + g.px + a;
          if ((unsigned)X >= (unsigned)g.W) continue;
          const unsigned idx = (unsigned)((Y * g.W + X) * g.N) + nv * VEC;
          float acc[VEC], old[VEC];
#pragma unroll
          for (int v = 0; v < VEC; v++) { acc[v] = 0.f; old[v] = 0.f; }
          if (st != 0.f) vload<VEC>(out + idx, old);
#pragma unroll
          for (int j = 0; j < 2; j++) {
            const int dy = 2 * (1 - j) + b;                   // the element's row inside window my-1+j
            if (dy >= 3) continue;                            // (rows / columns beyond a smaller window never have their bit set)
#pragma unroll
            for (int i = 0; i < 2; i++) {
              const int dx = 2 * (1 - i) + a;
              if (dx >= 3) continue;
              const unsigned bit = 1u << (dx + 3 * dy);
#pragma unroll
              for (int v = 0; v < VEC; v++) acc[v] += (mk[j * 2 + i][v] & bit) ? gs[j * 2 + i][v] : 0.f;
            }
          }
#pragma unroll
          for (int v = 0; v < VEC; v++) acc[v] += st * old[v];
          vstore<VEC>(out + idx, acc);
          if (out16) vemit<VEC>(out16 + idx, acc);
          if (rowsum) {
#pragma unroll
            for (int v = 0; v < VEC; v++) total += acc[v];
          }
        }
      }
    }
  }
  if (rowsum) block_rowsum(total, rowsum);
}

// Compare-based max-pool undo (no cached masks) in the same patch organisation: per thread the 2 x 2 inputs of a patch and
// the 2 x 2 windows that cover them, each loaded once.
template <int VEC>
__global__ void __launch_bounds__(256) pool_undo_patch_kernel(PoolGeom g, const float* __restrict__ images,
                                                              const float* __restrict__ grads, const float* __restrict__ acts,
                                                              float* targets, float st, float so,
                                                              const float* __restrict__ relu_mask, int nv_shift,
                                                              __nv_bfloat16* __restrict__ targets16,
                                                              float* __restrict__ rowsum, int PX, int PY) {
  pdl_wait();
  pdl_trigger();
  const unsigned NV = g.N / VEC;
  const unsigned rowlen = NV * PX;
  const long long in_plane = (long long)g.N * g.W * g.H * blockIdx.y, out_plane = (long long)g.N * g.modX * g.modY * blockIdx.y;
  const float* img = images + in_plane;
  const float* gr_p = grads + out_plane;
  const float* ac_p = acts + out_plane;
  const float* mk_p = relu_mask ? relu_mask + in_plane : nullptr;
  const bool mask_is_input = relu_mask == images;
  float* out = targets + in_plane;
  __nv_bfloat16* out16 = targets16 ? targets16 + in_plane : nullptr;
  float total = 0.f;
  for (int my = blockIdx.x; my < PY; my += gridDim.x) {
    for (unsigned t = threadIdx.x; t < rowlen; t += blockDim.x) {
      const unsigned mx = nv_shift >= 0 ? (t >> nv_shift) : t / NV;
      const unsigned nv = t - mx * NV;
      float gr[4][VEC], ac[4][VEC], im[4][VEC];
      bool ok[4], in[4];
#pragma unroll
      for (int j = 0; j < 2; j++)
#pragma unroll
        for (int i = 0; i < 2; i++) {
          const int wx = (int)mx - 1 + i, wy = my - 1 + j;
          ok[j * 2 + i] = (unsigned)wx < (unsigned)g.modX && (unsigned)wy < (unsigned)g.modY;
          if (ok[j * 2 + i]) {
            const unsigned off = (unsigned)((wy * g.modX + wx) * g.N) + nv * VEC;
            vload<VEC>(gr_p + off, gr[j * 2 + i]);
            vload<VEC>(ac_p + off, ac[j * 2 + i]);
          }
          const int X = 2 * (int)mx + g.px + i, Y = 2 * my + g.py + j;        // (a, b) = (i, j) for the patch's own elements
          in[j * 2 + i] = (unsigned)X < (unsigned)g.W && (unsigned)Y < (unsigned)g.H;
          if (in[j * 2 + i]) vload<VEC>(img + (unsigned)((Y * g.W + X) * g.N) + nv * VEC, im[j * 2 + i]);
        }
#pragma unroll
      for (int b = 0; b < 2; b++)
#pragma unroll
        for (int a = 0; a < 2; a++) {
          if (!in[b * 2 + a]) continue;
          const int X = 2 * (int)mx + g.px + a, Y = 2 * my + g.py + b;
          const unsigned idx = (unsigned)((Y * g.W + X) * g.N) + nv * VEC;
          float acc[VEC], old[VEC];
#pragma unroll
          for (int v = 0; v < VEC; v++) { acc[v] = 0.f; old[v] = 0.f; }
          if (st != 0.f) vload<VEC>(out + idx, old);
#pragma unroll
          for (int j = 0; j < 2; j++) {
            if (2 * (1 - j) + b >= g.ky) continue;
#pragma unroll
            for (int i = 0; i < 2; i++) {
              if (2 * (1 - i) + a >= g.kx || !ok[j * 2 + i]) continue;
#pragma unroll
              for (int v = 0; v < VEC; v++) acc[v] += (im[b * 2 + a][v] == ac[j * 2 + i][v]) ? so * gr[j * 2 + i][v] : 0.f;   // gemm.cu:291
            }
          }
#pragma unroll
          for (int v = 0; v < VEC; v++) acc[v] += st * old[v];
          if (relu_mask) mask_step<VEC>(acc, mk_p, idx, mask_is_input, im[b * 2 + a]);
          vstore<VEC>(out + idx, acc);
          if (out16) vemit<VEC>(out16 + idx, acc);
          if (rowsum) {
#pragma unroll
            for (int v = 0; v < VEC; v++) total += acc[v];
          }
        }
    }
  }
  if (rowsum) block_rowsum(total, rowsum);
}

static int pow2_shift(unsigned v) { int s = 0; while ((1u << s) < v) s++; return (1u << s) == v ? s : -1; }

static unsigned long long pool_sig(const PoolGeom& g) {
  unsigned long long sig = 1469598103934665603ULL;
  for (int v : {g.N, g.W, g.H, g.C, g.modX, g.modY, g.kx, g.ky, g.sx, g.sy, g.px, g.py}) sig = (sig ^ (unsigned)v) * 1099511628211ULL;
  return sig;
}
// the geometry of the patch kernels: 2-D, stride 2, windows up to 3 x 3 with a side of 3 (at most 2 x 2 covering windows),
// padding offsets in [-2, 0], in-plane offsets in 32 bits.  The forward pass records tie masks (pool_fwd_rows_kernel<K = 3>
// bit layout) for exactly this geometry, the only one whose undo reads them.
static bool patch_geometry(const PoolGeom& g) {
  return g.kt == 1 && g.T == 1 && g.modT == 1 && std::max(g.kx, g.ky) == 3 && g.sx == 2 && g.sy == 2 && g.px <= 0 &&
         g.py <= 0 && g.px >= -2 && g.py >= -2 && (long long)g.N * g.W * g.H < (1LL << 31);
}

// f(std::integral_constant<T, v>()) for the run-time value v, which is one of Vs: the kernel instance of a run-time choice
template <typename T, T... Vs, typename F>
static void with_const(T v, F&& f) {
  (void)((v == Vs && (f(std::integral_constant<T, Vs>()), true)) || ...);
}
// the S of the row kernels: the stride as a template constant (1 or 2), or 0 (read at run time)
static int row_stride(const PoolGeom& g) { return (g.sx == g.sy && g.sx <= 2) ? g.sx : 0; }

template <int VEC, bool MAX>
static PoolOutcome launch_fwd(const PoolGeom& g, const float* images, float* targets, float so, uint16_t* masks,
                              const PoolEpi& epi) {
  cudaStream_t s = state().stream;
  const int planes = g.C * g.modT;
  const long long per_plane = (long long)g.modX * g.modY * (g.N / VEC);
  CNB_REQUIRE(per_plane < (1LL << 30) && planes <= 65535, "pool_forward: plane too large");
  PoolOutcome o;
  const int k = (g.kt == 1 && g.T == 1 && g.modT == 1) ? std::max(g.kx, g.ky) : 99;
  if (k <= 3 && (long long)g.N * g.W * g.H < (1LL << 31)) {          // 2-D, small window: the row-structured kernels
    const bool e = epi.steps() || epi.mask || epi.colsum;    // (never with max pooling: the EPI instances are average's)
    const int sh = pow2_shift(g.N / VEC);
    o.emitted = epi.twin != nullptr;
    o.colsum_slices = epi.colsum ? g.modY : 0;
    with_const<int, 2, 3>(k <= 2 ? 2 : 3, [&](auto K) {
      with_const<int, 0, 1, 2>(row_stride(g), [&](auto S) {
        launch_pdl(e ? pool_fwd_rows_kernel<VEC, false, K, S, true> : pool_fwd_rows_kernel<VEC, MAX, K, S, false>,
                   dim3((unsigned)g.modY, planes), dim3(256), 0, s, g, images, targets, so, sh, epi.twin, masks, epi);
      });
    });
    return o;
  }
  o.fused = false;
  const dim3 grid((unsigned)std::max<long long>(1, std::min<long long>(ceil_div<long long>(per_plane, 256), 64)), planes);
  with_const<int, 2, 3, 4, 0>(k <= 2 ? 2 : k <= 4 ? k : 0, [&](auto K) {
    pool_fwd_kernel<VEC, MAX, K><<<grid, 256, 0, s>>>(g, images, targets, so);
  });
  return o;
}

PoolOutcome pool_forward(const PoolGeom& g, bool is_max, const float* images, float* targets, float so, const PoolEpi& epi) {
  CNB_REQUIRE(!is_max || !(epi.steps() || epi.mask || epi.colsum), "pool_forward: max pooling fuses only the twin and the tie masks");
  const bool v4 = (g.N % 4 == 0) && aligned16(images) && aligned16(targets) && (!epi.mask || aligned16(epi.mask));
  // tie masks for the matching undo: unscaled outputs only
  uint16_t* masks = nullptr;
  if (epi.cache_masks && is_max && so == 1.f && patch_geometry(g))
    masks = pool_masks_slot(targets, (long long)g.modX * g.modY * g.C * g.modT * g.N, images,
                            (long long)g.N * g.W * g.H * g.C, pool_sig(g));
  PoolOutcome o;
  with_const<int, 1, 4>(v4 ? 4 : 1, [&](auto VEC) {
    with_const<bool, false, true>(is_max, [&](auto MAX) { o = launch_fwd<VEC, MAX>(g, images, targets, so, masks, epi); });
  });
  count_launch();
  CNB_LAUNCH_CHECK("pool_forward");
  return o;
}

// ---- max-pool R-operator (kMaxPoolRprop) ---------------------------------------------------------------------------------
// targets[window] = st * targets[window] + the sum of R_images over every element of the clipped window whose image value
// equals the stored maximum, ties counted once each, in the reference's (Y, X) order: the reference adds these terms with
// atomicAdd, but one thread adds all terms of one output in that order, so the sum is the same.  One thread per VEC images
// of one window: a gather with no atomics.
template <int VEC>
__global__ void __launch_bounds__(256) pool_rprop_kernel(PoolGeom g, const float* __restrict__ images,
                                                          const float* __restrict__ R_images, const float* __restrict__ maxes,
                                                          float* targets, float st) {
  pdl_wait();
  pdl_trigger();
  const unsigned NV = g.N / VEC;
  const unsigned plane = NV * g.modX * g.modY;
  const float* img = images + (long long)g.N * g.W * g.H * blockIdx.y;
  const float* rim = R_images + (long long)g.N * g.W * g.H * blockIdx.y;
  for (unsigned pidx = blockIdx.x * blockDim.x + threadIdx.x; pidx < plane; pidx += gridDim.x * blockDim.x) {
    const unsigned nv = pidx % NV, r = pidx / NV;
    const int mx = r % g.modX, my = r / g.modX;
    const long long idx = ((long long)blockIdx.y * plane + pidx) * VEC;
    float m[VEC], acc[VEC];
    vload<VEC>(maxes + idx, m);
    if (st != 0.f) {
      vload<VEC>(targets + idx, acc);
#pragma unroll
      for (int v = 0; v < VEC; v++) acc[v] *= st;
    } else {
#pragma unroll
      for (int v = 0; v < VEC; v++) acc[v] = 0.f;
    }
    const int sX = max(mx * g.sx + g.px, 0), sY = max(my * g.sy + g.py, 0);
    const int eX = min(mx * g.sx + g.px + g.kx, g.W), eY = min(my * g.sy + g.py + g.ky, g.H);
    for (int Y = sY; Y < eY; Y++)
      for (int X = sX; X < eX; X++) {
        const long long off = (long long)g.N * (X + (long long)g.W * Y) + nv * VEC;
        float a[VEC], ra[VEC];
        vload<VEC>(img + off, a);
        vload<VEC>(rim + off, ra);
#pragma unroll
        for (int v = 0; v < VEC; v++)
          if (a[v] == m[v]) acc[v] += ra[v];           // (not `+= tie ? r : 0`: adding +0 would turn a -0 sum into +0)
      }
    vstore<VEC>(targets + idx, acc);
  }
}

void max_pool_rprop(const PoolGeom& g, const float* images, const float* R_images, const float* maxes, float* targets, float st) {
  CNB_REQUIRE(g.T == 1 && g.modT == 1 && g.kt == 1, "MaxPoolRpropGemm: 2-D pooling only");
  const bool v4 = (g.N % 4 == 0) && aligned16(images) && aligned16(R_images) && aligned16(maxes) && aligned16(targets);
  const long long per_plane = (long long)g.modX * g.modY * (v4 ? g.N / 4 : g.N);
  CNB_REQUIRE(per_plane < (1LL << 30) && g.C <= 65535, "MaxPoolRpropGemm: plane too large");
  const dim3 grid((unsigned)std::max<long long>(1, std::min<long long>(ceil_div<long long>(per_plane, 256), 64)), g.C);
  if (v4) launch_pdl(pool_rprop_kernel<4>, grid, dim3(256), 0, state().stream, g, images, R_images, maxes, targets, st);
  else launch_pdl(pool_rprop_kernel<1>, grid, dim3(256), 0, state().stream, g, images, R_images, maxes, targets, st);
  count_launch();
  CNB_LAUNCH_CHECK("max_pool_rprop");
}

template <int VEC, bool MAX>
static PoolOutcome launch_undo(const PoolGeom& g, const float* images, const float* grads, const float* acts, float* targets,
                               float st, float so, const PoolEpi& epi) {
  cudaStream_t s = state().stream;
  const int planes = g.C * g.T;
  const long long per_plane = (long long)g.W * g.H * (g.N / VEC);
  CNB_REQUIRE(per_plane < (1LL << 30) && planes <= 65535, "pool_undo: plane too large");
  PoolOutcome o;
  // windows covering one element per axis: ceil(k / stride)
  const int q = (g.kt == 1 && g.T == 1 && g.modT == 1) ? std::max(ceil_div(g.kx, g.sx), ceil_div(g.ky, g.sy)) : 99;
  if (q <= 2 && per_plane * VEC < (1LL << 31)) {   // 2-D, at most 2 x 2 covering windows: the row-structured kernels
    const int sh = pow2_shift(g.N / VEC);
    o.emitted = epi.twin != nullptr;
    if (MAX && patch_geometry(g)) {
      // patches: element X belongs to patch (X - px) / 2; the first patch holds X = 0, the last X = W - 1
      const int PX = (g.W - 1 - g.px) / 2 + 1, PY = (g.H - 1 - g.py) / 2 + 1;
      o.colsum_slices = epi.colsum ? PY : 0;
      // the forward pass left tie masks for exactly this (input, output) pair and nothing wrote either since: no need to
      // reload and compare them.  A fused ReLU' mask is only expressible when it IS the pool input (bit 15 = maximum > 0).
      // (with scaleTargets != 0 the compare path also zeroes the OLD target where the mask fails; the tie masks cannot say
      // that for elements that are no window's maximum, so that combination stays on the compare path)
      const uint16_t* tm = epi.mask == nullptr || (epi.mask == images && st == 0.f)
                               ? pool_masks_find(acts, (long long)g.N * g.modX * g.modY * g.C, images, pool_sig(g)) : nullptr;
      if (tm)
        launch_pdl(pool_undo_masked_patch_kernel<VEC>, dim3((unsigned)PY, planes), dim3(256), 0, s, g, grads, tm, targets, st, so,
                   epi.mask != nullptr ? 1 : 0, sh, epi.twin, epi.colsum, PX, PY);
      else
        launch_pdl(pool_undo_patch_kernel<VEC>, dim3((unsigned)PY, planes), dim3(256), 0, s, g, images, grads, acts, targets, st,
                   so, epi.mask, sh, epi.twin, epi.colsum, PX, PY);
      return o;
    }
    o.colsum_slices = epi.colsum ? g.H : 0;
    with_const<int, 1, 2>(q, [&](auto Q) {
      with_const<int, 0, 1, 2>(row_stride(g), [&](auto S) {
        auto* kernel = epi.steps() ? pool_undo_rows_kernel<VEC, false, Q, S, true> : pool_undo_rows_kernel<VEC, MAX, Q, S, false>;
        kernel<<<dim3((unsigned)g.H, planes), 256, 0, s>>>(g, images, grads, acts, targets, st, so, epi.mask, sh, epi.twin,
                                                           epi.colsum, epi);
      });
    });
    return o;
  }
  // the flat-index kernels fuse a bare ReLU' mask: with steps to run, the caller's passes apply the mask after them
  o.fused = !epi.steps();
  const dim3 grid((unsigned)std::max<long long>(1, std::min<long long>(ceil_div<long long>(per_plane, 256), 64)), planes);
  with_const<int, 1, 2, 0>(q <= 2 ? q : 0, [&](auto Q) {
    pool_undo_kernel<VEC, MAX, Q><<<grid, 256, 0, s>>>(g, images, grads, acts, targets, st, so, o.fused ? epi.mask : nullptr);
  });
  return o;
}

PoolOutcome pool_undo(const PoolGeom& g, bool is_max, const float* images, const float* grads, const float* acts,
                      float* targets, float st, float so, const PoolEpi& epi) {
  CNB_REQUIRE(!is_max || !epi.steps(), "pool_undo: max pooling fuses no activation, dropout or scale");
  const bool v4 = (g.N % 4 == 0) && aligned16(grads) && aligned16(targets) && (!epi.mask || aligned16(epi.mask)) &&
                  (!is_max || (aligned16(images) && aligned16(acts)));
  PoolOutcome o;
  with_const<int, 1, 4>(v4 ? 4 : 1, [&](auto VEC) {
    with_const<bool, false, true>(is_max, [&](auto MAX) {
      o = launch_undo<VEC, MAX>(g, images, grads, acts, targets, st, so, epi);
    });
  });
  count_launch();
  CNB_LAUNCH_CHECK("pool_undo");
  return o;
}

}  // namespace cnb
