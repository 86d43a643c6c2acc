// rnorm.cu — cross-map response normalisation, forward and backward. HBM-bound.
//
// Replaces kCrossMapRNorm / kCrossMapDenoms / kCrossMapRNormUndo
// (cudamat_conv_gemm.cu:438-543) and kFCNorm / kFRNormUndo2
// (cudamat_conv_others.cu:1158-1300,1562-1660).
//
// One thread owns one location (n, x, y) and walks the channels at stride num_locs,
// so a warp reads/writes one full 128-byte line per channel.  The sliding window
// lives in a per-thread shared-memory ring (k entries), which makes both passes
// single-read / single-write per element:
//   forward : reads x once, writes y once                    (2 floats/element)
//   backward: reads x and dy once, writes dx once            (3 floats/element)
// The reference's backward needs a cudaMalloc'd `denoms` scratch and two kernels per
// 4096-location batch (gemm.cu:1365-1399); here it is one launch with no scratch.
// For windows too large for shared memory the ring spills to library workspace.
//
//   forward window of channel j : [j - a, j + b]  with a = k/2, b = k - k/2 - 1   (gemm.cu:475-477)
//   inverse window of channel j : [j - b, j + a]                                 (gemm.cu:528-530)
//   blocked: both are the block [ (j/k)*k, (j/k)*k + k ).
#include <cuda_bf16.h>

#include <algorithm>

#include "conv_kernels.h"

namespace cnb {

constexpr int RN_THREADS = 128;

// VEC consecutive locations per thread (16-byte accesses when VEC == 4): the scalar version spent ~70 instructions per
// channel step on one float, which makes it issue-bound; the vector version shares the ring
// bookkeeping, branches and address arithmetic between four values.
template <int VEC> __device__ __forceinline__ void rld(const float* p, float (&v)[VEC]);
template <> __device__ __forceinline__ void rld<4>(const float* p, float (&v)[4]) {
  const float4 t = __ldg(reinterpret_cast<const float4*>(p)); v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
}
template <> __device__ __forceinline__ void rld<1>(const float* p, float (&v)[1]) { v[0] = __ldg(p); }
template <int VEC> __device__ __forceinline__ void rget(const float* p, float (&v)[VEC]);      // ring (smem / scratch) read
template <> __device__ __forceinline__ void rget<4>(const float* p, float (&v)[4]) {
  const float4 t = *reinterpret_cast<const float4*>(p); v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
}
template <> __device__ __forceinline__ void rget<1>(const float* p, float (&v)[1]) { v[0] = *p; }
template <int VEC> __device__ __forceinline__ void rput(float* p, const float (&v)[VEC]);
template <> __device__ __forceinline__ void rput<4>(float* p, const float (&v)[4]) {
  *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
}
template <> __device__ __forceinline__ void rput<1>(float* p, const float (&v)[1]) { *p = v[0]; }
#define RN_V _Pragma("unroll") for (int v = 0; v < VEC; v++)

// ring element (slot, thread): ring[slot * ring_stride + lane].
// blockIdx.y selects a channel SEGMENT [f0, f1) (host: only when there are too few locations to fill the GPU); a
// segment re-reads the k-1 (forward) / 2(k-1) (backward) halo channels of its neighbours instead of waiting for them.
template <bool BLOCKED, int VEC>
__global__ void __launch_bounds__(RN_THREADS) rnorm_fwd_kernel(const float* __restrict__ x, float* __restrict__ y,
                                                                long long L, int F, int k, float alpha, float beta,
                                                                float* gring, long long gstride, int seg) {
  // L, gstride and all ring strides are in FLOATS; a thread owns floats [loc, loc + VEC)
  extern __shared__ __align__(16) float sring[];
  const long long loc = (blockIdx.x * (long long)RN_THREADS + threadIdx.x) * VEC;
  if (loc >= L) return;
  float* ring = gring ? gring + loc + (long long)blockIdx.y * k * gstride : sring + threadIdx.x * VEC;
  const long long rs = gring ? gstride : RN_THREADS * VEC;
  x += loc; y += loc;
  const int f0 = blockIdx.y * seg, f1 = min(F, f0 + seg);
  if (BLOCKED) {                                        // host guarantees seg % k == 0
    for (int s = f0; s < f1; s += k) {
      const int e = min(F, s + k);
      float sum[VEC];
      RN_V sum[v] = 0.f;
      for (int i = s; i < e; i++) {
        float t[VEC]; rld<VEC>(x + (long long)i * L, t); rput<VEC>(ring + (i - s) * rs, t);
        RN_V sum[v] += t[v] * t[v];
      }
      float sc[VEC];
      RN_V sc[v] = __powf(1.f + alpha * sum[v], -beta);
      for (int i = s; i < e; i++) {
        float t[VEC]; rget<VEC>(ring + (i - s) * rs, t);
        RN_V t[v] *= sc[v];
        rput<VEC>(y + (long long)i * L, t);
      }
    }
    return;
  }
  const int a = k / 2, b = k - a - 1;
  float sum[VEC];
  RN_V sum[v] = 0.f;
  // q = entering channel; output channel j = q - b; window [j-a, j+b] = [q-k+1, q].
  // Loads are hoisted four steps ahead of the (serial) ring updates to keep HBM requests in flight.
  constexpr int U = VEC == 4 ? 4 : 8;
  const int q0 = max(0, f0 - a), q1 = f1 + b;      // channels >= F enter as zeros
  int slot_q = q0 % k, slot_j = ((q0 - b) % k + k) % k;           // ring slots of q and of j = q - b, advanced with wrap
  for (int qb = q0; qb < q1; qb += U) {
    float xv[U][VEC];
#pragma unroll
    for (int u = 0; u < U; u++) {
      if (qb + u < F) rld<VEC>(x + (long long)(qb + u) * L, xv[u]);
      else { RN_V xv[u][v] = 0.f; }
    }
#pragma unroll
    for (int u = 0; u < U; u++) {
      const int q = qb + u;
      if (q >= q1) break;
      const int slot = slot_q;
      float old[VEC];
      RN_V old[v] = 0.f;
      if (q - q0 >= k) rget<VEC>(ring + slot * rs, old);
      if (q < F) rput<VEC>(ring + slot * rs, xv[u]);
      RN_V sum[v] += xv[u][v] * xv[u][v] - old[v] * old[v];
      const int j = q - b;
      if (j >= f0 && j < f1) {
        float xj[VEC];
        if (j == q) { RN_V xj[v] = xv[u][v]; } else rget<VEC>(ring + slot_j * rs, xj);
        RN_V xj[v] *= __powf(1.f + alpha * sum[v], -beta);
        rput<VEC>(y + (long long)j * L, xj);
      }
      if (++slot_q == k) slot_q = 0;
      if (++slot_j == k) slot_j = 0;
    }
  }
}

template <bool BLOCKED>
__global__ void __launch_bounds__(RN_THREADS) rnorm_undo_kernel(const float* __restrict__ dy, const float* __restrict__ x,
                                                                 float* __restrict__ dx, long long L, int F, int k,
                                                                 float alpha, float beta, float* gring, long long gstride,
                                                                 int seg) {
  // three rings of k entries per thread: x, t = dy*x*denom, p = dy*denom^(beta/(beta+1))
  constexpr int VEC = 1;                                 // one location per thread (launch_undo)
  extern __shared__ __align__(16) float sring[];
  const long long loc = (blockIdx.x * (long long)RN_THREADS + threadIdx.x) * VEC;
  if (loc >= L) return;
  const long long rs = gring ? gstride : RN_THREADS * VEC;
  float* rx = gring ? gring + loc + (long long)blockIdx.y * 3 * k * gstride : sring + threadIdx.x * VEC;
  float* rt = rx + (long long)k * rs;
  float* rp = rt + (long long)k * rs;
  x += loc; dy += loc; dx += loc;
  const float c2 = 2.f * alpha * beta;
  const int f0 = blockIdx.y * seg, f1 = min(F, f0 + seg);
  if (BLOCKED) {
    for (int s = f0; s < f1; s += k) {
      const int e = min(F, s + k);
      float sum[VEC];
      RN_V sum[v] = 0.f;
      for (int i = s; i < e; i++) {
        float t[VEC]; rld<VEC>(x + (long long)i * L, t); rput<VEC>(rx + (i - s) * rs, t);
        RN_V sum[v] += t[v] * t[v];
      }
      float denom[VEC], pw[VEC], st[VEC];
      RN_V { const float base = 1.f + alpha * sum[v]; denom[v] = __powf(base, -beta - 1.f); pw[v] = __powf(base, -beta); st[v] = 0.f; }
      for (int i = s; i < e; i++) {
        float g[VEC], xi[VEC]; rld<VEC>(dy + (long long)i * L, g); rget<VEC>(rx + (i - s) * rs, xi);
        rput<VEC>(rt + (i - s) * rs, g);
        RN_V st[v] += g[v] * xi[v] * denom[v];
      }
      for (int i = s; i < e; i++) {
        float g[VEC], xi[VEC]; rget<VEC>(rt + (i - s) * rs, g); rget<VEC>(rx + (i - s) * rs, xi);
        RN_V g[v] = g[v] * pw[v] - c2 * xi[v] * st[v];
        rput<VEC>(dx + (long long)i * L, g);
      }
    }
    return;
  }
  const int a = k / 2, b = k - a - 1;
  float sumsq[VEC], sumt[VEC];
  RN_V { sumsq[v] = 0.f; sumt[v] = 0.f; }
  // stage 1: entering channel q; channel i = q - b gets its forward sum, t_i and p_i
  // stage 2: output channel j = i - a gets sum of t over [j-b, j+a] = [i-k+1, i]
  const int q0 = max(0, f0 - (k - 1));                   // first x needed: (f0 - b) - a
  const int i0 = max(0, f0 - b);                         // first t needed
  const int Qend = f1 + a + b;                           // last output f1-1 needs t up to f1-1+a, i.e. q up to f1-1+a+b
  // ring slots of q, i = q - b and j = i - a, advanced with wrap instead of three `% k` per channel
  int slot_q = q0 % k, slot_i = ((q0 - b) % k + k) % k, slot_j = ((q0 - b - a) % k + k) % k;
  constexpr int U = 4;
  for (int qb = q0; qb < Qend; qb += U) {
    float xv[U][VEC], gv[U][VEC];
#pragma unroll
    for (int u = 0; u < U; u++) {
      const int q = qb + u, i = q - b;
      if (q < F) rld<VEC>(x + (long long)q * L, xv[u]); else { RN_V xv[u][v] = 0.f; }
      if (i >= i0 && i < F) rld<VEC>(dy + (long long)i * L, gv[u]); else { RN_V gv[u][v] = 0.f; }
    }
#pragma unroll
    for (int u = 0; u < U; u++) {
      const int q = qb + u;
      if (q >= Qend) break;
      const int sq = slot_q, si = slot_i, sj = slot_j;
      if (++slot_q == k) slot_q = 0;
      if (++slot_i == k) slot_i = 0;
      if (++slot_j == k) slot_j = 0;
      {
        float old[VEC];
        RN_V old[v] = 0.f;
        if (q - q0 >= k) rget<VEC>(rx + sq * rs, old);
        rput<VEC>(rx + sq * rs, xv[u]);                 // zeros once q >= F
        RN_V sumsq[v] += xv[u][v] * xv[u][v] - old[v] * old[v];
      }
      const int i = q - b;
      if (i < i0) continue;
      {
        float told[VEC], t[VEC];
        RN_V { told[v] = 0.f; t[v] = 0.f; }
        if (i - i0 >= k) rget<VEC>(rt + si * rs, told);
        if (i < F) {
          float xi[VEC], pv[VEC];
          rget<VEC>(rx + si * rs, xi);
          RN_V {
            const float base = 1.f + alpha * sumsq[v];
            const float denom = __powf(base, -beta - 1.f);
            t[v] = gv[u][v] * xi[v] * denom;
            pv[v] = gv[u][v] * denom * base;           // = g * base^(-beta)  (== denom^(beta/(beta+1)), gemm.cu:538)
          }
          rput<VEC>(rp + si * rs, pv);
        }
        rput<VEC>(rt + si * rs, t);
        RN_V sumt[v] += t[v] - told[v];
      }
      const int j = i - a;
      if (j >= f0 && j < f1) {
        float pj[VEC], xj[VEC];
        rget<VEC>(rp + sj * rs, pj); rget<VEC>(rx + sj * rs, xj);
        RN_V pj[v] -= c2 * xj[v] * sumt[v];
        rput<VEC>(dx + (long long)j * L, pj);
      }
    }
  }
}


// ------------------------------------------------------------------------------------------------
// Tile kernels (the default whenever one tile fits in shared memory).
//
// The channel walk above is a serial dependency chain per location with its loads inside the chain, which leaves the
// backward pass issue/latency-bound well below the HBM bandwidth.  Here a CTA owns a tile of TL consecutive locations x ALL
// channels and works in phases that are either fully parallel or touch shared memory only:
//   1. the whole x (and dy) tile is fetched with 16-byte cp.async — every load of the tile is in flight at once;
//   2. an exclusive prefix sum of x^2 along the channels is built in shared memory (a thread per (location, channel
//      segment); two short passes: segment totals, then the running prefix offset by the earlier segments);
//   3. every (channel, location) in parallel: S = Q[hi] - Q[lo] (the window sum as a prefix difference), base, one
//      __powf, then y (forward) or t = dy x base^(-b-1) and p = dy base^(-b) (backward);
//   4. backward only: exclusive prefix of t in place, then dx_j = p_j - 2ab x_j (R[hi'] - R[lo']) in parallel;
//   5. results leave with 16-byte stores (optionally ReLU'd, optionally also as a bf16 copy for the next conv).
// Windows (cudamat_conv_gemm.cu:475-477, 528-530): forward [i-a, i+b], inverse [j-b, j+a], a = k/2, b = k-a-1;
// blocked: both are [(i/k)k, (i/k)k + k).  Prefix differences cost ~F/k ulps of relative error on S (<= 1e-6 here).
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void rn_cp16(float* smem_dst, const float* gsrc) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void rn_cp_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

template <int TL>
__device__ __forceinline__ void rn_load_tile(float* dst, const float* __restrict__ src, long long L, long long l0, int F,
                                             int valid, bool vec) {
  if (vec && valid == TL) {
    constexpr int Q4 = TL / 4;
    for (int idx = threadIdx.x; idx < F * Q4; idx += RN_THREADS) {
      const int f = idx / Q4, c = idx - f * Q4;
      rn_cp16(dst + f * TL + 4 * c, src + (long long)f * L + l0 + 4 * c);
    }
  } else {
    for (int idx = threadIdx.x; idx < F * TL; idx += RN_THREADS) {
      const int f = idx / TL, l = idx - f * TL;
      dst[idx] = l < valid ? __ldg(src + (long long)f * L + l0 + l) : 0.f;
    }
  }
}

// exclusive prefix along channels of SQ ? v^2 : v, `src` -> `dst` (may alias), dst has F+1 rows; all 128 threads call it
template <int TL, bool SQ>
__device__ __forceinline__ void rn_prefix(const float* src, float* dst, float* segtot, int F) {
  constexpr int NSEG = RN_THREADS / TL;
  const int l = threadIdx.x % TL, s = threadIdx.x / TL;
  const int fs = (F + NSEG - 1) / NSEG, f0 = min(F, s * fs), f1 = min(F, f0 + fs);
  float tot = 0.f;
  if (NSEG > 1) {
    for (int f = f0; f < f1; f++) { const float v = src[f * TL + l]; tot += SQ ? v * v : v; }
    segtot[s * TL + l] = tot;
    __syncthreads();
    tot = 0.f;
    for (int q = 0; q < s; q++) tot += segtot[q * TL + l];
  }
  float run = tot;
  for (int f = f0; f < f1; f++) { const float v = src[f * TL + l]; dst[f * TL + l] = run; run += SQ ? v * v : v; }
  if (f1 == F && (s == NSEG - 1 || f0 < F)) dst[F * TL + l] = run;       // the segment that ends at F writes the total
  __syncthreads();
}

__device__ __forceinline__ void rn_window(int i, int F, int k, int a, int b, bool blocked, int& lo, int& hi) {
  if (blocked) { lo = (i / k) * k; hi = min(F, lo + k); }
  else { lo = max(0, i - a); hi = min(F, i + b + 1); }
}

__device__ __forceinline__ void rn_store4(float* __restrict__ out, __nv_bfloat16* __restrict__ out16, long long off, float4 r,
                                          int l, int valid, bool vec) {
  if (vec && valid >= l + 4) {
    *reinterpret_cast<float4*>(out + off) = r;
    if (out16) {
      const __nv_bfloat162 lo = __floats2bfloat162_rn(r.x, r.y), hi = __floats2bfloat162_rn(r.z, r.w);
      uint2 o; o.x = *reinterpret_cast<const uint32_t*>(&lo); o.y = *reinterpret_cast<const uint32_t*>(&hi);
      *reinterpret_cast<uint2*>(out16 + off) = o;
    }
  } else {
    const float rv[4] = {r.x, r.y, r.z, r.w};
    for (int v = 0; v < 4; v++)
      if (l + v < valid) { out[off + v] = rv[v]; if (out16) out16[off + v] = __float2bfloat16_rn(rv[v]); }
  }
}

template <int TL>
__global__ void __launch_bounds__(RN_THREADS) rnorm_fwd_tile_kernel(const float* __restrict__ x, float* __restrict__ y,
                                                                     __nv_bfloat16* __restrict__ y16, long long L, int F,
                                                                     int k, float alpha, float beta, int blocked, int relu,
                                                                     int vec) {
  pdl_wait();
  pdl_trigger();
  extern __shared__ __align__(16) float sm[];
  float* X = sm;                               // [F][TL]
  float* Q = X + (size_t)F * TL;               // [F+1][TL] exclusive prefix of x^2
  float* segtot = Q + (size_t)(F + 1) * TL;    // [128/TL][TL]
  const long long l0 = (long long)blockIdx.x * TL;
  const int valid = (int)min((long long)TL, L - l0);
  rn_load_tile<TL>(X, x, L, l0, F, valid, vec != 0);
  rn_cp_wait_all();
  __syncthreads();
  rn_prefix<TL, true>(X, Q, segtot, F);
  const int a = k / 2, b = k - a - 1;
  constexpr int Q4 = TL / 4;
  for (int idx = threadIdx.x; idx < F * Q4; idx += RN_THREADS) {
    const int f = idx / Q4, l = 4 * (idx - f * Q4);
    if (l >= valid) continue;
    int lo, hi; rn_window(f, F, k, a, b, blocked != 0, lo, hi);
    const float4 qh = *reinterpret_cast<const float4*>(Q + hi * TL + l), ql = *reinterpret_cast<const float4*>(Q + lo * TL + l);
    const float4 xv = *reinterpret_cast<const float4*>(X + f * TL + l);
    float4 r;
    r.x = xv.x * __powf(1.f + alpha * (qh.x - ql.x), -beta);
    r.y = xv.y * __powf(1.f + alpha * (qh.y - ql.y), -beta);
    r.z = xv.z * __powf(1.f + alpha * (qh.z - ql.z), -beta);
    r.w = xv.w * __powf(1.f + alpha * (qh.w - ql.w), -beta);
    if (relu) { r.x = fmaxf(r.x, 0.f); r.y = fmaxf(r.y, 0.f); r.z = fmaxf(r.z, 0.f); r.w = fmaxf(r.w, 0.f); }
    rn_store4(y, y16, (long long)f * L + l0 + l, r, l, valid, vec != 0);
  }
}

template <int TL>
__global__ void __launch_bounds__(RN_THREADS) rnorm_undo_tile_kernel(const float* __restrict__ dy, const float* __restrict__ x,
                                                                      float* __restrict__ dx, long long L, int F, int k,
                                                                      float alpha, float beta, int blocked, int vec) {
  pdl_wait();
  pdl_trigger();
  extern __shared__ __align__(16) float sm[];
  float* X = sm;                               // [F][TL]
  float* G = X + (size_t)F * TL;               // [F][TL]   dy, then p = dy * base^(-beta)
  float* Q = G + (size_t)F * TL;               // [F+1][TL] exclusive prefix of x^2
  float* T = Q + (size_t)(F + 1) * TL;         // [F+1][TL] t = dy * x * base^(-beta-1), then its exclusive prefix
  float* segtot = T + (size_t)(F + 1) * TL;
  const long long l0 = (long long)blockIdx.x * TL;
  const int valid = (int)min((long long)TL, L - l0);
  rn_load_tile<TL>(X, x, L, l0, F, valid, vec != 0);
  rn_load_tile<TL>(G, dy, L, l0, F, valid, vec != 0);
  rn_cp_wait_all();
  __syncthreads();
  rn_prefix<TL, true>(X, Q, segtot, F);
  const int a = k / 2, b = k - a - 1;
  constexpr int Q4 = TL / 4;
  for (int idx = threadIdx.x; idx < F * Q4; idx += RN_THREADS) {
    const int f = idx / Q4, l = 4 * (idx - f * Q4);
    int lo, hi; rn_window(f, F, k, a, b, blocked != 0, lo, hi);
    const float4 qh = *reinterpret_cast<const float4*>(Q + hi * TL + l), ql = *reinterpret_cast<const float4*>(Q + lo * TL + l);
    const float4 xv = *reinterpret_cast<const float4*>(X + f * TL + l), g = *reinterpret_cast<const float4*>(G + f * TL + l);
    float4 t, p;
    { const float base = 1.f + alpha * (qh.x - ql.x), den = __powf(base, -beta - 1.f); t.x = g.x * xv.x * den; p.x = g.x * den * base; }
    { const float base = 1.f + alpha * (qh.y - ql.y), den = __powf(base, -beta - 1.f); t.y = g.y * xv.y * den; p.y = g.y * den * base; }
    { const float base = 1.f + alpha * (qh.z - ql.z), den = __powf(base, -beta - 1.f); t.z = g.z * xv.z * den; p.z = g.z * den * base; }
    { const float base = 1.f + alpha * (qh.w - ql.w), den = __powf(base, -beta - 1.f); t.w = g.w * xv.w * den; p.w = g.w * den * base; }
    *reinterpret_cast<float4*>(T + f * TL + l) = t;
    *reinterpret_cast<float4*>(G + f * TL + l) = p;
  }
  __syncthreads();
  rn_prefix<TL, false>(T, T, segtot, F);
  const float c2 = 2.f * alpha * beta;
  for (int idx = threadIdx.x; idx < F * Q4; idx += RN_THREADS) {
    const int j = idx / Q4, l = 4 * (idx - j * Q4);
    if (l >= valid) continue;
    int lo, hi;                                                       // inverse window: [j-b, j+a]
    if (blocked) { lo = (j / k) * k; hi = min(F, lo + k); } else { lo = max(0, j - b); hi = min(F, j + a + 1); }
    const float4 rh = *reinterpret_cast<const float4*>(T + hi * TL + l), rl = *reinterpret_cast<const float4*>(T + lo * TL + l);
    const float4 xv = *reinterpret_cast<const float4*>(X + j * TL + l), p = *reinterpret_cast<const float4*>(G + j * TL + l);
    float4 r;
    r.x = p.x - c2 * xv.x * (rh.x - rl.x); r.y = p.y - c2 * xv.y * (rh.y - rl.y);
    r.z = p.z - c2 * xv.z * (rh.z - rl.z); r.w = p.w - c2 * xv.w * (rh.w - rl.w);
    rn_store4(dx, nullptr, (long long)j * L + l0 + l, r, l, valid, vec != 0);
  }
}

// tile width for `arrays` F-row arrays (+2 spare rows and the segment totals): the widest of 64 / 32 that lets two CTAs
// share an SM, else the widest that fits at all; 0 = no tile kernel (window walk with the ring instead)
static int pick_tile(int F, int arrays, size_t* smem_out) {
  auto bytes = [&](int tl) { return sizeof(float) * ((size_t)arrays * (F + 1) * tl + RN_THREADS); };
  // a CTA works in phases (load everything, scan, compute, store): the loads of one CTA only overlap the arithmetic of
  // ANOTHER one on the same SM, so prefer the width that leaves room for >= 3 resident CTAs, then 2, then whatever fits
  const size_t sm = 224 * 1024;
  for (int per_sm : {3, 2, 1})
    for (int tl : {64, 32})
      if (bytes(tl) + 1024 <= sm / per_sm) { *smem_out = bytes(tl); return tl; }
  return 0;
}

static constexpr size_t kMaxRingSmem = 160 * 1024;

// channel segments per location: 1 unless the location count cannot fill the GPU
static int pick_segments(long long L, int F, int k) {
  const long long blocks = ceil_div<long long>(L, RN_THREADS);
  const long long want = ceil_div<long long>(2LL * num_sms(), blocks);
  int segs = (int)std::min<long long>(want, std::max(1, F / std::max(k, 1)));      // segment >= k: halo <= 2x / 3x reads
  if (segs < 1) segs = 1;
  return segs;
}

template <int VEC>
static void launch_fwd(const float* images, float* targets, long long L, int F, int k, float alpha, float beta, bool blocked) {
  const long long owners = L / VEC;                      // threads needed
  const int blocks = (int)ceil_div<long long>(owners, RN_THREADS);
  int segs = pick_segments(owners, F, k);
  int seg = ceil_div(F, segs);
  if (blocked) seg = ceil_div(seg, k) * k;
  segs = ceil_div(F, seg);
  size_t smem = sizeof(float) * (size_t)k * RN_THREADS * VEC;
  float* gring = nullptr;
  if (smem > kMaxRingSmem) { gring = (float*)workspace(sizeof(float) * (size_t)k * L * segs); smem = 0; }
  auto kern = blocked ? rnorm_fwd_kernel<true, VEC> : rnorm_fwd_kernel<false, VEC>;
  if (smem > 48 * 1024) CNB_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kern<<<dim3(blocks, segs), RN_THREADS, smem, state().stream>>>(images, targets, L, F, k, alpha, beta, gring, L, seg);
}

template <int TL>
static void launch_fwd_tile(const float* images, float* targets, __nv_bfloat16* t16, long long L, int F, int k, float alpha,
                            float beta, bool blocked, bool relu, size_t smem, bool vec) {
  static int attr_dev_mask = 0;
  const int dev = current_device();
  if (smem > 48 * 1024 && (dev >= 31 || !((attr_dev_mask >> dev) & 1))) {
    CNB_CUDA_CHECK(cudaFuncSetAttribute(rnorm_fwd_tile_kernel<TL>, cudaFuncAttributeMaxDynamicSharedMemorySize, 224 * 1024));
    if (dev < 31) attr_dev_mask |= 1 << dev;
  }
  const long long tiles = ceil_div<long long>(L, TL);
  launch_pdl(rnorm_fwd_tile_kernel<TL>, dim3((unsigned)tiles), dim3(RN_THREADS), smem, state().stream, images, targets, t16, L, F, k,
             alpha, beta, blocked ? 1 : 0, relu ? 1 : 0, vec ? 1 : 0);
}
template <int TL>
static void launch_undo_tile(const float* outGrads, const float* inputs, float* targets, long long L, int F, int k, float alpha,
                             float beta, bool blocked, size_t smem, bool vec) {
  static int attr_dev_mask = 0;
  const int dev = current_device();
  if (smem > 48 * 1024 && (dev >= 31 || !((attr_dev_mask >> dev) & 1))) {
    CNB_CUDA_CHECK(cudaFuncSetAttribute(rnorm_undo_tile_kernel<TL>, cudaFuncAttributeMaxDynamicSharedMemorySize, 224 * 1024));
    if (dev < 31) attr_dev_mask |= 1 << dev;
  }
  const long long tiles = ceil_div<long long>(L, TL);
  launch_pdl(rnorm_undo_tile_kernel<TL>, dim3((unsigned)tiles), dim3(RN_THREADS), smem, state().stream, outGrads, inputs, targets, L,
             F, k, alpha, beta, blocked ? 1 : 0, vec ? 1 : 0);
}

void rnorm_forward(const float* images, float* targets, long long L, int F, int k, float alpha, float beta,
                   bool blocked, bool relu, __nv_bfloat16* targets_bf16) {
  CNB_REQUIRE(k >= 1 && F >= 1, "ResponseNormCrossMap");
  size_t tsmem = 0;
  const int tl = L < (1LL << 31) * 32 ? pick_tile(F, 2, &tsmem) : 0;
  if (tl) {
    const bool vec = L % 4 == 0 && aligned16(images) && aligned16(targets) &&
                     (!targets_bf16 || (reinterpret_cast<uintptr_t>(targets_bf16) & 7) == 0);
    if (tl == 64) launch_fwd_tile<64>(images, targets, targets_bf16, L, F, k, alpha, beta, blocked, relu, tsmem, vec);
    else launch_fwd_tile<32>(images, targets, targets_bf16, L, F, k, alpha, beta, blocked, relu, tsmem, vec);
    count_launch();
    CNB_LAUNCH_CHECK("rnorm_forward(tile)");
    return;
  }
  CNB_REQUIRE(!relu && !targets_bf16, "rnorm_forward: the ring fallback has no fused epilogue (callers check rnorm_can_fuse)");
  // four locations per thread only when that still leaves >= 4 blocks per SM: the channel walk is a serial dependency
  // chain, so small problems need the thread count more than the shorter instruction stream (measured: 105 -> 75 us on
  // 96 x 55 x 55 x 128, but 39 -> 47 us on 256 x 14 x 14 x 128)
  const bool wide = L % 4 == 0 && aligned16(images) && aligned16(targets) && L / 4 / RN_THREADS >= 4LL * num_sms();
  if (wide) launch_fwd<4>(images, targets, L, F, k, alpha, beta, blocked);
  else launch_fwd<1>(images, targets, L, F, k, alpha, beta, blocked);
  count_launch();
  CNB_LAUNCH_CHECK("rnorm_forward");
}

// one location per thread: the backward walk carries three rings and two dependent stages per channel, so it is
// latency-bound, and a version with four locations per thread (a quarter of the threads, 4x the shared memory per block)
// was slower when measured before the port to the H100
static void launch_undo(const float* outGrads, const float* inputs, float* targets, long long L, int F, int k, float alpha,
                        float beta, bool blocked) {
  const int blocks = (int)ceil_div<long long>(L, RN_THREADS);
  int segs = pick_segments(L, F, k);
  int seg = ceil_div(F, segs);
  if (blocked) seg = ceil_div(seg, k) * k;
  segs = ceil_div(F, seg);
  size_t smem = sizeof(float) * 3 * (size_t)k * RN_THREADS;
  float* gring = nullptr;
  if (smem > kMaxRingSmem) { gring = (float*)workspace(sizeof(float) * 3 * (size_t)k * L * segs); smem = 0; }
  auto kern = blocked ? rnorm_undo_kernel<true> : rnorm_undo_kernel<false>;
  if (smem > 48 * 1024) CNB_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kern<<<dim3(blocks, segs), RN_THREADS, smem, state().stream>>>(outGrads, inputs, targets, L, F, k, alpha, beta, gring, L, seg);
}

bool rnorm_can_fuse(int F) { size_t b; return pick_tile(F, 2, &b) != 0; }

void rnorm_undo(const float* outGrads, const float* inputs, float* targets, long long L, int F, int k,
                float alpha, float beta, bool blocked) {
  CNB_REQUIRE(k >= 1 && F >= 1, "ResponseNormCrossMapUndo");
  size_t tsmem = 0;
  const int tl = pick_tile(F, 4, &tsmem);
  if (tl) {
    const bool vec = L % 4 == 0 && aligned16(outGrads) && aligned16(inputs) && aligned16(targets);
    if (tl == 64) launch_undo_tile<64>(outGrads, inputs, targets, L, F, k, alpha, beta, blocked, tsmem, vec);
    else launch_undo_tile<32>(outGrads, inputs, targets, L, F, k, alpha, beta, blocked, tsmem, vec);
    count_launch();
    CNB_LAUNCH_CHECK("rnorm_undo(tile)");
    return;
  }
  launch_undo(outGrads, inputs, targets, L, F, k, alpha, beta, blocked);
  count_launch();
  CNB_LAUNCH_CHECK("rnorm_undo");
}

}  // namespace cnb
