// mapnorm.cu — within-map (spatial) response / contrast normalisation, forward and backward, and the RGB -> YUV colour
// transform of the reference's cudamat_conv.cuh surface.  HBM-bound.
//
// Replaces kCNorm_fewfilter / kCNorm_manyfilter / kCNorm2 (cudamat_conv_others.cu:868-1150), kRNormUndoPrelims +
// kRNormUndo / kRNormUndo2 (:1866-2100) and kRGBToYUV (:303-325).
//
// Layout (numFilters, S, S, numImages) with the images fastest: element (n, x, y, f) at n + N*(x + S*(y + S*f)).
//   forward : denoms = 1 + addScale * sum_{window(p)} meanDiffs^2,  targets = images * denoms^(-powScale)
//   backward: targets = inputs * sum_{inverse window(p)} (-2 addScale powScale * acts * outGrads / denoms)
//                       + outGrads * denoms^(-powScale)
// window(p) along each axis: [p - sizeX/2, p - sizeX/2 + sizeX) clipped to the image (kCNorm_*: startPx = -sizeX/2 + px);
// the inverse window, the pixels q whose window holds p: [p + sizeX/2 - sizeX + 1, p + sizeX/2] (kRNormUndo: startY).
// Both are [p + off, p + off + sizeX) with off = -sizeX/2 (forward) or sizeX/2 - sizeX + 1 (backward).
//
// The 2-D window sum is separable.  A CTA owns one channel plane and TI consecutive images and walks the rows of the plane
// top to bottom: each step loads one input row of the summed quantity v into shared memory, forms its ROW sums over the x
// window (a loop of sizeX over shared memory) into a ring of the last min(sizeX, S) + 1 row-sum rows, and emits the output
// row whose y window ends at that input row as the COLUMN sum over the ring (a loop of at most sizeX).  2 sizeX additions
// per element instead of the reference's sizeX^2, each input element read once, each output written once.  No atomics.
#include <algorithm>

#include "conv_kernels.h"

namespace cnb {

constexpr int MN_THREADS = 256;

template <int VEC> __device__ __forceinline__ void mld(const float* p, float (&v)[VEC]);
template <> __device__ __forceinline__ void mld<4>(const float* p, float (&v)[4]) {
  const float4 t = __ldg(reinterpret_cast<const float4*>(p)); v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
}
template <> __device__ __forceinline__ void mld<1>(const float* p, float (&v)[1]) { v[0] = __ldg(p); }
template <int VEC> __device__ __forceinline__ void mst(float* p, const float (&v)[VEC]);
template <> __device__ __forceinline__ void mst<4>(float* p, const float (&v)[4]) {
  *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
}
template <> __device__ __forceinline__ void mst<1>(float* p, const float (&v)[1]) { *p = v[0]; }

// UNDO = false: a = meanDiffs, b = images, outputs denoms (o1) and targets (o0).
// UNDO = true : a = acts, b = outGrads, c = denoms, d = inputs; output targets (o0).
// TI images per CTA (TI / VEC threads per pixel); shared memory: the input row [S][TI] and the ring [R][S][TI].
template <bool UNDO, int VEC>
__global__ void __launch_bounds__(MN_THREADS) mapnorm_kernel(const float* __restrict__ a, const float* __restrict__ b,
                                                          const float* __restrict__ c, const float* __restrict__ d,
                                                          float* __restrict__ o0, float* __restrict__ o1, int N, int S,
                                                          int sizeX, int off, int R, int TI, float alpha, float beta) {
  pdl_wait();
  pdl_trigger();
  extern __shared__ __align__(16) float msm[];
  float* row = msm;                                   // [S][TI]  v of the input row being added
  float* ring = msm + (size_t)S * TI;                 // [R][S][TI] row sums of the last R input rows (row y in slot y % R)
  const long long plane = (long long)N * S * S * blockIdx.y;
  const int n0 = blockIdx.x * TI;
  const int ni = min(TI, N - n0);                     // images of this CTA
  const int per_px = TI / VEC;                        // threads per pixel
  const int units = S * per_px;                       // VEC-wide units per row
  const float c2 = -2.f * alpha * beta;
  const int last = S - 1 + off + sizeX - 1;           // step at which the last output row (S - 1) is complete
  for (int t = 0; t <= last; t++) {
    if (t < S) {                                      // input row t: v into `row`
      for (int u = threadIdx.x; u < units; u += MN_THREADS) {
        const int x = u / per_px, i = (u - x * per_px) * VEC;
        float v[VEC];
#pragma unroll
        for (int e = 0; e < VEC; e++) v[e] = 0.f;
        if (i < ni) {
          const long long g = plane + (long long)N * (x + (long long)S * t) + n0 + i;
          if (!UNDO) {
            mld<VEC>(a + g, v);
#pragma unroll
            for (int e = 0; e < VEC; e++) v[e] = v[e] * v[e];
          } else {
            float ac[VEC], og[VEC], dn[VEC];
            mld<VEC>(a + g, ac); mld<VEC>(b + g, og); mld<VEC>(c + g, dn);
#pragma unroll
            for (int e = 0; e < VEC; e++) v[e] = ac[e] * og[e] / dn[e];
          }
        }
        mst<VEC>(row + x * TI + i, v);
      }
      __syncthreads();
      float* rs = ring + (size_t)(t % R) * S * TI;    // row sums over the x window
      for (int u = threadIdx.x; u < units; u += MN_THREADS) {
        const int x = u / per_px, i = (u - x * per_px) * VEC;
        const int x0 = max(0, x + off), x1 = min(S, x + off + sizeX);
        float s[VEC];
#pragma unroll
        for (int e = 0; e < VEC; e++) s[e] = 0.f;
        for (int xx = x0; xx < x1; xx++) {
          const float* p = row + xx * TI + i;
#pragma unroll
          for (int e = 0; e < VEC; e++) s[e] += p[e];
        }
        mst<VEC>(rs + x * TI + i, s);
      }
    }
    __syncthreads();
    const int y = t - (off + sizeX - 1);              // the output row whose y window ends at input row t
    if (y < 0 || y >= S) continue;
    const int y0 = max(0, y + off), y1 = min(S, y + off + sizeX);
    for (int u = threadIdx.x; u < units; u += MN_THREADS) {
      const int x = u / per_px, i = (u - x * per_px) * VEC;
      if (i >= ni) continue;
      float s[VEC];
#pragma unroll
      for (int e = 0; e < VEC; e++) s[e] = 0.f;
      for (int yy = y0; yy < y1; yy++) {
        const float* p = ring + ((size_t)(yy % R) * S + x) * TI + i;
#pragma unroll
        for (int e = 0; e < VEC; e++) s[e] += p[e];
      }
      const long long g = plane + (long long)N * (x + (long long)S * y) + n0 + i;
      float r[VEC];
      if (!UNDO) {
        float im[VEC], dn[VEC];
        mld<VEC>(b + g, im);
#pragma unroll
        for (int e = 0; e < VEC; e++) { dn[e] = 1.f + alpha * s[e]; r[e] = im[e] * __powf(dn[e], -beta); }
        mst<VEC>(o1 + g, dn);
      } else {
        float og[VEC], dn[VEC], in[VEC];
        mld<VEC>(b + g, og); mld<VEC>(c + g, dn); mld<VEC>(d + g, in);
#pragma unroll
        for (int e = 0; e < VEC; e++) r[e] = in[e] * (c2 * s[e]) + og[e] * __powf(dn[e], -beta);
      }
      mst<VEC>(o0 + g, r);
    }
    // the next step writes `row` (read above only before the first barrier of this step) and ring slot (t + 1) % R,
    // which is outside the y window read here: R = min(sizeX, S) + 1 slots
  }
}

static size_t mapnorm_smem(int S, int R, int TI) { return sizeof(float) * (size_t)(R + 1) * S * TI; }

// the images per CTA: 16 (four 16-byte accesses per pixel, two full 32-byte sectors) on the vector path, else 8, halved
// while the ring would not fit in shared memory
static int mapnorm_width(int S, int R, bool vec) {
  int ti = vec ? 16 : 8;
  while (ti > (vec ? 4 : 1) && mapnorm_smem(S, R, ti) > 200 * 1024) ti /= 2;
  return ti;
}

template <bool UNDO, int VEC>
static void launch_mapnorm(const float* a, const float* b, const float* c, const float* d, float* o0, float* o1, int N, int S,
                           int F, int sizeX, float alpha, float beta) {
  const int R = std::min(sizeX, S) + 1;
  const int TI = mapnorm_width(S, R, VEC == 4);
  const size_t smem = mapnorm_smem(S, R, TI);
  CNB_REQUIRE(smem <= 200 * 1024, UNDO ? "ResponseNormUndo: image too large for the row ring" : "ResponseNorm: image too large for the row ring");
  smem_opt_in(mapnorm_kernel<UNDO, VEC>, 200 * 1024);
  const int off = UNDO ? sizeX / 2 - sizeX + 1 : -(sizeX / 2);
  launch_pdl(mapnorm_kernel<UNDO, VEC>, dim3((unsigned)ceil_div(N, TI), (unsigned)F), dim3(MN_THREADS), smem, state().stream,
             a, b, c, d, o0, o1, N, S, sizeX, off, R, TI, alpha, beta);
}

void mapnorm_forward(const float* images, const float* meanDiffs, float* denoms, float* targets, int N, int S, int F,
                     int sizeX, float addScale, float powScale) {
  CNB_REQUIRE(sizeX >= 1 && S >= 1 && F >= 1 && N >= 1, "ResponseNorm");
  CNB_REQUIRE(F <= 65535, "ResponseNorm: at most 65535 channels");
  const bool vec = N % 4 == 0 && aligned16(images) && aligned16(meanDiffs) && aligned16(denoms) && aligned16(targets);
  if (vec) launch_mapnorm<false, 4>(meanDiffs, images, nullptr, nullptr, targets, denoms, N, S, F, sizeX, addScale, powScale);
  else launch_mapnorm<false, 1>(meanDiffs, images, nullptr, nullptr, targets, denoms, N, S, F, sizeX, addScale, powScale);
  count_launch();
  CNB_LAUNCH_CHECK("mapnorm_forward");
}

void mapnorm_undo(const float* outGrads, const float* denoms, const float* inputs, const float* acts, float* targets, int N,
                  int S, int F, int sizeX, float addScale, float powScale) {
  CNB_REQUIRE(sizeX >= 1 && S >= 1 && F >= 1 && N >= 1, "ResponseNormUndo");
  CNB_REQUIRE(F <= 65535, "ResponseNormUndo: at most 65535 channels");
  const bool vec = N % 4 == 0 && aligned16(outGrads) && aligned16(denoms) && aligned16(inputs) && aligned16(acts) &&
                   aligned16(targets);
  if (vec) launch_mapnorm<true, 4>(acts, outGrads, denoms, inputs, targets, nullptr, N, S, F, sizeX, addScale, powScale);
  else launch_mapnorm<true, 1>(acts, outGrads, denoms, inputs, targets, nullptr, N, S, F, sizeX, addScale, powScale);
  count_launch();
  CNB_LAUNCH_CHECK("mapnorm_undo");
}

// ---- RGB -> YUV (kRGBToYUV): per pixel and image, the 3 x 3 transform of the reference, in its expression order --------
template <int VEC>
__global__ void __launch_bounds__(256) rgb_to_yuv_kernel(const float* __restrict__ imgs, float* __restrict__ target,
                                                         long long plane, long long units) {
  pdl_wait();
  pdl_trigger();
  for (long long u = blockIdx.x * (long long)blockDim.x + threadIdx.x; u < units; u += (long long)gridDim.x * blockDim.x) {
    const long long i = u * VEC;
    float R[VEC], G[VEC], B[VEC], y[VEC], uu[VEC], vv[VEC];
    mld<VEC>(imgs + i, R); mld<VEC>(imgs + plane + i, G); mld<VEC>(imgs + 2 * plane + i, B);
#pragma unroll
    for (int e = 0; e < VEC; e++) {
      y[e] = 0.2126f * R[e] + 0.7152f * G[e] + 0.0722f * B[e];
      uu[e] = -0.09991f * R[e] + -0.33609f * G[e] + 0.436f * B[e];
      vv[e] = 0.615f * R[e] + -0.55861f * G[e] + -0.05639f * B[e];
    }
    mst<VEC>(target + i, y); mst<VEC>(target + plane + i, uu); mst<VEC>(target + 2 * plane + i, vv);
  }
}

void rgb_to_yuv(const float* images, float* targets, long long plane) {
  const bool vec = plane % 4 == 0 && aligned16(images) && aligned16(targets);
  const long long units = vec ? plane / 4 : plane;
  const unsigned blocks = (unsigned)std::max<long long>(1, std::min<long long>(ceil_div<long long>(units, 256), 16LL * num_sms()));
  if (vec) launch_pdl(rgb_to_yuv_kernel<4>, dim3(blocks), dim3(256), 0, state().stream, images, targets, plane, units);
  else launch_pdl(rgb_to_yuv_kernel<1>, dim3(blocks), dim3(256), 0, state().stream, images, targets, plane, units);
  count_launch();
  CNB_LAUNCH_CHECK("rgb_to_yuv");
}

}  // namespace cnb
