/* convnet_b200_conv.h — ABI-2: the cuda-convnet2-derived surface the reference
 * builds with USE_GEMM_KERNELS=no (libcudamat_conv.so), declared in
 * cudamat/cudamat_conv.cuh:8-78.  Same math as ABI-1, different signatures for
 * pooling (no scale args), response-norm undo (takes `acts`) and wgrad
 * (partial sums).  Implemented here on the SAME sm_90a kernels as ABI-1, so the
 * reference's own restrictions (square kernels, Cin<=3 or %4, Cout%16, batch
 * multiple of 32 — cudamat_conv_filteracts.cu:1222-1240) are NOT imposed.
 */
#ifndef CONVNET_B200_CONV_H_
#define CONVNET_B200_CONV_H_

#include <stdbool.h>
#include "cudamat_abi.h"

#ifdef __cplusplus
extern "C" {
#endif
#if defined(__GNUC__)
#pragma GCC visibility push(default)   /* the library is built with -fvisibility=hidden */
#endif

/* cudamat_conv_util.cu (texture-object cache): nothing to set up on sm_90a; no-op. */
void SetupTexture(cudamat* mat);

/* replaces cudamat_conv_filteracts.cu:2085 (convUp) / :2093 (localUp). */
void convUp(cudamat* images, cudamat* filters, cudamat* targets,
            Shape4D* images_shape, Shape4D* filters_shape, Shape4D* targets_shape,
            ConvDesc conv_desc, float scaleTargets);
void localUp(cudamat* images, cudamat* filters, cudamat* targets,
             Shape4D* images_shape, Shape4D* filters_shape, Shape4D* targets_shape,
             ConvDesc conv_desc, float scaleTargets);

/* replaces cudamat_conv_imgacts.cu:2347 (convDown) / :2354 (localDown). */
void convDown(cudamat* derivs, cudamat* filters, cudamat* targets,
              Shape4D* derivs_shape, Shape4D* filters_shape, Shape4D* targets_shape,
              ConvDesc conv_desc, float scaleTargets);
void localDown(cudamat* derivs, cudamat* filters, cudamat* targets,
               Shape4D* derivs_shape, Shape4D* filters_shape, Shape4D* targets_shape,
               ConvDesc conv_desc, float scaleTargets);

/* replaces cudamat_conv_weightacts.cu:3873.  targets holds
 * ceil(modY/partialSumY)*ceil(modX/partialSumX) consecutive [Cout x K] blocks
 * (targets_shape = {Cout, kx, ky, Cin*chunks}); block id =
 * (my/partialSumY)*chunksX + mx/partialSumX (py/conv_cpu.py:119-123).
 * partialSum == 0 means "all modules" (one block). */
void convOutp(cudamat* images, cudamat* derivs, cudamat* targets,
              Shape4D* images_shape, Shape4D* derivs_shape, Shape4D* targets_shape,
              ConvDesc conv_desc, int partialSumY, int partialSumX,
              float scaleTargets, float scaleOutput);
/* replaces cudamat_conv_weightacts.cu:3881 (partial sum 1x1 == one block per module). */
void localOutp(cudamat* images, cudamat* derivs, cudamat* targets,
               Shape4D* images_shape, Shape4D* derivs_shape, Shape4D* targets_shape,
               ConvDesc conv_desc, float scaleTargets, float scaleOutput);

/* replaces cudamat_conv_others.cu:3660 / :3665.  `acts` is accepted and ignored
 * (denominators are recomputed from `inputs`); targets always overwritten. */
void ResponseNormCrossMap(cudamat* images, cudamat* targets, int numFilters,
                          int sizeF, float addScale, float powScale, bool blocked);
void ResponseNormCrossMapUndo(cudamat* outGrads, cudamat* inputs, cudamat* acts,
                              cudamat* targets, int numFilters, int sizeF,
                              float addScale, float powScale, bool blocked);

/* Within-map response / contrast normalisation (cudamat_conv_others.cu:3670-3684):
 * no Edge type reaches them (src/edge.cc:17-60) — out of scope; link, print, abort(). */
void ResponseNorm(cudamat* images, cudamat* denoms, cudamat* targets,
                  int numFilters, int sizeX, float addScale, float powScale);
void ResponseNormUndo(cudamat* outGrads, cudamat* denoms, cudamat* inputs,
                      cudamat* acts, cudamat* targets, int numFilters, int sizeX,
                      float addScale, float powScale);
void ContrastNorm(cudamat* images, cudamat* meanDiffs, cudamat* denoms,
                  cudamat* targets, int numFilters, int sizeX, float addScale,
                  float powScale);
void ContrastNormUndo(cudamat* outGrads, cudamat* denoms, cudamat* meanDiffs,
                      cudamat* acts, cudamat* targets, int numFilters, int sizeX,
                      float addScale, float powScale);

/* replaces cudamat_conv_others.cu:3686-3711: overwrite, scaleOutput = 1. */
void MaxPool(cudamat* images, cudamat* targets, Shape4D* images_shape,
             Shape4D* targets_shape, ConvDesc conv_desc);
void AvgPool(cudamat* images, cudamat* targets, Shape4D* images_shape,
             Shape4D* targets_shape, ConvDesc conv_desc);
void MaxPoolUndo(cudamat* images, cudamat* maxGrads, cudamat* maxActs,
                 cudamat* targets, Shape4D* images_shape, Shape4D* maxGrads_shape,
                 ConvDesc conv_desc, float scaleTargets);
void AvgPoolUndo(cudamat* avgGrads, cudamat* targets, Shape4D* avgGrads_shape,
                 Shape4D* targets_shape, ConvDesc conv_desc, float scaleTargets);

/* replaces cudamat_conv_others.cu:3713-3755. */
void UpSample(cudamat* images, cudamat* targets, Shape4D* images_shape,
              Shape4D* targets_shape, int factor, float scaleTargets);
void DownSample(cudamat* images, cudamat* targets, Shape4D* images_shape,
                Shape4D* targets_shape, int factor);

/* cudamat_conv_others.cu:3757: out of scope (RGBToYUVEdge uses a 3x3 dot); abort()s. */
void RGBToYUV(cudamat* images, cudamat* targets);

#if defined(__GNUC__)
#pragma GCC visibility pop
#endif
#ifdef __cplusplus
}
#endif
#endif  /* CONVNET_B200_CONV_H_ */
