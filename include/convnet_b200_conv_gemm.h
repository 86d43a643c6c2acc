/* convnet_b200_conv_gemm.h — ABI-1: the reference's DEFAULT conv library surface
 * (USE_GEMM_KERNELS=yes, libcudamat_conv_gemm.so), re-implemented for sm_90a.
 *
 * Every entry point below replaces the reference symbol of the same name and
 * signature declared in cudamat/cudamat_conv_gemm.cuh:36-138 (definitions in
 * cudamat/cudamat_conv_gemm.cu and cudamat/cudamat_conv3d_gemm.cu); the only
 * caller in the reference is src/matrix.cc:785-1011.  All functions return void,
 * use the CURRENT device, and enqueue on the library stream (legacy default
 * stream 0 unless convnet_b200_set_stream() was called — convnet_b200_ext.h).
 * Shape errors abort() after a message on stderr (the reference assert()s);
 * CUDA errors print and exit(EXIT_FAILURE) like cudamat_conv_gemm.cu:35-42.
 *
 * Layouts: SURVEY.md Appendix A.  images (N, W, H, Cin[*T]) with N fastest;
 * filters column-major [Cout x K], K index = x + kx*(y + ky*c);
 * targets (N, modX, modY, Cout[*modT]).
 */
#ifndef CONVNET_B200_CONV_GEMM_H_
#define CONVNET_B200_CONV_GEMM_H_

#include <stdbool.h>
#include "cudamat_abi.h"

#ifdef __cplusplus
extern "C" {
#endif
#if defined(__GNUC__)
#pragma GCC visibility push(default)   /* the library is built with -fvisibility=hidden */
#endif

/* fprop.  targets = scaleTargets*targets + conv(images, filters).
 * replaces cudamat_conv_gemm.cu:1411 (-> _convUpGemm :545-682).
 * scaleTargets == 0 never reads targets. */
void convUpGemm(cudamat* images, cudamat* filters, cudamat* targets,
                Shape4D* images_shape, Shape4D* filters_shape,
                Shape4D* targets_shape, ConvDesc conv_desc, float scaleTargets);

/* dgrad.  targets = scaleTargets*targets + conv^T(derivs, filters).
 * replaces cudamat_conv_gemm.cu:1427 (-> _convDownGemm :684-825). Deterministic
 * gather formulation (the reference scatters with atomicAdd). */
void convDownGemm(cudamat* derivs, cudamat* filters, cudamat* targets,
                  Shape4D* derivs_shape, Shape4D* filters_shape,
                  Shape4D* targets_shape, ConvDesc conv_desc, float scaleTargets);

/* wgrad.  targets = scaleTargets*targets + scaleOutput * sum_{n,module} derivs (x) im2col(images).
 * replaces cudamat_conv_gemm.cu:1434 (-> _convOutpGemm :827-960). */
void convOutpGemm(cudamat* images, cudamat* derivs, cudamat* targets,
                  Shape4D* images_shape, Shape4D* derivs_shape,
                  Shape4D* targets_shape, ConvDesc conv_desc,
                  float scaleTargets, float scaleOutput);

/* per-channel ("depthwise") wgrad, cudamat_conv_gemm.cu:1441 (-> _convInnerpGemm :962-1125).
 * No C++ caller in the reference (SURVEY.md §2.3): links, prints and abort()s. */
void convInnerpGemm(cudamat* images, cudamat* derivs, cudamat* targets,
                    Shape4D* images_shape, Shape4D* derivs_shape,
                    Shape4D* targets_shape, ConvDesc conv_desc,
                    float scaleTargets, float scaleOutput);

/* Untied ("locally connected") variants: same math with one filter bank per
 * module, filters [Cout x K*modules] module-major.  replaces
 * cudamat_conv_gemm.cu:1448-1467 (conv=false path of _conv{Up,Down,Outp}Gemm). */
void localUpGemm(cudamat* images, cudamat* filters, cudamat* targets,
                 Shape4D* images_shape, Shape4D* filters_shape,
                 Shape4D* targets_shape, ConvDesc conv_desc, float scaleTargets);
void localDownGemm(cudamat* derivs, cudamat* filters, cudamat* targets,
                   Shape4D* derivs_shape, Shape4D* filters_shape,
                   Shape4D* targets_shape, ConvDesc conv_desc, float scaleTargets);
void localOutpGemm(cudamat* images, cudamat* derivs, cudamat* targets,
                   Shape4D* images_shape, Shape4D* derivs_shape,
                   Shape4D* targets_shape, ConvDesc conv_desc,
                   float scaleTargets, float scaleOutput);

/* Pooling (2-D, or 3-D when kernel_size_t/stride_t say so; T is inferred as
 * shape[3]/channels).  targets = scaleOutput * pool(images): the reference
 * kernel kPool (cudamat_conv_gemm.cu:153-200) ASSIGNS, so scaleTargets has no
 * visible effect (the pre-scale at :1169 is overwritten); kept for ABI parity.
 * Window clipped to the image; avg divides by the CLIPPED count; max starts at -2e38.
 * replaces cudamat_conv_gemm.cu:1469-1481. */
void MaxPoolGemm(cudamat* images, cudamat* targets, Shape4D* images_shape,
                 Shape4D* targets_shape, ConvDesc conv_desc, float scaleTargets,
                 float scaleOutput);
void AvgPoolGemm(cudamat* images, cudamat* targets, Shape4D* images_shape,
                 Shape4D* targets_shape, ConvDesc conv_desc, float scaleTargets,
                 float scaleOutput);

/* targets = scaleTargets*targets + sum over windows m covering the element of
 * maxGrads[m] * [images == maxActs[m]]  (ties duplicate gradient).
 * replaces cudamat_conv_gemm.cu:1483 (kMaxPoolUndo :252-300); gather form, no atomics. */
void MaxPoolUndoGemm(cudamat* images, cudamat* maxGrads, cudamat* maxActs,
                     cudamat* targets, Shape4D* images_shape,
                     Shape4D* maxGrads_shape, ConvDesc conv_desc,
                     float scaleTargets);

/* R-operator of max-pool, cudamat_conv_gemm.cu:1490. No C++ caller: abort()s. */
void MaxPoolRpropGemm(cudamat* images, cudamat* R_images, cudamat* maxActs,
                      cudamat* targets, Shape4D* images_shape,
                      Shape4D* maxGrads_shape, ConvDesc conv_desc,
                      float scaleTargets);

/* targets = scaleTargets*targets + sum over covering windows of avgGrads[m]/clippedCount(m).
 * replaces cudamat_conv_gemm.cu:1497 (kAvgPoolUndo :203-249). */
void AvgPoolUndoGemm(cudamat* avgGrads, cudamat* targets,
                     Shape4D* avgGrads_shape, Shape4D* targets_shape,
                     ConvDesc conv_desc, float scaleTargets);

/* x`factor` nearest-neighbour up-sample == avg-pool undo with scaleOutput =
 * factor^2, and its adjoint == non-overlapping avg-pool.
 * replaces cudamat_conv_gemm.cu:1503-1541. */
void UpSampleGemm(cudamat* images, cudamat* targets, Shape4D* images_shape,
                  Shape4D* targets_shape, int factor, float scaleTargets);
void DownSampleGemm(cudamat* images, cudamat* targets, Shape4D* images_shape,
                    Shape4D* targets_shape, int factor);

/* Cross-map response normalisation: y_j = x_j * (1 + addScale * sum_{i in win(j)} x_i^2)^(-powScale),
 * win(j) = [j - sizeF/2, j - sizeF/2 + sizeF) ∩ [0, numFilters) or the block
 * containing j when `blocked`.  replaces cudamat_conv_gemm.cu:1543 (kCrossMapRNorm :465-489). */
void ResponseNormCrossMapGemm(cudamat* images, cudamat* targets, int numFilters,
                              int sizeF, float addScale, float powScale,
                              bool blocked);

/* Backward of the above; ALWAYS overwrites targets, recomputes denominators
 * from `inputs`.  replaces cudamat_conv_gemm.cu:1549 (_CrossMapRNormUndo :1365-1399). */
void ResponseNormCrossMapUndoGemm(cudamat* outGrads, cudamat* inputs,
                                  cudamat* targets, int numFilters, int sizeF,
                                  float addScale, float powScale, bool blocked);

/* R-operator, cudamat_conv_gemm.cu:1556. No C++ caller: abort()s. */
void ResponseNormCrossMapRpropGemm(cudamat* images, cudamat* R_images,
                                   cudamat* targets, int numFilters, int sizeF,
                                   float addScale, float powScale, bool blocked);

/* mat *= scale (scale == 0 -> memset, never reads).  replaces cudamat_conv_gemm.cu:1562 / :44-50. */
void Scale(cudamat* mat, float scale);

/* 3-D convolution: filters (Cout, kx, ky, Cin, kt); requires padding_t == 0.
 * replaces cudamat_conv3d_gemm.cu:13-165.  Unlike the reference these do NOT
 * temporarily mutate the caller's cudamat structs. */
void convUp3DGemm(cudamat* images, cudamat* filters, cudamat* targets,
                  Shape4D* images_shape, Shape4D* filters_shape,
                  Shape4D* targets_shape, ConvDesc conv_desc, float scaleTargets);
void convDown3DGemm(cudamat* derivs, cudamat* filters, cudamat* targets,
                    Shape4D* derivs_shape, Shape4D* filters_shape,
                    Shape4D* targets_shape, ConvDesc conv_desc, float scaleTargets);
void convOutp3DGemm(cudamat* images, cudamat* derivs, cudamat* targets,
                    Shape4D* images_shape, Shape4D* derivs_shape,
                    Shape4D* targets_shape, ConvDesc conv_desc,
                    float scaleTargets, float scaleOutput);

/* Per-frame cross-map response norm, replaces cudamat_conv3d_gemm.cu:167-214. */
void ResponseNormCrossMap3DGemm(cudamat* images, cudamat* targets, int numFilters,
                                int sizeF, float addScale, float powScale,
                                bool blocked, int image_size_t);
void ResponseNormCrossMap3DUndoGemm(cudamat* outGrads, cudamat* inputs,
                                    cudamat* targets, int numFilters, int sizeF,
                                    float addScale, float powScale, bool blocked,
                                    int image_size_t);

#if defined(__GNUC__)
#pragma GCC visibility pop
#endif
#ifdef __cplusplus
}
#endif
#endif  /* CONVNET_B200_CONV_GEMM_H_ */
