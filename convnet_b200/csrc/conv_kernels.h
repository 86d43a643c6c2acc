// conv_kernels.h — host-side entry points of the kernel translation units.
#pragma once
#include <cuda_bf16.h>

#include "common.cuh"
#include "geom.h"

namespace cnb {

// conv_simt.cu — fp32 CUDA-core implicit GEMM (exact mode + shapes the tensor path skips)
void simt_conv_up(const ConvGeom& g, const float* images, const float* filters, float* targets,
                  float scaleTargets, float scaleOutput, const Fuse& fuse);
void simt_conv_down(const ConvGeom& g, const float* derivs, const float* filters, float* targets,
                    float scaleTargets, float scaleOutput, const Fuse& fuse);
// rectH x rectW: module rectangle per reduction chunk; keep_partials: one output block per chunk
void simt_conv_outp(const ConvGeom& g, const float* images, const float* derivs, float* targets,
                    int rectH, int rectW, bool keep_partials, float scaleTargets, float scaleOutput);
void scale_buffer(float* a, long long n, float s);
void reduce_partials(const float* part, float* out, long long elems, int groups, int per, float st, float so);

// conv_tc.cu — TMA-fed implicit GEMM on the sm_90a tensor cores (wgmma bf16, mma.sync tf32)
// What a tensor-core call did: the path it took (kPathNone: it declined the call), whether its kernel wrote the bf16 twin
// `targets_bf16` it was handed, and whether it applied the requested dropout itself.
struct ConvOutcome { int path = kPathNone; bool emitted = false, dropped = false; };
ConvOutcome tc_conv_up(const ConvGeom& g, const float* images, const float* filters, float* targets,
                       float scaleTargets, float scaleOutput, const Fuse& fuse, __nv_bfloat16* targets_bf16);
void dropout_apply(float* x, long long n, float dropprob, float scale, unsigned long long seed, __nv_bfloat16* out16);   // elementwise.cu
void tc_conv_down_prestage(const ConvGeom& g, const float* derivs, const float* filters);   // builds the dgrad filter banks, if that path will run
ConvOutcome tc_conv_down(const ConvGeom& g, const float* derivs, const float* filters, float* targets,
                         float scaleTargets, float scaleOutput, const Fuse& fuse, __nv_bfloat16* targets_bf16);
ConvPath tc_conv_outp(const ConvGeom& g, const float* images, const float* derivs, float* targets,
                      float scaleTargets, float scaleOutput);                  // kPathNone: declined

// stage.cu — bf16 operand copies and their coherence (convnet_b200_bf16_stage / _ensure / _invalidate / emit)
bool want_bf16();
void to_bf16(const float* src, __nv_bfloat16* dst, long long n);
const __nv_bfloat16* bf16_staged(const float* src, long long n);      // valid copy covering [src, src+n), or nullptr
void bf16_stage(const float* ptr, long long n);                        // convert now
void bf16_ensure(const float* ptr, long long n);                       // convert unless a valid copy exists
void bf16_invalidate(const float* ptr);
void bf16_note_write(const float* ptr, long long n);                   // [ptr, ptr+n) is being overwritten: overlapping copies go stale
__nv_bfloat16* bf16_emit_slot(const float* ptr, long long n);          // buffer a producing kernel fills itself (marked valid)
__nv_bfloat16* bf16_refresh_slot(const float* ptr, long long n);       // the existing buffer of exactly this tensor, or nullptr
void bf16_release();                                                   // drops the buffers too
// dgrad in fprop form (stage.cu): stride phases and the per-phase filter banks [c][tap''][o]
constexpr int kMaxDgradPhases = 16;
struct DgradPhase {
  int a, b;            // input pixel phase: x = sx*i + a, y = sy*j + b
  int rx, ry;          // tap residues: tx = rx + sx*u
  int ku, kv;          // taps of this phase
  int px, py;          // (negative) window start offsets of the stride-1 correlation over the derivative
  int Wp, Hp;          // pixels of this phase
  long long offset;    // element offset of the phase's bank
};
struct DgradBanks { int count; DgradPhase phase[kMaxDgradPhases]; };
int dgrad_phases(const ConvGeom& g, DgradBanks* b);                    // number of phases, or -1 if there are too many
// built on first use and cached per (filters, geometry); `prestage`: the build is a prestage request's (counted apart)
const __nv_bfloat16* dgrad_weights(const float* filters, const ConvGeom& g, const DgradBanks& b, bool prestage);
// max-pool tie masks (stage.cu), see pool.cu
uint16_t* pool_masks_slot(const float* acts, long long n_out, const float* images, long long n_in, unsigned long long sig);
const uint16_t* pool_masks_find(const float* acts, long long n_out, const float* images, unsigned long long sig);
// Writer protocol of every entry point that writes a tensor: construction drops the staged bf16 copies overlapping the
// target.  When the caller asked for a fresh copy (`want`, convnet_b200_emit_bf16_next) and the kernel can write it, `buf`
// is the twin it fills (nullptr outside bf16 mode), and the caller sets `done` once a kernel has filled it; finish()
// converts in a trailing pass when nobody did.
struct Emit {
  float* target; long long n; bool want; __nv_bfloat16* buf = nullptr; bool done = false;
  Emit(float* target, long long n, bool want, bool kernel_can_emit = true);
  void finish();
};

// pool.cu
// Everything a pool call may fuse into the tensor it writes; the default fuses nothing.  Each result, after scaleOutput
// (and after scaleTargets * old for an undo), goes through the steps, in the order of the stand-alone passes they replace
// and bit-identical to them: relu: max(., 0) (cnb_relu); dropout (drop_scale != 0): times the keep value of cnb_dropout at
// the element's index; times `scale` (cnb_mult); then the ReLU' mask: zeroed where mask[i] <= 0 (cnb_relu_deriv).  The
// stored values then give colsum[slice * planes + plane], per-(row slice, plane) sums — the bias gradient of the edge
// below, finished by colsum_finish — and the bf16 twin.  cache_masks (max forward): record the tie masks its undo reads.
//   - Max pooling takes no steps, and its forward no mask or colsum either (a request that does is refused).
//   - The row and patch kernels (2-D, windows up to 3 wide, or covered by at most 2 x 2 windows for an undo) apply it all.
//   - The flat-index kernels apply none of it, except that the undo applies a mask when there are no steps.
// What the call did: `emitted`: its kernel wrote the twin; `colsum_slices`: the slices of colsum it wrote (0: none);
// `fused`: it applied the steps and the mask.  When fused is false it applied none of them, nor the twin or colsum: the
// caller runs the steps and the mask as passes, in the order above, then sums and converts the result.
struct PoolEpi {
  int relu = 0;
  float drop_prob = 0.f, drop_scale = 0.f; unsigned long long drop_seed = 0;
  float scale = 1.f;
  const float* mask = nullptr;
  float* colsum = nullptr;
  __nv_bfloat16* twin = nullptr;
  bool cache_masks = false;
  bool steps() const { return relu || drop_scale != 0.f || scale != 1.f; }
};
struct PoolOutcome { bool emitted = false; bool fused = true; int colsum_slices = 0; };
PoolOutcome pool_forward(const PoolGeom& g, bool is_max, const float* images, float* targets, float scaleOutput,
                         const PoolEpi& epi);
// images and acts (the pool input and output) are read by max pooling only
PoolOutcome pool_undo(const PoolGeom& g, bool is_max, const float* images, const float* grads, const float* acts,
                      float* targets, float scaleTargets, float scaleOutput, const PoolEpi& epi);
// max-pool R-operator: targets = st * targets + sum of R_images over the window elements equal to the stored maximum
void max_pool_rprop(const PoolGeom& g, const float* images, const float* R_images, const float* maxes, float* targets, float st);
// grad_bias[c] = st*grad_bias[c] + so * sum_slices part[slice*cols + c]   (elementwise.cu)
void colsum_finish(const float* part, float* grad_bias, int cols, int slices, float st, float so);

// rnorm.cu — each call runs the tile kernel when one tile of numFilters channels fits in shared memory, else the ring
// kernel.  The forward may fuse max(., 0) (`relu`) and write the bf16 twin `targets_bf16` (nullptr: none).  It returns
// whether it did: true from the tile kernel, which applies both; false from the ring kernel, which applies neither, and
// the caller then runs the ReLU and converts the twin as passes.
bool rnorm_forward(const float* images, float* targets, long long num_locs, int numFilters, int sizeF,
                   float addScale, float powScale, bool blocked, bool relu, __nv_bfloat16* targets_bf16);
void rnorm_undo(const float* outGrads, const float* inputs, float* targets, long long num_locs,
                int numFilters, int sizeF, float addScale, float powScale, bool blocked);
// R-operator: t_j = R_j d_j^-b - 2ab x_j d_j^(-b-1) sum_{i in window(j)} x_i R_i,  d_j = 1 + a sum_{i in window(j)} x_i^2
void rnorm_rprop(const float* images, const float* R_images, float* targets, long long num_locs, int numFilters, int sizeF,
                 float addScale, float powScale, bool blocked);

// mapnorm.cu — within-map normalisation over sizeX x sizeX windows of square S x S maps, and the colour transform
void mapnorm_forward(const float* images, const float* meanDiffs, float* denoms, float* targets, int N, int S, int F,
                     int sizeX, float addScale, float powScale);
void mapnorm_undo(const float* outGrads, const float* denoms, const float* inputs, const float* acts, float* targets, int N,
                  int S, int F, int sizeX, float addScale, float powScale);
void rgb_to_yuv(const float* images, float* targets, long long plane);   // plane = pixels x images per colour

// conv_simt.cu — filter-tap inner products of convInnerpGemm: targets[tap] = st * targets[tap] + so * sum over images,
// modules and channels c of image(tap at the module, c) * derivs(module, c); `splits` partial sums (0: chosen here)
int conv_innerp(const ConvGeom& g, const float* images, const float* derivs, float* targets, float st, float so, int splits = 0);

}  // namespace cnb
