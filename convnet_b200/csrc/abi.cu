// abi.cu — the extern "C" surface: ABI-1 (include/convnet_b200_conv_gemm.h, the
// reference's cudamat_conv_gemm.cuh) and ABI-2 (include/convnet_b200_conv.h, the
// reference's cudamat_conv.cuh), both on the same kernels.
#include <nvtx3/nvToolsExt.h>

#include <algorithm>

#include "../../include/convnet_b200_conv.h"
#include "../../include/convnet_b200_conv_gemm.h"
#include "../../include/convnet_b200_ext.h"
#include "conv_kernels.h"

using namespace cnb;

namespace {

ConvDesc as_2d(ConvDesc d) { d.kernel_size_t = 1; d.stride_t = 1; d.padding_t = 0; return d; }

// one NVTX range per C-ABI entry (named after the entry point), so an nsys / ncu timeline of a host application shows
// which reference call every kernel belongs to; header-only NVTX3: a no-op costing a few ns when no tool is attached
struct Range {
  explicit Range(const char* name) { nvtxRangePushA(name); }
  ~Range() { nvtxRangePop(); }
};

// ---- dispatch: tensor-core path when the mode and the shape allow, else fp32 CUDA cores; every write follows the writer
// protocol (Emit, stage.cu)

// bias gradient requested with the write (convnet_b200_fuse_next_bias_grad): finish from the kernel's per-slice sums, or
// run the column-sum pass when the kernel did not produce them.  rows = images x positions, cols = channels.
void finish_bias_grad(const Fuse& fuse, const float* part, int slices, const float* target, long long rows, int cols) {
  if (!fuse.bias_grad) return;
  if (slices > 0) colsum_finish(part, fuse.bias_grad, cols, slices, fuse.bg_st, fuse.bg_so);
  else cnb_channel_bias_grad(target, fuse.bias_grad, rows, cols, fuse.bg_st, fuse.bg_so);
}

void conv_up(const ConvGeom& g, const float* images, const float* filters, float* targets, float st, float so) {
  const Fuse fuse = take_fuse();
  CNB_REQUIRE(!fuse.bias_grad, "convUp: a fused bias gradient belongs to a backward call");
  Emit emit(targets, g.out_total, fuse.emit_bf16 != 0);
  ConvOutcome r;
  if (state().precision != kPrecFP32) r = tc_conv_up(g, images, filters, targets, st, so, fuse, emit.buf);
  if (r.path == kPathNone) {
    simt_conv_up(g, images, filters, targets, st, so, fuse);
    r.path = kPathSimt;
  }
  state().last_conv_path = r.path;
  emit.done = r.emitted;
  if (fuse.drop_scale != 0.f && !r.dropped) {      // the kernel could not apply the dropout: one pass, which also (re)writes the bf16 twin
    dropout_apply(targets, g.out_total, fuse.drop_prob, fuse.drop_scale, fuse.drop_seed, emit.buf);
    emit.done = true;
  }
  emit.finish();
}

void conv_down(const ConvGeom& g, const float* derivs, const float* filters, float* targets, float st, float so) {
  Fuse fuse = take_fuse();
  if (fuse.prestage) {                             // filters-only preparation of this call (convnet_b200_prestage_next)
    if (state().precision != kPrecFP32) tc_conv_down_prestage(g, derivs, filters);
    return;
  }
  so *= fuse.out_scale;
  // the mask can ride in the epilogue only when one launch produces the final value of every target element
  const bool whole = g.conv && g.frames == 1 && g.cin0 == 0 && g.Cin == g.CinT;
  const float* late_mask = nullptr;
  const int late_act = fuse.state_act;
  if (fuse.act_state && !whole) { late_mask = fuse.act_state; fuse.act_state = nullptr; fuse.state_act = kActNone; }
  // a late mask changes the values after the kernel: convert afterwards
  Emit emit(targets, g.img_total, fuse.emit_bf16 != 0, !late_mask);
  ConvOutcome r;
  if (state().precision != kPrecFP32) r = tc_conv_down(g, derivs, filters, targets, st, so, fuse, emit.buf);
  if (r.path == kPathNone) {
    simt_conv_down(g, derivs, filters, targets, st, so, fuse);
    r.path = kPathSimt;
  }
  state().last_conv_path = r.path;
  emit.done = r.emitted;
  if (late_mask) {
    const long long n4 = g.img_total;             // (these passes would consume a pending fuse request; none is pending here)
    if (late_act == kActLogistic) cnb_logistic_deriv(targets, late_mask, n4);
    else cnb_relu_deriv(targets, late_mask, n4);
  }
  CNB_REQUIRE(!fuse.bias_grad || g.frames == 1, "convDown: fused bias gradient is 2-D only");
  finish_bias_grad(fuse, nullptr, 0, targets, (long long)g.N * g.W * g.H, g.CinT);
  emit.finish();
}

// reduction split for the CUDA-core wgrad: enough (tile x chunk) blocks to fill the GPU
void simt_outp_auto(const ConvGeom& g, const float* images, const float* derivs, float* targets, float st, float so) {
  const long long tiles = (long long)ceil_div(g.Cout, 128) * ceil_div(g.K, 128);
  const long long want = std::max<long long>(1, (4LL * num_sms()) / tiles);
  long long chunksY = std::min<long long>(g.modY, std::max<long long>(1, want / g.frames));
  // keep the partial-sum scratch below 1 GiB
  const long long elems = (long long)g.Cout * g.K;
  while (chunksY > 1 && elems * chunksY * g.frames * 4 > (1LL << 30)) chunksY--;
  const int rectH = (int)ceil_div<long long>(g.modY, chunksY);
  simt_conv_outp(g, images, derivs, targets, rectH, g.modX, false, st, so);
}

void conv_outp(const ConvGeom& g, const float* images, const float* derivs, float* targets, float st, float so) {
  take_fuse();                                 // a wgrad call has no epilogue to fuse: a pending request must not leak to a later call
  ConvPath path = kPathNone;
  if (state().precision != kPrecFP32) path = tc_conv_outp(g, images, derivs, targets, st, so);
  if (path == kPathNone) {
    if (!g.conv) simt_conv_outp(g, images, derivs, targets, 1, 1, true, st, so);   // untied: one [Cout x K] block per module
    else simt_outp_auto(g, images, derivs, targets, st, so);
    path = kPathSimt;
  }
  state().last_conv_path = path;
}

void do_conv_up(const char* what, cudamat* images, cudamat* filters, cudamat* targets, Shape4D* is, Shape4D* fs,
                Shape4D* ts, ConvDesc d, float st, bool conv) {
  Range nvtx_range(what);
  ConvGeom g = conv_geom(*is, *fs, *ts, images, filters, targets, d, conv, what);
  conv_up(g, images->data_device, filters->data_device, targets->data_device, st, 1.f);
}
void do_conv_down(const char* what, cudamat* derivs, cudamat* filters, cudamat* targets, Shape4D* ds, Shape4D* fs,
                  Shape4D* ts, ConvDesc d, float st, bool conv) {
  Range nvtx_range(what);
  ConvGeom g = conv_geom(*ts, *fs, *ds, targets, filters, derivs, d, conv, what);
  conv_down(g, derivs->data_device, filters->data_device, targets->data_device, st, 1.f);
}
void do_conv_outp(const char* what, cudamat* images, cudamat* derivs, cudamat* targets, Shape4D* is, Shape4D* ds,
                  Shape4D* ts, ConvDesc d, float st, float so, bool conv) {
  Range nvtx_range(what);
  ConvGeom g = conv_geom(*is, *ts, *ds, images, targets, derivs, d, conv, what);
  conv_outp(g, images->data_device, derivs->data_device, targets->data_device, st, so);
}

// A pool call's request split into the PoolEpi its kernel is asked to fuse and the passes that follow the kernel whatever
// it did: sigma with the dropout after it (late_act) and sigma' (late_state), which no pool kernel applies.  When a late
// pass is to change the values, the bf16 twin and the bias-gradient sums wait for it too.  Max pooling honours no
// activation, dropout or scale request, and its forward pass no derivative or bias-gradient request either.
// colsum_floats: the workspace the kernel's per-slice channel sums need (0: the call is 3-D and a pass sums them).
struct PoolRequest {
  Fuse fuse;                                       // the request as the call honours it
  PoolEpi epi;
  bool late_act = false, late_state = false;
};
PoolRequest pool_request(Fuse f, bool is_max, bool undo, __nv_bfloat16* twin, size_t colsum_floats) {
  if (is_max) {
    f.act = kActNone; f.drop_scale = 0.f; f.out_scale = 1.f;
    if (!undo) { f.act_state = nullptr; f.state_act = kActNone; f.bias_grad = nullptr; }
  }
  PoolRequest r;
  const int act = f.act_state ? kActNone : f.act;   // (a request with a state is the derivative's)
  r.late_act = act == kActLogistic;
  r.late_state = f.state_act == kActLogistic;
  r.epi.relu = act == kActRelu;
  if (!r.late_act) { r.epi.drop_prob = f.drop_prob; r.epi.drop_scale = f.drop_scale; r.epi.drop_seed = f.drop_seed; }
  r.epi.scale = f.out_scale;
  r.epi.mask = f.relu_mask();
  r.epi.cache_masks = f.pool_cache != 0;
  if (!r.late_act && !r.late_state) {
    r.epi.twin = twin;
    if (f.bias_grad && colsum_floats) r.epi.colsum = (float*)workspace(sizeof(float) * colsum_floats);
  }
  r.fuse = f;
  return r;
}
// the end of every pool call: the steps and the mask as passes when the kernel applied none of them (the order of
// PoolEpi, bit-identical), the late passes, the bias gradient of `rows` x `channels` from the kernel's sums or a
// column-sum pass, and the twin where no kernel wrote it
void finish_pool(const PoolRequest& r, const PoolOutcome& o, Emit& emit, long long rows, int channels) {
  float* t = emit.target;
  const long long n = emit.n;
  const PoolEpi& e = r.epi;
  if (!o.fused) {
    if (e.relu) cnb_relu(t, n);
    if (e.drop_scale != 0.f) dropout_apply(t, n, e.drop_prob, e.drop_scale, e.drop_seed, nullptr);
    if (e.scale != 1.f) scale_buffer(t, n, e.scale);
    if (e.mask) cnb_relu_deriv(t, e.mask, n);
  }
  if (r.late_act) {
    cnb_logistic(t, n);
    if (r.fuse.drop_scale != 0.f) dropout_apply(t, n, r.fuse.drop_prob, r.fuse.drop_scale, r.fuse.drop_seed, nullptr);
  }
  if (r.late_state) cnb_logistic_deriv(t, r.fuse.act_state, n);
  finish_bias_grad(r.fuse, e.colsum, o.colsum_slices, t, rows, channels);
  emit.done = o.emitted;
  emit.finish();
}

void do_pool(const char* what, bool is_max, cudamat* images, cudamat* targets, Shape4D* is, Shape4D* ts, ConvDesc d,
             float so) {
  Range nvtx_range(what);
  PoolGeom g = pool_geom(*is, *ts, images, targets, d, what);
  const Fuse fuse = take_fuse();
  Emit emit(targets->data_device, (long long)targets->size[0] * targets->size[1], fuse.emit_bf16 != 0);
  const PoolRequest r = pool_request(fuse, is_max, false, emit.buf, g.T == 1 ? (size_t)(g.modY + 2) * g.C * g.modT : 0);
  const PoolOutcome o = pool_forward(g, is_max, images->data_device, targets->data_device, so, r.epi);
  finish_pool(r, o, emit, (long long)g.N * g.modX * g.modY * g.modT, g.C);
}
// is: the shape of the pool input, which the undo writes; images and acts (the pool input and output): max pooling only
void do_pool_undo(const char* what, bool is_max, cudamat* images, cudamat* grads, cudamat* acts, cudamat* targets,
                  Shape4D* is, Shape4D* gs, ConvDesc d, float st, float so) {
  Range nvtx_range(what);
  PoolGeom g = pool_geom(*is, *gs, targets, grads, d, what);
  if (is_max) {
    CNB_REQUIRE(images->size[0] == g.N && images->size[1] == targets->size[1], what);
    CNB_REQUIRE(acts->size[0] == g.N && acts->size[1] == grads->size[1], what);
  }
  const Fuse fuse = take_fuse();
  Emit emit(targets->data_device, (long long)targets->size[0] * targets->size[1], fuse.emit_bf16 != 0);
  const PoolRequest r = pool_request(fuse, is_max, true, emit.buf, g.T == 1 ? (size_t)(g.H + 2) * g.C * g.T : 0);
  const PoolOutcome o = pool_undo(g, is_max, is_max ? images->data_device : nullptr, grads->data_device,
                                  is_max ? acts->data_device : nullptr, targets->data_device, st, so, r.epi);
  finish_pool(r, o, emit, (long long)g.N * g.W * g.H * g.T, g.C);
}

ConvDesc sample_desc(Shape4D* is, Shape4D* ts, int factor) {      // gemm.cu:1503-1541
  ConvDesc d;
  d.kernel_size_y = d.kernel_size_x = factor; d.kernel_size_t = 1;
  d.stride_y = d.stride_x = factor; d.stride_t = 1;
  d.padding_y = d.padding_x = d.padding_t = 0;
  d.num_input_channels = is->shape[3]; d.num_output_channels = ts->shape[3];
  d.input_channel_begin = d.output_channel_begin = 0;
  d.input_channel_end = is->shape[3]; d.output_channel_end = ts->shape[3];
  d.num_groups = 1;
  return d;
}

void do_rnorm(const char* what, cudamat* images, cudamat* targets, int F, int sizeF, float a, float b, bool blocked,
              int frames) {
  Range nvtx_range(what);
  CNB_REQUIRE(F > 0 && frames > 0, what);
  const long long els = (long long)images->size[0] * images->size[1];
  CNB_REQUIRE(els % ((long long)F * frames) == 0, what);
  CNB_REQUIRE(targets->size[0] == images->size[0] && targets->size[1] == images->size[1], what);
  const long long L = els / F / frames;          // locations per frame
  // fused epilogue (convnet_b200_fuse_next relu / convnet_b200_emit_bf16_next): in the tile kernel when it applies, else
  // as trailing passes; the logistic activation is always a trailing pass
  const Fuse fuse = take_fuse();
  const bool fusable = rnorm_can_fuse(F) && fuse.act != kActLogistic;
  const bool relu = fuse.act == kActRelu;
  Emit emit(targets->data_device, els, fuse.emit_bf16 != 0);
  for (int t = 0; t < frames; t++)               // conv3d_gemm.cu:167-189: independent per frame
    rnorm_forward(images->data_device + (long long)t * L * F, targets->data_device + (long long)t * L * F, L, F, sizeF,
                  a, b, blocked, fusable && relu, fusable && emit.buf ? emit.buf + (long long)t * L * F : nullptr);
  if (relu && !fusable) cnb_relu(targets->data_device, els);
  if (fuse.act == kActLogistic) cnb_logistic(targets->data_device, els);
  emit.done = fusable;
  emit.finish();
}
void do_rnorm_undo(const char* what, cudamat* outGrads, cudamat* inputs, cudamat* targets, int F, int sizeF, float a,
                   float b, bool blocked, int frames) {
  Range nvtx_range(what);
  CNB_REQUIRE(F > 0 && frames > 0, what);
  const long long els = (long long)inputs->size[0] * inputs->size[1];
  CNB_REQUIRE(els % ((long long)F * frames) == 0, what);
  CNB_REQUIRE(targets->size[0] == inputs->size[0] && targets->size[1] == inputs->size[1], what);
  CNB_REQUIRE(outGrads->size[0] == inputs->size[0] && outGrads->size[1] == inputs->size[1], what);
  const long long L = els / F / frames;
  const Fuse fuse = take_fuse();
  CNB_REQUIRE(!fuse.bias_grad, "ResponseNormCrossMapUndo: no fused bias gradient here");
  Emit emit(targets->data_device, els, fuse.emit_bf16 != 0, false);
  for (int t = 0; t < frames; t++)
    rnorm_undo(outGrads->data_device + (long long)t * L * F, inputs->data_device + (long long)t * L * F,
               targets->data_device + (long long)t * L * F, L, F, sizeF, a, b, blocked);
  emit.finish();
}

// ---- the R-operators, within-map normalisation, the colour transform and the tap inner products: kernels that cannot
// write a bf16 twin, so a requested copy is converted after them (Emit::finish) and every other tensor they write has its
// staged copies dropped (bf16_note_write)

// both matrices hold `n` floats as (rows, cols) and are not transposed
bool same_shape(const cudamat* a, const cudamat* b) {
  return a->size[0] == b->size[0] && a->size[1] == b->size[1] && !a->is_trans && !b->is_trans;
}

void do_max_rprop(const char* what, cudamat* images, cudamat* R_images, cudamat* maxes, cudamat* targets, Shape4D* is,
                  Shape4D* ms, ConvDesc d, float st) {
  Range nvtx_range(what);
  PoolGeom g = pool_geom(*is, *ms, images, maxes, as_2d(d), what);
  CNB_REQUIRE(same_shape(R_images, images), what);
  CNB_REQUIRE(same_shape(targets, maxes), what);
  const Fuse fuse = take_fuse();
  Emit emit(targets->data_device, (long long)targets->size[0] * targets->size[1], fuse.emit_bf16 != 0, false);
  max_pool_rprop(g, images->data_device, R_images->data_device, maxes->data_device, targets->data_device, st);
  emit.finish();
}

void do_rnorm_rprop(const char* what, cudamat* images, cudamat* R_images, cudamat* targets, int F, int sizeF, float a,
                    float b, bool blocked) {
  Range nvtx_range(what);
  CNB_REQUIRE(F > 0 && sizeF >= 1, what);
  const long long els = (long long)images->size[0] * images->size[1];
  CNB_REQUIRE(els % F == 0, what);
  CNB_REQUIRE(same_shape(R_images, images) && same_shape(targets, images), what);
  const Fuse fuse = take_fuse();
  Emit emit(targets->data_device, els, fuse.emit_bf16 != 0, false);
  rnorm_rprop(images->data_device, R_images->data_device, targets->data_device, els / F, F, sizeF, a, b, blocked);
  emit.finish();
}

// the (numFilters, S, S, numImages) geometry of the cudamat_conv.cuh norms: square maps (convContrastNorm's assert)
int map_side(const char* what, const cudamat* m, int F) {
  CNB_REQUIRE(F > 0 && m->size[1] % F == 0, what);
  const int pixels = m->size[1] / F;
  int S = 0;
  while ((long long)(S + 1) * (S + 1) <= pixels) S++;
  CNB_REQUIRE((long long)S * S == pixels, what);          // square images only
  CNB_REQUIRE(!m->is_trans, what);
  return S;
}

void do_mapnorm(const char* what, cudamat* images, cudamat* meanDiffs, cudamat* denoms, cudamat* targets, int F, int sizeX,
                float a, float b) {
  Range nvtx_range(what);
  const int S = map_side(what, images, F);
  CNB_REQUIRE(sizeX >= 1, what);
  CNB_REQUIRE(same_shape(meanDiffs, images) && same_shape(denoms, images) && same_shape(targets, images), what);
  const Fuse fuse = take_fuse();
  const long long n = (long long)images->size[0] * images->size[1];
  bf16_note_write(denoms->data_device, n);
  Emit emit(targets->data_device, n, fuse.emit_bf16 != 0, false);
  mapnorm_forward(images->data_device, meanDiffs->data_device, denoms->data_device, targets->data_device, images->size[0], S,
                  F, sizeX, a, b);
  emit.finish();
}

void do_mapnorm_undo(const char* what, cudamat* outGrads, cudamat* denoms, cudamat* inputs, cudamat* acts, cudamat* targets,
                     int F, int sizeX, float a, float b) {
  Range nvtx_range(what);
  const int S = map_side(what, outGrads, F);
  CNB_REQUIRE(sizeX >= 1, what);
  CNB_REQUIRE(same_shape(denoms, outGrads) && same_shape(inputs, outGrads) && same_shape(acts, outGrads) &&
              same_shape(targets, outGrads), what);
  const Fuse fuse = take_fuse();
  CNB_REQUIRE(!fuse.bias_grad, what);
  Emit emit(targets->data_device, (long long)outGrads->size[0] * outGrads->size[1], fuse.emit_bf16 != 0, false);
  mapnorm_undo(outGrads->data_device, denoms->data_device, inputs->data_device, acts->data_device, targets->data_device,
               outGrads->size[0], S, F, sizeX, a, b);
  emit.finish();
}

void do_innerp(const char* what, cudamat* images, cudamat* derivs, cudamat* targets, Shape4D* is, Shape4D* ds, Shape4D* ts,
               ConvDesc d, float st, float so) {
  Range nvtx_range(what);
  d = as_2d(d);
  // the target is one value per filter tap, shape [1][kx][ky][1] (gemm.cu:993-996)
  CNB_REQUIRE(ts->shape[0] == 1 && ts->shape[3] == 1, what);
  CNB_REQUIRE(ts->shape[1] == d.kernel_size_x && ts->shape[2] == d.kernel_size_y, what);
  CNB_REQUIRE((long long)targets->size[0] * targets->size[1] == (long long)d.kernel_size_x * d.kernel_size_y, what);
  CNB_REQUIRE(is->shape[3] == d.num_input_channels && ds->shape[3] == d.num_output_channels, what);   // 2-D only
  Shape4D fs;                                   // the filter bank of the matching convolution, for the shared checks
  fs.shape[0] = (d.output_channel_end == 0 ? d.num_output_channels : d.output_channel_end) - d.output_channel_begin;
  fs.shape[1] = d.kernel_size_x; fs.shape[2] = d.kernel_size_y;
  fs.shape[3] = (d.input_channel_end == 0 ? d.num_input_channels : d.input_channel_end) - d.input_channel_begin;
  ConvGeom g = conv_geom(*is, fs, *ds, images, nullptr, derivs, d, true, what);
  CNB_REQUIRE(g.Cin == g.Cout, what);           // each channel of the images meets the derivative of the same channel
  take_fuse();
  bf16_note_write(targets->data_device, (long long)g.kx * g.ky);
  conv_innerp(g, images->data_device, derivs->data_device, targets->data_device, st, so);
}

}  // namespace

extern "C" {

// =============================== ABI-1 (cudamat_conv_gemm.cuh) ===============================
void convUpGemm(cudamat* images, cudamat* filters, cudamat* targets, Shape4D* is, Shape4D* fs, Shape4D* ts,
                ConvDesc d, float scaleTargets) {
  do_conv_up("convUpGemm", images, filters, targets, is, fs, ts, as_2d(d), scaleTargets, true);
}
void convDownGemm(cudamat* derivs, cudamat* filters, cudamat* targets, Shape4D* ds, Shape4D* fs, Shape4D* ts,
                  ConvDesc d, float scaleTargets) {
  do_conv_down("convDownGemm", derivs, filters, targets, ds, fs, ts, as_2d(d), scaleTargets, true);
}
void convOutpGemm(cudamat* images, cudamat* derivs, cudamat* targets, Shape4D* is, Shape4D* ds, Shape4D* ts,
                  ConvDesc d, float scaleTargets, float scaleOutput) {
  do_conv_outp("convOutpGemm", images, derivs, targets, is, ds, ts, as_2d(d), scaleTargets, scaleOutput, true);
}
void convInnerpGemm(cudamat* images, cudamat* derivs, cudamat* targets, Shape4D* is, Shape4D* ds, Shape4D* ts,
                    ConvDesc d, float scaleTargets, float scaleOutput) {
  do_innerp("convInnerpGemm", images, derivs, targets, is, ds, ts, d, scaleTargets, scaleOutput);
}
void localUpGemm(cudamat* images, cudamat* filters, cudamat* targets, Shape4D* is, Shape4D* fs, Shape4D* ts,
                 ConvDesc d, float scaleTargets) {
  do_conv_up("localUpGemm", images, filters, targets, is, fs, ts, as_2d(d), scaleTargets, false);
}
void localDownGemm(cudamat* derivs, cudamat* filters, cudamat* targets, Shape4D* ds, Shape4D* fs, Shape4D* ts,
                   ConvDesc d, float scaleTargets) {
  do_conv_down("localDownGemm", derivs, filters, targets, ds, fs, ts, as_2d(d), scaleTargets, false);
}
void localOutpGemm(cudamat* images, cudamat* derivs, cudamat* targets, Shape4D* is, Shape4D* ds, Shape4D* ts,
                   ConvDesc d, float scaleTargets, float scaleOutput) {
  do_conv_outp("localOutpGemm", images, derivs, targets, is, ds, ts, as_2d(d), scaleTargets, scaleOutput, false);
}

void MaxPoolGemm(cudamat* images, cudamat* targets, Shape4D* is, Shape4D* ts, ConvDesc d, float /*scaleTargets*/,
                 float scaleOutput) {
  do_pool("MaxPoolGemm", true, images, targets, is, ts, d, scaleOutput);
}
void AvgPoolGemm(cudamat* images, cudamat* targets, Shape4D* is, Shape4D* ts, ConvDesc d, float /*scaleTargets*/,
                 float scaleOutput) {
  do_pool("AvgPoolGemm", false, images, targets, is, ts, d, scaleOutput);
}
void MaxPoolUndoGemm(cudamat* images, cudamat* maxGrads, cudamat* maxActs, cudamat* targets, Shape4D* is,
                     Shape4D* gs, ConvDesc d, float scaleTargets) {
  do_pool_undo("MaxPoolUndoGemm", true, images, maxGrads, maxActs, targets, is, gs, d, scaleTargets, 1.f);
}
void MaxPoolRpropGemm(cudamat* images, cudamat* R_images, cudamat* maxActs, cudamat* targets, Shape4D* is,
                      Shape4D* ms, ConvDesc d, float scaleTargets) {
  do_max_rprop("MaxPoolRpropGemm", images, R_images, maxActs, targets, is, ms, d, scaleTargets);
}
void AvgPoolUndoGemm(cudamat* avgGrads, cudamat* targets, Shape4D* gs, Shape4D* ts, ConvDesc d, float scaleTargets) {
  do_pool_undo("AvgPoolUndoGemm", false, nullptr, avgGrads, nullptr, targets, ts, gs, d, scaleTargets, 1.f);
}
void UpSampleGemm(cudamat* images, cudamat* targets, Shape4D* is, Shape4D* ts, int factor, float scaleTargets) {
  CNB_REQUIRE(factor >= 1, "UpSampleGemm");
  // up-sampling == avg-pool undo with output scale factor^2 (gemm.cu:1503-1521)
  do_pool_undo("UpSampleGemm", false, nullptr, images, nullptr, targets, ts, is, sample_desc(ts, is, factor), scaleTargets,
               (float)(factor * factor));
}
void DownSampleGemm(cudamat* images, cudamat* targets, Shape4D* is, Shape4D* ts, int factor) {
  CNB_REQUIRE(factor >= 1, "DownSampleGemm");
  do_pool("DownSampleGemm", false, images, targets, is, ts, sample_desc(is, ts, factor), 1.f);
}

void ResponseNormCrossMapGemm(cudamat* images, cudamat* targets, int numFilters, int sizeF, float addScale,
                              float powScale, bool blocked) {
  do_rnorm("ResponseNormCrossMapGemm", images, targets, numFilters, sizeF, addScale, powScale, blocked, 1);
}
void ResponseNormCrossMapUndoGemm(cudamat* outGrads, cudamat* inputs, cudamat* targets, int numFilters, int sizeF,
                                  float addScale, float powScale, bool blocked) {
  do_rnorm_undo("ResponseNormCrossMapUndoGemm", outGrads, inputs, targets, numFilters, sizeF, addScale, powScale,
                blocked, 1);
}
void ResponseNormCrossMapRpropGemm(cudamat* images, cudamat* R_images, cudamat* targets, int numFilters, int sizeF,
                                   float addScale, float powScale, bool blocked) {
  do_rnorm_rprop("ResponseNormCrossMapRpropGemm", images, R_images, targets, numFilters, sizeF, addScale, powScale, blocked);
}
void Scale(cudamat* mat, float scale) {
  bf16_note_write(mat->data_device, (long long)mat->size[0] * mat->size[1]);
  scale_buffer(mat->data_device, (long long)mat->size[0] * mat->size[1], scale);
}

void convUp3DGemm(cudamat* images, cudamat* filters, cudamat* targets, Shape4D* is, Shape4D* fs, Shape4D* ts,
                  ConvDesc d, float scaleTargets) {
  do_conv_up("convUp3DGemm", images, filters, targets, is, fs, ts, d, scaleTargets, true);
}
void convDown3DGemm(cudamat* derivs, cudamat* filters, cudamat* targets, Shape4D* ds, Shape4D* fs, Shape4D* ts,
                    ConvDesc d, float scaleTargets) {
  do_conv_down("convDown3DGemm", derivs, filters, targets, ds, fs, ts, d, scaleTargets, true);
}
void convOutp3DGemm(cudamat* images, cudamat* derivs, cudamat* targets, Shape4D* is, Shape4D* ds, Shape4D* ts,
                    ConvDesc d, float scaleTargets, float scaleOutput) {
  do_conv_outp("convOutp3DGemm", images, derivs, targets, is, ds, ts, d, scaleTargets, scaleOutput, true);
}
void ResponseNormCrossMap3DGemm(cudamat* images, cudamat* targets, int numFilters, int sizeF, float addScale,
                                float powScale, bool blocked, int image_size_t) {
  do_rnorm("ResponseNormCrossMap3DGemm", images, targets, numFilters, sizeF, addScale, powScale, blocked, image_size_t);
}
void ResponseNormCrossMap3DUndoGemm(cudamat* outGrads, cudamat* inputs, cudamat* targets, int numFilters, int sizeF,
                                    float addScale, float powScale, bool blocked, int image_size_t) {
  do_rnorm_undo("ResponseNormCrossMap3DUndoGemm", outGrads, inputs, targets, numFilters, sizeF, addScale, powScale,
                blocked, image_size_t);
}

// =============================== ABI-2 (cudamat_conv.cuh) ====================================
void SetupTexture(cudamat*) {}   // texture-object cache of cudamat_conv_util.cu: nothing to do on sm_90a

void convUp(cudamat* images, cudamat* filters, cudamat* targets, Shape4D* is, Shape4D* fs, Shape4D* ts, ConvDesc d,
            float scaleTargets) {
  do_conv_up("convUp", images, filters, targets, is, fs, ts, as_2d(d), scaleTargets, true);
}
void localUp(cudamat* images, cudamat* filters, cudamat* targets, Shape4D* is, Shape4D* fs, Shape4D* ts, ConvDesc d,
             float scaleTargets) {
  do_conv_up("localUp", images, filters, targets, is, fs, ts, as_2d(d), scaleTargets, false);
}
void convDown(cudamat* derivs, cudamat* filters, cudamat* targets, Shape4D* ds, Shape4D* fs, Shape4D* ts, ConvDesc d,
              float scaleTargets) {
  do_conv_down("convDown", derivs, filters, targets, ds, fs, ts, as_2d(d), scaleTargets, true);
}
void localDown(cudamat* derivs, cudamat* filters, cudamat* targets, Shape4D* ds, Shape4D* fs, Shape4D* ts, ConvDesc d,
               float scaleTargets) {
  do_conv_down("localDown", derivs, filters, targets, ds, fs, ts, as_2d(d), scaleTargets, false);
}
void convOutp(cudamat* images, cudamat* derivs, cudamat* targets, Shape4D* is, Shape4D* ds, Shape4D* ts, ConvDesc d,
              int partialSumY, int partialSumX, float scaleTargets, float scaleOutput) {
  d = as_2d(d);
  const int modX = ds->shape[1], modY = ds->shape[2];
  if (partialSumY <= 0) partialSumY = modY;
  if (partialSumX <= 0) partialSumX = modX;
  const int chunks = ceil_div(modX, partialSumX) * ceil_div(modY, partialSumY);
  if (chunks == 1) {
    do_conv_outp("convOutp", images, derivs, targets, is, ds, ts, d, scaleTargets, scaleOutput, true);
    return;
  }
  // targets = `chunks` consecutive [Cout x K] blocks: shape {Cout, kx, ky, Cin*chunks} (weightacts.cu:3126-3170)
  CNB_REQUIRE(ts->shape[3] % chunks == 0, "convOutp");
  Shape4D one = *ts; one.shape[3] = ts->shape[3] / chunks;
  ConvGeom g = conv_geom(*is, one, *ds, images, nullptr, derivs, d, true, "convOutp");
  CNB_REQUIRE(targets->size[0] == g.Cout && (long long)targets->size[1] == (long long)g.K * chunks, "convOutp");
  simt_conv_outp(g, images->data_device, derivs->data_device, targets->data_device, partialSumY, partialSumX, true,
                 scaleTargets, scaleOutput);
  state().last_conv_path = kPathSimt;
}
void localOutp(cudamat* images, cudamat* derivs, cudamat* targets, Shape4D* is, Shape4D* ds, Shape4D* ts, ConvDesc d,
               float scaleTargets, float scaleOutput) {
  do_conv_outp("localOutp", images, derivs, targets, is, ds, ts, as_2d(d), scaleTargets, scaleOutput, false);
}

void ResponseNormCrossMap(cudamat* images, cudamat* targets, int numFilters, int sizeF, float addScale, float powScale,
                          bool blocked) {
  do_rnorm("ResponseNormCrossMap", images, targets, numFilters, sizeF, addScale, powScale, blocked, 1);
}
void ResponseNormCrossMapUndo(cudamat* outGrads, cudamat* inputs, cudamat* /*acts*/, cudamat* targets, int numFilters,
                              int sizeF, float addScale, float powScale, bool blocked) {
  do_rnorm_undo("ResponseNormCrossMapUndo", outGrads, inputs, targets, numFilters, sizeF, addScale, powScale, blocked, 1);
}
// within-map normalisation (cudamat_conv_others.cu:3669-3683): ResponseNorm is ContrastNorm with meanDiffs = images, and
// both undos are one kernel with `inputs` = the images or the meanDiffs.  `acts` is read, not overwritten (the reference
// leaves its scratch product in it).
void ResponseNorm(cudamat* images, cudamat* denoms, cudamat* targets, int numFilters, int sizeX, float addScale,
                  float powScale) {
  do_mapnorm("ResponseNorm", images, images, denoms, targets, numFilters, sizeX, addScale, powScale);
}
void ResponseNormUndo(cudamat* outGrads, cudamat* denoms, cudamat* inputs, cudamat* acts, cudamat* targets, int numFilters,
                      int sizeX, float addScale, float powScale) {
  do_mapnorm_undo("ResponseNormUndo", outGrads, denoms, inputs, acts, targets, numFilters, sizeX, addScale, powScale);
}
void ContrastNorm(cudamat* images, cudamat* meanDiffs, cudamat* denoms, cudamat* targets, int numFilters, int sizeX,
                  float addScale, float powScale) {
  do_mapnorm("ContrastNorm", images, meanDiffs, denoms, targets, numFilters, sizeX, addScale, powScale);
}
void ContrastNormUndo(cudamat* outGrads, cudamat* denoms, cudamat* meanDiffs, cudamat* acts, cudamat* targets,
                      int numFilters, int sizeX, float addScale, float powScale) {
  do_mapnorm_undo("ContrastNormUndo", outGrads, denoms, meanDiffs, acts, targets, numFilters, sizeX, addScale, powScale);
}

void MaxPool(cudamat* images, cudamat* targets, Shape4D* is, Shape4D* ts, ConvDesc d) {
  do_pool("MaxPool", true, images, targets, is, ts, d, 1.f);
}
void AvgPool(cudamat* images, cudamat* targets, Shape4D* is, Shape4D* ts, ConvDesc d) {
  do_pool("AvgPool", false, images, targets, is, ts, d, 1.f);
}
void MaxPoolUndo(cudamat* images, cudamat* maxGrads, cudamat* maxActs, cudamat* targets, Shape4D* is, Shape4D* gs,
                 ConvDesc d, float scaleTargets) {
  do_pool_undo("MaxPoolUndo", true, images, maxGrads, maxActs, targets, is, gs, d, scaleTargets, 1.f);
}
void AvgPoolUndo(cudamat* avgGrads, cudamat* targets, Shape4D* gs, Shape4D* ts, ConvDesc d, float scaleTargets) {
  do_pool_undo("AvgPoolUndo", false, nullptr, avgGrads, nullptr, targets, ts, gs, d, scaleTargets, 1.f);
}
void UpSample(cudamat* images, cudamat* targets, Shape4D* is, Shape4D* ts, int factor, float scaleTargets) {
  UpSampleGemm(images, targets, is, ts, factor, scaleTargets);
}
void DownSample(cudamat* images, cudamat* targets, Shape4D* is, Shape4D* ts, int factor) {
  DownSampleGemm(images, targets, is, ts, factor);
}
// images (3, pixels, numImages) -> targets of the same shape (convRGBToYUV, cudamat_conv_others.cu:2715-2755)
void RGBToYUV(cudamat* images, cudamat* targets) {
  Range nvtx_range("RGBToYUV");
  CNB_REQUIRE(images->size[1] % 3 == 0, "RGBToYUV: three colour planes");
  CNB_REQUIRE(same_shape(images, targets), "RGBToYUV");
  const Fuse fuse = take_fuse();
  const long long n = (long long)images->size[0] * images->size[1];
  Emit emit(targets->data_device, n, fuse.emit_bf16 != 0, false);
  rgb_to_yuv(images->data_device, targets->data_device, n / 3);
  emit.finish();
}

}  // extern "C"
