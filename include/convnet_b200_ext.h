/* convnet_b200_ext.h — additions to the reference's C surface (everything here is
 * new; nothing replaces a reference symbol).  Plain C ABI: pointers and scalars only.
 */
#ifndef CONVNET_B200_EXT_H_
#define CONVNET_B200_EXT_H_

#include "cudamat_abi.h"

#ifdef __cplusplus
extern "C" {
#endif
#if defined(__GNUC__)
#pragma GCC visibility push(default)   /* the library is built with -fvisibility=hidden */
#endif

/* Library version (major*10000 + minor*100 + patch). */
int convnet_b200_version(void);

/* Stream every kernel of this library is enqueued on.  Default: the legacy
 * default stream 0, which is what every reference kernel uses
 * (cudamat_conv_filteracts.cu:1259), so ordering against libcudamat.so is kept.
 * `cuda_stream` is a cudaStream_t / CUstream handle. */
void convnet_b200_set_stream(void* cuda_stream);
void* convnet_b200_get_stream(void);

/* Arithmetic of the three conv ops (pool / response-norm are always fp32):
 *   0  FP32  fp32 FMA on CUDA cores (the DEFAULT: a drop-in caller gets the reference's arithmetic); meets the
 *            reference's own 1e-4 kernel test tolerance (py/test_conv.py:387); what run_grad_check uses
 *   1  TF32  tensor-core tf32 (mma.sync) on the caller's fp32 buffers, fp32 accumulate;
 *            Diff <= 5e-3 (operands truncated to 10 mantissa bits by the tensor core)
 *   2  BF16  tensor-core bf16 (wgmma) on bf16 copies, fp32 accumulate; Diff <= 2e-2
 * Shapes the tensor-core path does not take fall through to FP32.  The tensor-core modes are opt-in: this call, or
 * CONVNET_B200_PRECISION={fp32,tf32,bf16} in the environment before first use (host/ConvNet and bench.py opt in). */
void convnet_b200_set_conv_precision(int mode);
int convnet_b200_get_conv_precision(void);

/* Which path the most recent conv call took: 0 CUDA-core fp32, 1 tensor-core tf32,
 * 2 tensor-core bf16, -1 none yet.  (tests assert the tensor path really ran) */
int convnet_b200_last_conv_path(void);

/* Number of kernels this library has launched since the last reset. */
unsigned long long convnet_b200_launch_count(void);
void convnet_b200_reset_launch_count(void);

/* One-shot: the NEXT pool-undo (MaxPoolUndo*, AvgPoolUndo*) or convDown* call also produces the shared-bias gradient of
 * the edge BELOW — the one whose output derivative is the tensor this call writes (src/conv_edge.cc:210-222 runs
 * SumRows over that tensor later):  grad_bias[c] = scaleTargets*grad_bias[c] + scaleOutput * sum_{n,pixels} target[n,pixel,c].
 * The sums come from the values the kernel is storing anyway (deterministic per-row partial sums + a tiny second
 * kernel), so the separate pass over the derivative disappears; calls that cannot do it run that pass themselves. */
void convnet_b200_fuse_next_bias_grad(float* grad_bias, float scaleTargets, float scaleOutput);

/* One-shot: the NEXT convDown* call multiplies its result by `scale` (before the relu_mask of convnet_b200_fuse_next);
 * so do AvgPool* / DownSample* (after scaleOutput), AvgPoolUndo* and UpSample* (after scaleTargets * old).
 * This is how the derivative of inverted dropout disappears as a pass: for a ReLU layer with dropout the state holds
 * relu(x) * m with m in {0, 1/(1-p)}, so  deriv * m * [state > 0]  (Layer::ApplyDerivativeofDropout followed by
 * ApplyDerivativeOfActivation, src/layer.cc:367-395,562-580)  ==  deriv * 1/(1-p) * [state > 0]. */
void convnet_b200_fuse_next_scale(float scale);

/* One-shot: the NEXT MaxPool* call also records which elements of every window equal its maximum (one 16-bit mask per
 * pooled element, in library scratch).  The MaxPoolUndo* call on the same (images, maxActs) pair then reads the gradients
 * and those masks instead of re-reading the pool input and output and comparing — 0.55x the bytes of the largest
 * memory-bound pass of the step, bit-identical results (ties duplicate the gradient exactly as kMaxPoolUndo's `==` test
 * does, cudamat_conv_gemm.cu:262-300).  The masks go stale, and the undo falls back to comparing, as soon as any entry
 * point of this library writes either tensor; a caller that overwrites them by other means between the two calls must
 * not use this request (or must call convnet_b200_bf16_invalidate(NULL)).  2-D windows up to 3 x 3 with a side of 3,
 * stride 2, padding up to 2; other pools ignore the request. */
void convnet_b200_pool_cache_next(void);

/* One-shot request for the next convUp* call (after its bias / ReLU, if those are requested too): dropout of the result with
 * the generator of cnb_dropout — element i of the target is kept iff hash(seed + i) >= dropprob, kept values are multiplied
 * by `scale` — exactly as if cnb_dropout(target, mask, n, dropprob, scale, seed) followed the call, except that NO mask
 * tensor is written: the caller's backward pass must not need one (for a ReLU layer the kept units are the non-zero ones:
 * convnet_b200_fuse_next_scale on the dgrad that produces this layer's derivative).  The tensor-core fprop applies it in
 * its epilogue; every other path runs one trailing pass inside the call. */
void convnet_b200_fuse_next_dropout(float dropprob, float scale, unsigned long long seed);

/* One-shot request for the next convDown* call: do not compute anything, only prepare on the current stream what that call
 * derives from the FILTERS alone — in bf16 mode the per-stride-phase, tap-flipped bf16 filter banks the dgrad kernels read
 * (DESIGN.md §3).  The derivative and target tensors are not touched (their shapes must still describe the call).  A
 * trainer issues this right after the optimizer step of a layer, on the optimizer's stream, so that the next step's
 * convDown finds the banks ready instead of rebuilding them on the critical path. */
void convnet_b200_prestage_next(void);

/* How many times the bf16 dgrad filter banks have been built since the library was loaded: in_prestage 0 counts the
 * builds inside a convDown* call (on its critical path), 1 those made for a convnet_b200_prestage_next request.  The
 * banks are cached per filter tensor and call geometry, so a filter tensor that several calls use at different strides,
 * paddings or image sizes keeps one set per geometry; any write to the filters drops them all. */
unsigned long long convnet_b200_dgrad_bank_builds(int in_prestage);

/* The conv kernels are persistent: one CTA per SM, each owning most of the SM's shared memory.  A kernel
 * of another library that must run CONCURRENTLY (an NCCL collective on a side stream) cannot co-reside with them and
 * would otherwise wait for — or push out — a whole wave.  convnet_b200_reserve_sms(n) makes the persistent grids leave
 * n SMs free until it is called again with 0.  (host/convnet.cc reserves the SMs of the gradient all-reduce while it
 * is in flight.) */
void convnet_b200_reserve_sms(int n);

/* Free cached device scratch (wgrad / split-K partial sums, bf16 staging buffers).  Never required. */
void convnet_b200_release_workspace(void);

/* One-shot epilogue fusion for the NEXT conv / pool-undo call of this library (cleared by that call):
 *   bias      (convUp*): adds bias[o] to every output of output channel o — the shared-bias AddRowVec of
 *             ConvEdge::ComputeUp (src/conv_edge.cc:143-152) without the extra pass;
 *             (localUp*): one value per output FEATURE — bias[m + modules*o] is added to output channel o of module m,
 *             i.e. bias[j] to column j of the target: the AddRowVec of LocalEdge::ComputeUp (src/local_edge.cc:117);
 *   relu      (convUp*, localUp*): clamps at 0 after the bias — Layer::ApplyActivation for RECTIFIED_LINEAR (src/layer.cc:550);
 *   relu_mask (convDown*, localDown*, MaxPoolUndo*, AvgPoolUndo*): result zeroed where relu_mask[i] <= 0; relu_mask has
 *             the shape of `targets` (it is the state of the layer receiving the derivative: ApplyDerivativeOfActivation);
 *             on localDown* always as a pass at the end of the call.
 * Pass NULL / 0 for the parts not wanted.  Calls that cannot fuse (3-D dgrad) apply the same maths in a second pass. */
void convnet_b200_fuse_next(const float* bias, int relu, const float* relu_mask);
/* The same request with an activation code (CNB_ACT_*) in place of the ReLU flag:
 *   act, fprop      (convUp*, localUp*): the activation after the bias — max(., 0), or the logistic sigma(.) of cnb_logistic
 *                   (LogisticLayer::ApplyActivation, src/layer.cc:598); any fused dropout comes after it;
 *   act_state, dgrad (convDown*, localDown*, MaxPoolUndo*, AvgPoolUndo*): the result times the derivative of `act` at the
 *                   state act_state — the ReLU' mask as above, or (r * s) * (1 - s) as cnb_logistic_deriv computes it.  The
 *                   pool-undo kernels and localDown* apply sigma' as a pass at the end of the call.
 * Results are bit-identical to the unfused call followed by cnb_relu / cnb_logistic (fprop) or cnb_relu_deriv /
 * cnb_logistic_deriv (dgrad).  convnet_b200_fuse_next(bias, relu, relu_mask) is fuse_next_act(bias, relu ? 1 : 0, ...) for
 * fprop and fuse_next_act(NULL, 1, relu_mask) for the derivative. */
enum { CNB_ACT_LINEAR = 0, CNB_ACT_RELU = 1, CNB_ACT_LOGISTIC = 2 };
void convnet_b200_fuse_next_act(const float* bias, int act, const float* act_state);
/* The average-pool calls (AvgPool*, DownSample*, AvgPoolUndo*, UpSample*) honour, besides convnet_b200_emit_bf16_next:
 *   act with act_state NULL: the forward activation of the result (max(., 0) in the kernel, sigma a pass in the call),
 *       then convnet_b200_fuse_next_dropout (mask-free, element i of the target kept iff cnb_dropout keeps it);
 *   act_state: the derivative of act at act_state, after convnet_b200_fuse_next_scale;
 *   convnet_b200_fuse_next_bias_grad: the per-channel sums of the stored values (AvgPool* / DownSample* here too).
 * Every result is bit-identical to the unfused call followed by cnb_relu / cnb_logistic, cnb_dropout, cnb_mult (by a
 * tensor of `scale`) and cnb_relu_deriv / cnb_logistic_deriv; the bias gradient equals cnb_channel_bias_grad's up to the
 * order of the fp32 sum.  Shapes the row-structured kernels do not take run the same passes inside the call. */

/* bf16 operand staging (precision mode 2 only; no-ops in the other modes).  In bf16 mode every conv call first rounds
 * its two fp32 operands to bf16 copies.  A caller that knows a tensor stays unchanged across several conv calls
 * (the layer input: fprop + wgrad; the output derivative: wgrad + dgrad; the weights: fprop + dgrad) can have it
 * converted ONCE: convnet_b200_bf16_stage(ptr, n) converts the n floats at ptr now (stream-ordered) and conv calls
 * that receive exactly `ptr` as an operand use that copy while it is valid.  convnet_b200_bf16_ensure converts only
 * when no valid copy exists.
 * Coherence: every entry point of THIS library that writes a tensor drops the staged copies overlapping what it
 * writes (and convnet_b200_emit_bf16_next makes it leave a fresh one), and cnb_sgd_momentum refreshes the copy of
 * the weights it updates.  Only writes the library cannot see (cudaMemcpy, another library's kernels) need an
 * explicit convnet_b200_bf16_invalidate(ptr) / _stage(ptr, n) from the caller; convnet_b200_bf16_invalidate(NULL)
 * forgets every staged tensor.  CONVNET_B200_STAGE_VERIFY=1 (environment) re-converts the fp32 source at every use of
 * a staged copy and aborts on a mismatch — the way to find such a missed write. */
void convnet_b200_bf16_stage(const float* ptr, long long n);
void convnet_b200_bf16_ensure(const float* ptr, long long n);
void convnet_b200_bf16_invalidate(const float* ptr);
int convnet_b200_bf16_is_staged(const float* ptr, long long n);   /* 1 if a valid staged copy covers [ptr, ptr+n) */

/* One-shot: the NEXT entry point of this library that writes a tensor (conv fprop / dgrad, pooling and its undo,
 * response norm and its undo, cnb_relu, cnb_dropout, cnb_mult, cnb_add_channel_bias*) also leaves a staged bf16 copy of
 * the WHOLE target tensor, exactly as convnet_b200_bf16_stage(target, n) right after the call would — but written by the
 * producing kernel from the same registers where that kernel supports it (the fp32 -> bf16 pass and its 6 bytes/element
 * of HBM traffic disappear), by a trailing conversion pass where it does not.  No-op outside bf16 mode. */
void convnet_b200_emit_bf16_next(void);

/* ---- steps either side of the conv ops that the Edge layer sequences ------------
 * (SURVEY.md §8(f) rank 2; in the reference these are libcudamat.so calls:
 *  add_row_vec cudamat.cu:1064, sum_by_axis :1614, lower_bound_scalar :1426,
 *  apply_rectified_linear_deriv :2475).  Names are prefixed so both libraries link. */

/* acts (N, locs, C): acts[n, l, c] += bias[c]  — ConvEdge::ComputeUp shared bias,
 * src/conv_edge.cc:143-152.  rows = N*locs, cols = C. */
void cnb_add_channel_bias(float* acts, const float* bias, long long rows, int cols);
/* same, fused with ReLU (Layer::ApplyActivation, src/layer.cc:550: LowerBound(0)). */
void cnb_add_channel_bias_relu(float* acts, const float* bias, long long rows, int cols);
/* grad_bias[c] = scaleTargets*grad_bias[c] + scaleOutput * sum_{rows} derivs[r, c]
 * — src/conv_edge.cc:210-222 (two-step SumRows). Deterministic. */
void cnb_channel_bias_grad(const float* derivs, float* grad_bias, long long rows, int cols,
                           float scaleTargets, float scaleOutput);
/* x = max(x, 0) ; dx *= (y > 0) */
void cnb_relu(float* x, long long n);
void cnb_relu_deriv(float* dx, const float* y, long long n);
/* binary dropout (Layer::ApplyDropoutAtTrainTime, src/layer.cc:367-395): mask[i] = Bernoulli(1-dropprob)*scale,
 * x *= mask; counter-based RNG keyed by (seed, i).  cnb_mult: a *= b (ApplyDerivativeofDropout). */
void cnb_dropout(float* x, float* mask, long long n, float dropprob, float scale, unsigned long long seed);
void cnb_mult(float* a, const float* b, long long n);
/* softmax over the classes of a column-major [rows=N x cols=classes] matrix, in place
 * (Layer::ApplyActivation for SOFTMAX layers, src/layer.cc) */
void cnb_softmax(float* x, int rows, int cols);
/* deriv = probs - onehot(labels); loss_per_image[n] = -log probs[n, label] (may be NULL)
 * (CrossEntropyMultinomial, src/loss_functions.cc:70-95) */
void cnb_softmax_ce_deriv(const float* probs, const int* labels, float* deriv, float* loss_per_image,
                          int rows, int cols);
/* the logistic unit (LogisticLayer, src/layer.cc:586-602):  x = 1 / (1 + expf(-x));  dx = (dx * y) * (1 - y).
 * Arithmetic: every operation rounded to nearest, expf within 2 ulp (CUDA Programming Guide), so
 *   |cnb_logistic(x) - sigma(x)| <= 3 * 2^-23 * sigma(x) + 2^-126            (sigma(x) = 0 below x = -88.7: expf overflows)
 *   |cnb_logistic_deriv - dx * y * (1 - y)| <= 3 * 2^-24 * |dx * y * (1 - y)| + 2^-148
 * The reference's CUDA uses __expf (cudamat_kernels.cu:146-148) and its derivative a * b * (1.0 - b) in double after
 * the first product (:810-816); the fused conv epilogues (convnet_b200_fuse_next_act) use exactly these functions.
 * Both honour convnet_b200_emit_bf16_next. */
void cnb_logistic(float* x, long long n);
void cnb_logistic_deriv(float* dx, const float* y, long long n);
/* loss functions and performance metrics of an output layer (proto/convnet_config.proto LossFunction numbers;
 * src/loss_functions.cc).  y, targets, deriv: column-major [rows = images x cols], images fastest (any number of pixels
 * per image).  labels: `rows` ints (CROSS_ENTROPY_MULTINOMIAL, CLASSIFICATION_MULTINOMIAL); targets: per-feature floats
 * (the others).  Per image, summed over its columns in order (DESIGN.md §5 has every rule):
 *   SQUARED_ERROR 0.5 * sum (y - t)^2;  LINEAR_ERROR sum (y - t);  CROSS_ENTROPY_MULTINOMIAL -log y[label];
 *   CROSS_ENTROPY_BINARY sum over t >= 0 of -t log(y + 1e-10) - (1 - t) log(1 - y + 1e-10);
 *   CROSS_ENTROPY_MULTINOMIAL_DISTRIBUTED sum -t log(y + 1e-10);
 *   CLASSIFICATION_MULTINOMIAL 1 if the argmax (kSoftMaxCorrectRowMajor's) is the label, else 0;
 *   CLASSIFICATION_BINARY the share of features with t >= 0 where (t >= .5) == (y >= .5).
 * cnb_loss_deriv writes deriv = weight * dLoss/dy ((y - t) | 1 | y - onehot; 0 where a binary target is < 0) and the
 * per-image loss (NOT weighted: the caller scales the sum, as Layer::GetLoss does); CROSS_ENTROPY_MULTINOMIAL with weight 1
 * is exactly cnb_softmax_ce_deriv.  cnb_metric writes the per-image value of a metric or a loss. */
enum {
  CNB_LOSS_SQUARED_ERROR = 0, CNB_LOSS_LINEAR_ERROR = 1, CNB_LOSS_CROSS_ENTROPY_MULTINOMIAL = 2,
  CNB_LOSS_CROSS_ENTROPY_BINARY = 3, CNB_LOSS_CROSS_ENTROPY_MULTINOMIAL_DISTRIBUTED = 4,
  CNB_LOSS_CLASSIFICATION_MULTINOMIAL = 5, CNB_LOSS_CLASSIFICATION_BINARY = 6
};
void cnb_loss_deriv(int loss, const float* y, const float* targets, const int* labels, float* deriv, float* loss_per_image,
                    int rows, int cols, float weight);
void cnb_metric(int metric, const float* y, const float* targets, const int* labels, float* metric_per_image, int rows,
                int cols);
/* *out = sum(a[0..n)) on the device (no host sync) */
void cnb_sum(const float* a, float* out, int n);
/* SGD with momentum and L2 decay, one fused pass (src/optimizer.cc:174-200):
 *   g' = lr*(g + l2*w);  h = momentum*h + g';  w -= h
 * (cnb_sgd_update_multi with one tensor, no clip and no norm) */
void cnb_sgd_momentum(float* w, float* hist, const float* grad, long long n, float lr,
                      float momentum, float l2);
/* the same update for `count` tensors in ONE launch (one call per all-reduce bucket / per net instead of one per
 * weight and bias matrix).  `tensors` is a host array.  In bf16 mode a staged copy of a weight tensor is refreshed
 * by the same pass (see convnet_b200_bf16_stage).  (cnb_sgd_update_multi without clip and norms) */
typedef struct CnbSgdTensor {
  float* w; float* hist; const float* grad; long long n; float lr, momentum, l2;
} CnbSgdTensor;
void cnb_sgd_momentum_multi(const CnbSgdTensor* tensors, int count);

/* The whole SGD step of SGDOptimizer::Optimize (src/optimizer.cc:174-200) for `count` tensors, in this order:
 *   g += l2*w;  g = clamp(g, -clip, clip) if clip > 0 (gradient_clip);  h = momentum*h + lr*g;  w -= h;
 *   then the row-norm rule (Optimizer::ApplyConstraints, optimizer.cc:75-81) on the updated w.
 * The caller supplies this step's lr and momentum (the schedules are host logic).  Row norms: the tensor is
 * [rows x n/rows] with the rows fastest — row r is the elements r + rows*k, one output unit's incoming weights in this
 * library's filter layout; a bias is one row.  CNB_NORM_LIMIT rescales the rows whose norm exceeds norm_value to
 * norm_value (weight_norm_limit), CNB_NORM_CONSTRAINT rescales every row to norm_value (weight_norm_constraint); a row of
 * norm 0 is left at 0 (the reference divides by 0 there).  One launch for the update — which also sums the squares of
 * the weights it stores, per row, into library scratch — plus one for the rescale when any tensor has a norm rule; no
 * atomics, so results are bit-reproducible.  Calls must be ordered on one stream (the scratch is shared between calls).
 * A tensor with clip <= 0 and no norm rule gets exactly the bits of cnb_sgd_momentum_multi. */
enum { CNB_NORM_NONE = 0, CNB_NORM_LIMIT = 1, CNB_NORM_CONSTRAINT = 2 };
typedef struct CnbOptTensor {
  float* w; float* hist; const float* grad; long long n; float lr, momentum, l2;
  float clip;          /* > 0: gradient clip */
  int rows;            /* norm groups (n % rows == 0); read only with a norm rule */
  int norm_mode;       /* CNB_NORM_* */
  float norm_value;    /* > 0 with a norm rule */
} CnbOptTensor;
void cnb_sgd_update_multi(const CnbOptTensor* tensors, int count);

/* cnb_sgd_update_multi with a rule per tensor: the SGD step above, or the adaptive steps of AdagradSGDOptimizer and
 * RMSPropSGDOptimizer::Optimize (src/optimizer.cc:202-279), which keep one more float per element, `state` (n floats;
 * the caller initialises it to adagrad_delta resp. 1).  Per element, every operation rounded to nearest, fma the one
 * fused operation (safe_div(x, s) = x / s, and 0 where x == 0: the reference's 0 / 0 gives NaN there):
 *   CNB_RULE_ADAGRAD  e = s - delta;  s = delta + sqrt(e*e + g*g);  g = safe_div(g, s) * scale   (before the SGD step;
 *                     rule_param = delta, scale = sqrt(step + 1) rounded to float; state_only != 0: only s is updated —
 *                     the reference accumulates it also before start_optimization_after)
 *   SGD step          d = fma(l2, w, g);  clip;  [RMSProp]  h = fma(momentum, h, lr*d);  w = w - h;  then the row-norm rule
 *   CNB_RULE_RMSPROP  at [RMSProp]:  s = sqrt((f*s)*s + ((1-f)*d)*d);  d = safe_div(d, s)   (rule_param = f, the factor)
 * A CNB_RULE_SGD tensor gets exactly the bits of cnb_sgd_update_multi.  Every rule goes into the same launches: one for
 * the update and one for the rescale of rows when any tensor has a norm rule.  The gradient is only read. */
enum { CNB_RULE_SGD = 0, CNB_RULE_ADAGRAD = 1, CNB_RULE_RMSPROP = 2 };
typedef struct CnbOptTensorEx {
  CnbOptTensor t;
  int rule;            /* CNB_RULE_* */
  int state_only;      /* CNB_RULE_ADAGRAD: update the state alone, leave w and hist as they are */
  float* state;        /* adaptive rules: n floats */
  float rule_param;    /* ADAGRAD: adagrad_delta; RMSPROP: rms_prop_factor */
  float scale;         /* ADAGRAD: sqrt(step + 1) */
} CnbOptTensorEx;
void cnb_opt_update_multi(const CnbOptTensorEx* tensors, int count);

/* ---- batch normalisation over the channels of a 2-D layer (Layer::ApplyBatchNormalization and
 * ApplyDerivativeofBatchNormalization, src/layer.cc:452-510).  x, y and deriv hold `channels` contiguous blocks of n
 * floats: channel c is [c*n, (c+1)*n), n = images * pixels (the layout of a layer state, DESIGN.md §3).  Per-channel
 * vectors hold `channels` floats.  Reductions use a fixed order and no atomics: results are bit-reproducible.  Calls must
 * be ordered on one stream (they share a library scratch buffer).
 *
 * cnb_bn_stats: batch_mu = mean(x), batch_sigma = sqrt(mean((x - batch_mu)^2) + eps) (two passes: the variance is taken
 *   about the mean); when run_mu / run_sigma are given (both or neither), the running averages
 *   run_mu = bn_f*run_mu + (1-bn_f)*batch_mu and run_sigma = bn_f*run_sigma + (1-bn_f)*batch_sigma (sigma, not the variance).
 * cnb_bn_apply: y = gamma*(x - mu)/sigma + beta, then max(y, 0) if relu.  mu / sigma are the batch statistics (training)
 *   or the running ones (test).  Honours convnet_b200_emit_bf16_next for y.
 * cnb_bn_backward: with xhat = (x - mu)/sigma,
 *   grad_beta = mean(deriv), grad_gamma = mean(deriv * xhat)            (1/n scaling, layer.cc:493-496), then in place
 *   deriv = gamma/sigma * (deriv - grad_beta - xhat * grad_gamma)     train != 0 (mu / sigma: the batch statistics)
 *   deriv = gamma/sigma * deriv                                       train == 0 (mu / sigma: the running statistics)
 *   Honours convnet_b200_emit_bf16_next for deriv. */
void cnb_bn_stats(const float* x, long long n, int channels, float eps, float bn_f, float* batch_mu, float* batch_sigma,
                  float* run_mu, float* run_sigma);
void cnb_bn_apply(const float* x, float* y, long long n, int channels, const float* gamma, const float* beta,
                  const float* mu, const float* sigma, int relu);
void cnb_bn_backward(float* deriv, const float* x, long long n, int channels, const float* gamma, const float* mu,
                     const float* sigma, int train, float* grad_gamma, float* grad_beta);

/* ---- Polyak averaging (ConvNet::LoadPolyakWeights, the reference's loop at src/convnet.cc:715-723).  `queue` holds k
 * slots of n floats, slot s at queue + s*slot_stride:
 *   out[j] = (((0 + s_0[j]) + s_1[j]) + ... + s_{k-1}[j]) / (float)k
 * summed in slot order, each addition from +0.0f and rounded to nearest (so -0.0 averages to +0.0, as in the reference).
 * `out` must not overlap the queue.  k >= 1.  Honours convnet_b200_emit_bf16_next for out; every other staged copy that
 * overlaps out (the weights' bf16 twins, the dgrad filter banks) is dropped.  Runs on the library's stream. */
void cnb_polyak_average(float* out, const float* queue, long long n, long long slot_stride, int k);

/* ---- input pipeline, device side (SURVEY.md §8 f4) -------------------------------------------------------------------
 * The reference keeps a chunk of the data set on the GPU, one image per COLUMN (pixel index = col + W*(row + H*color)),
 * and cuts every minibatch out of it with a random crop and mirror per image while transposing it into the image-fastest
 * layout of the input layer: its DataIterator::AddNoise (src/datahandler.cc:520-531) calls Matrix::ExtractPatches
 * (src/matrix.cc:1030-1042), which calls extract_patches (cudamat/cudamat.cuh:265, cudamat.cu:2699-2742, kernel
 * cudamat_kernels.cu:1655-1669).  convnet_b200_extract_patches is that last call: same arguments, same element-for-element
 * result, same error codes (ERROR_INCOMPATIBLE_DIMENSIONS = -1, CUDA_ERROR = -3); exported under its own name because the
 * reference's copy lives in libcudamat.so, which a drop-in build keeps linking:
 *   patches[n + N*(x + pw*(y + ph*c))] = images[sx + W*(height_offset[n] + y + H*(c + C*n))],
 *   sx = width_offset[n] + x, mirrored to W - 1 - sx when flip[n] > 0.5.
 * `images` is (C*W*H) x N in cudamat's size[] convention (size[1] = N images), `patches` is N x (C*pw*ph); the three
 * per-image vectors hold N floats on the device.  Source coordinates are clamped to the image (the reference reads out of
 * bounds for a crop that does not fit).  Runs on the library's stream. */
int convnet_b200_extract_patches(cudamat* images, cudamat* patches, cudamat* width_offset, cudamat* height_offset,
                                 cudamat* flip, int img_width, int img_height, int patch_width, int patch_height);

/* The launch behind both crop entry points, on raw device pointers (host/data.h's DataIterator::AddNoise calls it on a
 * slice of its chunk): `images` holds N or more images of C*W*H floats, `patches` is N x (C*pw*ph), and the formulas are
 * those of convnet_b200_extract_patches, or of cnb_extract_patches_indexed when `index` is not NULL.  Source coordinates
 * are clamped to the image.  The label and target gathers are those of cnb_extract_patches_indexed and need an index.
 * 0 ok (also when N, C, pw or ph is not positive: nothing to crop), -1 a source without its destination or the other way
 * round, a gather without an index, or a grid past 65535 blocks in y or z, -3 launch error.  Runs on the library's stream. */
int cnb_extract_patches(const float* images, float* patches, const int* index, const float* width_offset,
                        const float* height_offset, const float* flip, int N, int C, int W, int H, int pw, int ph,
                        const int* labels_src, int* labels_dst, const float* targets_src, float* targets_dst,
                        int target_dims);

/* The same crop through a permutation of the chunk, with the batch's labels and targets gathered in the same launch
 * (DataHandler, host/data.h).  Batch image n reads chunk column index[n] (device ints, each < the chunk's image count):
 *   patches[n + N*(x + pw*(y + ph*c))] = images[sx + W*(height_offset[n] + y + H*(c + C*index[n]))]
 * with sx as above, so the pixels are bit-identical to convnet_b200_extract_patches on a chunk whose column n is column
 * index[n] of this one.  The shuffle costs one index read per image instead of a rewrite of the chunk.
 *   labels_dst[n] = labels_src[index[n]]                                  (one int per chunk image)
 *   targets_dst[n + N*j] = targets_src[target_dims*index[n] + j]          (one row of target_dims floats per chunk image)
 * labels_src / labels_dst and targets_src / targets_dst are both NULL or both set.  The crop must fit the image
 * (pw <= W, ph <= H).  0 ok, -1 bad arguments, -3 launch error.  Runs on the library's stream. */
int cnb_extract_patches_indexed(const float* images, float* patches, const int* index, const float* width_offset,
                                const float* height_offset, const float* flip, int N, int C, int W, int H, int pw, int ph,
                                const int* labels_src, int* labels_dst, const float* targets_src, float* targets_dst,
                                int target_dims);

#if defined(__GNUC__)
#pragma GCC visibility pop
#endif
#ifdef __cplusplus
}
#endif
#endif  /* CONVNET_B200_EXT_H_ */
