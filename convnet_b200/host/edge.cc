// edge.cc — see edge.h.  Sequencing follows the reference's src/*_edge.cc line by line where cited.
#include "edge.h"

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <random>
#include <vector>

#ifndef DIVUP
#define DIVUP(x, y) (((x) + (y)-1) / (y))
#endif

namespace cnbhost {

// ---------------------------------------------------------------- Edge (src/edge.cc)
Edge::Edge(const EdgeConfig& c)
    : config_(c), name_(c.name.empty() ? c.source + ":" + c.dest : c.name), source_(nullptr), dest_(nullptr),
      num_input_channels_(0), num_output_channels_(0), image_size_y_(0), image_size_x_(0), image_size_t_(1),
      num_modules_y_(1), num_modules_x_(1), num_modules_t_(1), batch_size_(0) {}

Edge* Edge::ChooseEdgeClass(const EdgeConfig& c) {          // src/edge.cc:17-60
  switch (c.edge_type) {
    case FC: return new FCEdge(c);
    case CONVOLUTIONAL: return new ConvEdge(c);
    case MAXPOOL: return new MaxPoolEdge(c);
    case AVGPOOL: return new AvgPoolEdge(c);
    case RESPONSE_NORM: return new ResponseNormEdge(c);
    case CONV_ONETOONE: return new ConvOneToOneEdge(c);
    case LOCAL: return new LocalEdge(c);
  }
  fprintf(stderr, "Error: Undefined edge type.\n");
  exit(1);
}

ConvDesc Edge::GetConvDesc(const EdgeConfig& c) {           // src/edge.cc:87-106
  ConvDesc d;
  d.num_input_channels = 0; d.num_output_channels = 0;
  d.kernel_size_y = c.kernel_size_y > 0 ? c.kernel_size_y : c.kernel_size;
  d.kernel_size_x = c.kernel_size_x > 0 ? c.kernel_size_x : c.kernel_size;
  d.kernel_size_t = c.kernel_size_t;
  d.stride_y = c.stride_y > 0 ? c.stride_y : c.stride;
  d.stride_x = c.stride_x > 0 ? c.stride_x : c.stride;
  d.stride_t = c.stride_t;
  d.padding_y = -(c.padding_y >= 0 ? c.padding_y : c.padding);     // NEGATED: kernels add it to the window start
  d.padding_x = -(c.padding_x >= 0 ? c.padding_x : c.padding);
  d.padding_t = -c.padding_t;
  d.input_channel_begin = d.input_channel_end = d.output_channel_begin = d.output_channel_end = 0;
  d.num_groups = 1;
  return d;
}

void Edge::GetNumModules(const ConvDesc d, int image_size_y, int image_size_x, int image_size_t, int& my, int& mx,
                         int& mt) {                          // src/edge.cc:108-114
  my = (image_size_y - 2 * d.padding_y - d.kernel_size_y) / d.stride_y + 1;
  mx = (image_size_x - 2 * d.padding_x - d.kernel_size_x) / d.stride_x + 1;
  mt = (image_size_t - 2 * d.padding_t - d.kernel_size_t) / d.stride_t + 1;
}

void Edge::SetImageSize(int y, int x, int t) {
  image_size_y_ = y; image_size_x_ = x; image_size_t_ = t;
  num_modules_y_ = y; num_modules_x_ = x; num_modules_t_ = t;
}

// ---------------------------------------------------------------- EdgeWithWeight
void EdgeWithWeight::SetHistoryMemory(Matrix& p) {
  // same carving as the gradient slice: weights first, then the bias column(s)
  const int rows = grad_weights_.GetRows();
  p.Reshape(rows, -1);
  p.GetSlice(hist_weights_, 0, grad_weights_.GetCols());
  if (!has_no_bias_) {
    p.GetSlice(hist_bias_, grad_weights_.GetCols(), p.GetCols());
  }
}
void EdgeWithWeight::SetStateMemory(Matrix& p) {
  p.Reshape(grad_weights_.GetRows(), -1);
  p.GetSlice(state_weights_, 0, grad_weights_.GetCols());
  if (!has_no_bias_) p.GetSlice(state_bias_, grad_weights_.GetCols(), p.GetCols());
}
void EdgeWithWeight::InitState(int which) { InitAdaptiveState(Optimizer(which), which ? state_bias_ : state_weights_); }

void EdgeWithWeight::StageForUp(Matrix& input) {
  if (convnet_b200_get_conv_precision() != 2) return;
  if (bf_up_ == 1 || bf_outer_ == 1) convnet_b200_bf16_ensure(input.GetDevData(), (long long)input.GetNumEls());
  // the weights: also on the very first step (paths still unknown) — FC-shaped calls take the bf16 path only when they find
  // the copy, and from then on the SGD kernel keeps it fresh; an edge that turns out to stay on tf32 drops it again
  if (bf_up_ != 0 || bf_down_ != 0) convnet_b200_bf16_ensure(weights_.GetDevData(), (long long)weights_.GetNumEls());
}
void EdgeWithWeight::StageForBprop(Matrix& deriv_output) {
  if (convnet_b200_get_conv_precision() != 2) return;
  if (bf_outer_ == 1 || bf_down_ == 1) convnet_b200_bf16_ensure(deriv_output.GetDevData(), (long long)deriv_output.GetNumEls());
}
void EdgeWithWeight::SumBiasRows(Matrix& deriv_output, float scale_targets, float scale) {
  cudaEventRecord(side_->ready, Matrix::Stream());            // the derivative is final on the main stream
  cudaStreamWaitEvent(side_->stream, side_->ready, 0);
  void* main_stream = convnet_b200_get_stream();
  convnet_b200_set_stream(side_->stream);
  deriv_output.SumRows(grad_bias_, scale_targets, scale);
  convnet_b200_set_stream(main_stream);
  side_->used = true;
}
void EdgeWithWeight::NoteUp() { bf_up_ = convnet_b200_last_conv_path() == 2 ? 1 : 0; }
void EdgeWithWeight::NoteDown() {
  bf_down_ = convnet_b200_last_conv_path() == 2 ? 1 : 0;
  if (bf_up_ == 0 && bf_down_ == 0) convnet_b200_bf16_invalidate(weights_.GetDevData());     // nobody reads the bf16 weights
}
void EdgeWithWeight::NoteOuter() { bf_outer_ = convnet_b200_last_conv_path() == 2 ? 1 : 0; }

// ---------------------------------------------------------------- optimizer schedules (src/optimizer.cc)
const char* OptimizerConfigError(const OptimizerConfig& c) {
  if (c.epsilon_decay < DECAY_NONE || c.epsilon_decay > EXPONENTIAL_STEP) return "unknown epsilon_decay";
  if (c.epsilon_decay_timescale > 0 && c.epsilon_decay == DECAY_NONE)
    return "epsilon_decay_timescale > 0 needs an epsilon_decay rule";      // optimizer.cc:97-99 exits here
  if (c.optimizer_type == LBFGS) return "optimizer_type LBFGS is not supported (a full-batch method)";
  if (c.optimizer_type != STOCHASTIC_GRADIENT_DESCENT && !IsAdaptive(c)) return "unknown optimizer_type";
  if (!(c.rms_prop_factor >= 0.f && c.rms_prop_factor <= 1.f)) return "rms_prop_factor must lie in [0, 1]";
  return nullptr;
}
void InitAdaptiveState(const OptimizerConfig& c, Matrix& state) {      // optimizer.cc:206-210, 237-241
  if (IsAdaptive(c) && state.GetNumEls() > 0 && state.GetDevData())
    state.Set(c.optimizer_type == ADAGRAD_SGD ? c.adagrad_delta : 1.f);
}
void OptimizerSchedule(const OptimizerConfig& c, long long step, float* epsilon, float* momentum) {
  float eps = c.epsilon;                                                   // GetDecayedEpsilon, :83-104
  if (c.epsilon_decay_timescale > 0) {
    const float f = ((float)step) / c.epsilon_decay_timescale;
    if (c.epsilon_decay == EXPONENTIAL) eps = c.epsilon * std::exp(-f);
    else if (c.epsilon_decay == INVERSE_T) eps = c.epsilon / (1 + f);
    else if (c.epsilon_decay == LINEAR_DECAY) eps = (f < 1) ? (c.epsilon * (1 - f) + c.minimum_epsilon * f) : c.minimum_epsilon;
    else if (c.epsilon_decay == EXPONENTIAL_STEP)
      eps = (float)(c.epsilon * std::pow(c.decay_factor, (int)(step / c.epsilon_decay_timescale)));   // integer quotient
  }
  if (eps < c.minimum_epsilon) eps = c.minimum_epsilon;
  *epsilon = eps;
  *momentum = c.momentum_transition_timescale > 0                          // GetMomentum, :158-165
                  ? c.initial_momentum + (c.final_momentum - c.initial_momentum) *
                                             (1 - std::exp(-((float)step) / c.momentum_transition_timescale))
                  : c.final_momentum;
}

void AppendOptTensor(const OptimizerConfig& o, long long& step, float* w, float* hist, const float* grad, float* state,
                     long long n, int rows, std::vector<CnbOptTensorEx>& out) {   // src/optimizer.cc:174-279
  const bool adagrad = o.optimizer_type == ADAGRAD_SGD, started = step >= o.start_optimization_after;
  if (started || adagrad) {                        // AdagradSGDOptimizer::Optimize updates its history on every step
    float eps = 0.f, mom = 0.f;
    OptimizerSchedule(o, step, &eps, &mom);
    CnbOptTensor t{w, hist, grad, n, eps, mom, o.l2_decay > 0 ? o.l2_decay : 0.f, o.gradient_clip > 0 ? o.gradient_clip : 0.f,
                   rows, CNB_NORM_NONE, 0.f};
    // ApplyConstraints (:75-81): per row of the matrix
    if (o.weight_norm_constraint > 0) { t.norm_mode = CNB_NORM_CONSTRAINT; t.norm_value = o.weight_norm_constraint; }
    else if (o.weight_norm_limit > 0) { t.norm_mode = CNB_NORM_LIMIT; t.norm_value = o.weight_norm_limit; }
    CnbOptTensorEx x{t, CNB_RULE_SGD, 0, nullptr, 0.f, 1.f};
    if (adagrad) {                                 // gradient.Mult(sqrt(step_ + 1)): sqrt of an int, in double
      x.rule = CNB_RULE_ADAGRAD; x.state = state; x.rule_param = o.adagrad_delta;
      x.scale = (float)std::sqrt((double)(step + 1)); x.state_only = started ? 0 : 1;
    } else if (o.optimizer_type == RMSPROP_SGD) {
      x.rule = CNB_RULE_RMSPROP; x.state = state; x.rule_param = o.rms_prop_factor;
    }
    out.push_back(x);
  }
  step++;
}
void EdgeWithWeight::AppendSgdTensors(std::vector<CnbOptTensorEx>& out) {
  // the rows of the weights are the output units; the bias is ONE row (fc_edge.cc:29-32)
  auto add = [&out](const OptimizerConfig& o, long long& step, Matrix& w, Matrix& h, Matrix& g, Matrix& s) {
    AppendOptTensor(o, step, w.GetDevData(), h.GetDevData(), g.GetDevData(), s.GetDevData(), (long long)w.GetNumEls(),
                    w.GetRows(), out);
  };
  add(weight_opt_, weight_step_, weights_, hist_weights_, grad_weights_, state_weights_);
  if (!has_no_bias_) add(bias_opt_, bias_step_, bias_, hist_bias_, grad_bias_, state_bias_);
  num_grads_received_ = 0;
}
bool EdgeWithWeight::OfferFusedBiasGrad(BiasGradTarget* t) {
  if (!BiasIsPerChannel2D()) return false;
  t->grad_bias = grad_bias_.GetDevData();
  t->st = GetNumGradsReceived() > 0 ? 1.f : 0.f;
  t->so = scale_gradients_ / batch_size_;
  bias_grad_fused_ = true;
  return true;
}
void EdgeWithWeight::UpdateWeights() {                       // src/edge_with_weight.cc:96-107: this edge alone
  std::vector<CnbOptTensorEx> t;
  AppendSgdTensors(t);
  cnb_opt_update_multi(t.data(), (int)t.size());
}

void EdgeWithWeight::Initialize(unsigned seed) {             // DENSE_UNIFORM_SQRT_FAN_IN, edge_with_weight.cc:120-128
  const size_t n = weights_.GetNumEls();
  std::vector<float> h(n);
  std::mt19937 gen(seed);
  std::uniform_real_distribution<float> u(-0.5f, 0.5f);
  float init_wt = config_.init_wt > 0 ? config_.init_wt : 1.0f;
  const float scale = 2 * init_wt / std::sqrt(FanIn() / 3.0f);
  for (size_t i = 0; i < n; i++) h[i] = u(gen) * scale;
  weights_.CopyFromHost(h.data(), n);
  cudaStreamSynchronize(Matrix::Stream());
  if (!has_no_bias_) bias_.Set(0);
}

// ---------------------------------------------------------------- ConvEdge (src/conv_edge.cc)
ConvEdge::ConvEdge(const EdgeConfig& c)
    : EdgeWithWeight(c), conv_desc_(Edge::GetConvDesc(c)), partial_sum_y_(0), partial_sum_x_(0),
      shared_bias_(c.shared_bias) {}

void ConvEdge::SetImageSize(int y, int x, int t) {           // :27-38
  Edge::SetImageSize(y, x, t);
  conv_desc_.num_input_channels = num_input_channels_;
  conv_desc_.num_output_channels = num_output_channels_;
  conv_desc_.input_channel_end = num_input_channels_;
  conv_desc_.output_channel_end = num_output_channels_;
  Edge::GetNumModules(conv_desc_, y, x, t, num_modules_y_, num_modules_x_, num_modules_t_);
  if (partial_sum_y_ == 0) partial_sum_y_ = num_modules_y_;
  if (partial_sum_x_ == 0) partial_sum_x_ = num_modules_x_;
}

int ConvEdge::FanIn() const {
  return conv_desc_.kernel_size_y * conv_desc_.kernel_size_x * conv_desc_.kernel_size_t * conv_desc_.num_input_channels;
}

size_t ConvEdge::GetParameterMemoryRequirement() {           // :72-78
  const int input_size = FanIn();
  const int bias_locs = shared_bias_ ? 1 : (num_modules_y_ * num_modules_x_ * num_modules_t_);
  return (size_t)conv_desc_.num_output_channels * (input_size + (has_no_bias_ ? 0 : bias_locs));
}

void ConvEdge::SetMemory(Matrix& p) {                        // :80-96
  const int input_size = FanIn();
  const int bias_locs = shared_bias_ ? 1 : (num_modules_y_ * num_modules_x_ * num_modules_t_);
  p.Reshape(conv_desc_.num_output_channels, -1);
  p.GetSlice(weights_, 0, input_size);
  weights_.SetShape4D(conv_desc_.num_output_channels, conv_desc_.kernel_size_x, conv_desc_.kernel_size_y,
                      conv_desc_.num_input_channels * conv_desc_.kernel_size_t);
  if (!has_no_bias_) {
    p.GetSlice(bias_, input_size, input_size + bias_locs);
    bias_.Reshape(1, -1);
  }
}

void ConvEdge::SetGradMemory(Matrix& p) {                    // :108-136
  const int input_size = FanIn();
  const int bias_locs = shared_bias_ ? 1 : (num_modules_y_ * num_modules_x_ * num_modules_t_);
  p.Reshape(conv_desc_.num_output_channels, -1);
  p.GetSlice(grad_weights_, 0, input_size);
  grad_weights_.SetShape4D_like(weights_);
  if (!has_no_bias_) {
    p.GetSlice(grad_bias_, input_size, input_size + bias_locs);
    grad_bias_.Reshape(1, -1);
  }
}

void ConvEdge::ComputeUp(Matrix& input, Matrix& output, bool overwrite, bool train) {   // :138-170
  const float scale_targets = overwrite ? 0 : 1;
  const int mods = num_modules_y_ * num_modules_x_ * num_modules_t_;
  const bool fused = fuse_relu_ && CanFuseReLU();        // bias (+activation of the destination layer) in the conv epilogue
  StageForUp(input);
  const bool bias_pass = !has_no_bias_ && !fused;          // then the bias kernel, not the conv, writes the output last
  if (emit_up_ && !bias_pass) convnet_b200_emit_bf16_next();
  if (image_size_t_ == 1) {
    if (fused) convnet_b200_fuse_next_act(bias_.GetDevData(), up_act_, nullptr);
    ApplyDropoutRequest(fused);
    Matrix::ConvUp(input, weights_, output, conv_desc_, scale_targets);
  } else {
    Matrix::Conv3DUp(input, weights_, output, conv_desc_, scale_targets);
  }
  NoteUp();
  if (!has_no_bias_ && !fused) {
    if (shared_bias_ && image_size_t_ == 1) {
      output.Reshape(-1, conv_desc_.num_output_channels);
      if (emit_up_) convnet_b200_emit_bf16_next();
      output.AddRowVec(bias_);
      output.Reshape(-1, conv_desc_.num_output_channels * mods);
    } else if (shared_bias_) {                               // 3-D: per output frame (:157-164)
      output.Reshape(-1, conv_desc_.num_output_channels * num_modules_t_);
      for (int m = 0; m < num_modules_t_; m++) {
        Matrix slice;
        output.GetSlice(slice, m * conv_desc_.num_output_channels, (m + 1) * conv_desc_.num_output_channels);
        slice.AddRowVec(bias_);
      }
      output.Reshape(-1, conv_desc_.num_output_channels * mods);
    } else {
      output.AddRowVec(bias_);
    }
  }
}

void ConvEdge::ComputeDown(Matrix& deriv_output, Matrix& input, Matrix& output, Matrix& deriv_input,
                           bool overwrite) {                 // :172-181
  const float scale_targets = overwrite ? 0 : 1;
  StageForBprop(deriv_output);
  if (fuse_mask_) convnet_b200_fuse_next_act(nullptr, down_act_, input.GetDevData());      // activation' of the source layer
  if (emit_down_) convnet_b200_emit_bf16_next();
  ApplyBiasGradRequest();
  if (image_size_t_ == 1) Matrix::ConvDown(deriv_output, weights_, deriv_input, conv_desc_, scale_targets);
  else Matrix::Conv3DDown(deriv_output, weights_, deriv_input, conv_desc_, scale_targets);
  NoteDown();
  if (image_size_t_ == 1) RememberDown(deriv_output, deriv_input);
}
void ConvEdge::PrestageDown() {
  if (!down_out_ || !down_in_ || image_size_t_ != 1) return;
  convnet_b200_prestage_next();
  Matrix::ConvDown(*down_out_, weights_, *down_in_, conv_desc_, 0);
}

void ConvEdge::ComputeOuter(Matrix& input, Matrix& deriv_output) {   // :183-245
  const int batch_size = input.GetRows();
  const int scale_targets = GetNumGradsReceived() > 0 ? 1 : 0;
  const float scale = scale_gradients_ / batch_size;
  const int mods = num_modules_y_ * num_modules_x_ * num_modules_t_;
  StageForBprop(deriv_output);
  if (image_size_t_ == 1) {
    Matrix::ConvOutp(input, deriv_output, grad_weights_, conv_desc_, partial_sum_y_, partial_sum_x_, scale_targets, scale);
  } else {
    Matrix::Conv3DOutp(input, deriv_output, grad_weights_, conv_desc_, scale_targets, scale);
  }
  NoteOuter();
  const bool bias_done = bias_grad_fused_;            // the edge above summed the channels while it wrote the derivative
  bias_grad_fused_ = false;
  if (!has_no_bias_ && !bias_done) {
    if (shared_bias_ && image_size_t_ == 1) {
      // the reference sums in two steps through a temp (:212-218); one deterministic pass here
      deriv_output.Reshape(-1, conv_desc_.num_output_channels);
      SumBiasRows(deriv_output, scale_targets, scale);
      deriv_output.Reshape(batch_size, -1);
    } else if (shared_bias_) {
      deriv_output.Reshape(-1, conv_desc_.num_output_channels * num_modules_t_);
      for (int m = 0; m < num_modules_t_; m++) {
        Matrix slice;
        deriv_output.GetSlice(slice, m * conv_desc_.num_output_channels, (m + 1) * conv_desc_.num_output_channels);
        slice.SumRows(grad_bias_, (m == 0) ? scale_targets : 1, scale);
      }
      deriv_output.Reshape(batch_size, -1);
    } else {
      deriv_output.SumRows(grad_bias_, scale_targets, scale);
    }
  }
  (void)mods;
  IncrementNumGradsReceived();
}

double ConvEdge::FlopsUp() const {
  return 2.0 * batch_size_ * num_modules_y_ * num_modules_x_ * num_modules_t_ * conv_desc_.num_output_channels * FanIn();
}

// ---------------------------------------------------------------- LocalEdge (src/local_edge.cc)
void LocalEdge::SetImageSize(int y, int x, int t) {          // :20-33
  Edge::SetImageSize(y, x, t);
  conv_desc_.num_input_channels = num_input_channels_;
  conv_desc_.num_output_channels = num_output_channels_;
  conv_desc_.input_channel_end = num_input_channels_;
  conv_desc_.output_channel_end = num_output_channels_;
  Edge::GetNumModules(conv_desc_, y, x, t, num_modules_y_, num_modules_x_, num_modules_t_);
}
size_t LocalEdge::GetParameterMemoryRequirement() {           // :53-57
  return (size_t)num_output_channels_ * ((size_t)KernelSize() * Modules() + (has_no_bias_ ? 0 : Modules()));
}
void LocalEdge::SetMemory(Matrix& p) {                        // :59-72
  const int cols = KernelSize() * Modules();
  p.Reshape(num_output_channels_, -1);
  p.GetSlice(weights_, 0, cols);
  weights_.SetShape4D(num_output_channels_, conv_desc_.kernel_size_x, conv_desc_.kernel_size_y,
                      conv_desc_.num_input_channels * Modules());
  if (!has_no_bias_) {
    p.GetSlice(bias_, cols, cols + Modules());
    bias_.Reshape(1, -1);
  }
}
void LocalEdge::SetGradMemory(Matrix& p) {                    // :74-101
  const int cols = KernelSize() * Modules();
  p.Reshape(num_output_channels_, -1);
  p.GetSlice(grad_weights_, 0, cols);
  grad_weights_.SetShape4D_like(weights_);
  if (!has_no_bias_) {
    p.GetSlice(grad_bias_, cols, cols + Modules());
    grad_bias_.Reshape(1, -1);
  }
}
void LocalEdge::ComputeUp(Matrix& input, Matrix& output, bool overwrite, bool train) {   // :103-119
  const bool fused = fuse_relu_ && CanFuseReLU();        // per-feature bias (+activation of the destination layer) in the epilogue
  StageForUp(input);
  const bool bias_pass = !has_no_bias_ && !fused;
  if (emit_up_ && !bias_pass) convnet_b200_emit_bf16_next();
  if (fused) convnet_b200_fuse_next_act(bias_.GetDevData(), up_act_, nullptr);
  ApplyDropoutRequest(fused);
  Matrix::LocalUp(input, weights_, output, conv_desc_, overwrite ? 0 : 1);
  NoteUp();
  if (bias_pass) {                                       // output.AddRowVec(bias_): bias[j] to column j
    if (emit_up_) convnet_b200_emit_bf16_next();
    output.AddRowVec(bias_);
  }
}
void LocalEdge::ComputeDown(Matrix& deriv_output, Matrix& input, Matrix& output, Matrix& deriv_input,
                            bool overwrite) {                 // :121-126
  StageForBprop(deriv_output);
  if (fuse_mask_) convnet_b200_fuse_next_act(nullptr, down_act_, input.GetDevData());
  if (emit_down_) convnet_b200_emit_bf16_next();
  ApplyBiasGradRequest();
  Matrix::LocalDown(deriv_output, weights_, deriv_input, conv_desc_, overwrite ? 0 : 1);
  NoteDown();
}
void LocalEdge::ComputeOuter(Matrix& input, Matrix& deriv_output) {   // :128-139
  const int batch_size = input.GetRows();
  const int scale_targets = GetNumGradsReceived() > 0 ? 1 : 0;
  const float scale = scale_gradients_ / batch_size;
  StageForBprop(deriv_output);
  Matrix::LocalOutp(input, deriv_output, grad_weights_, conv_desc_, scale_targets, scale);
  NoteOuter();
  bias_grad_fused_ = false;                              // (BiasIsPerChannel2D is false: never offered)
  if (!has_no_bias_) SumBiasRows(deriv_output, scale_targets, scale);   // one sum per output feature
  IncrementNumGradsReceived();
}
double LocalEdge::FlopsUp() const { return 2.0 * batch_size_ * Modules() * (double)num_output_channels_ * KernelSize(); }

// ---------------------------------------------------------------- FCEdge (src/fc_edge.cc) as a 1x1 conv on a 1x1 image
static ConvDesc one_by_one(int cin, int cout) {
  ConvDesc d;
  d.num_input_channels = cin; d.num_output_channels = cout;
  d.kernel_size_y = d.kernel_size_x = d.kernel_size_t = 1;
  d.stride_y = d.stride_x = d.stride_t = 1;
  d.padding_y = d.padding_x = d.padding_t = 0;
  d.input_channel_begin = 0; d.input_channel_end = cin; d.output_channel_begin = 0; d.output_channel_end = cout;
  d.num_groups = 1;
  return d;
}

void FCEdge::SetImageSize(int y, int x, int t) {
  Edge::SetImageSize(y, x, t);
  num_modules_y_ = num_modules_x_ = num_modules_t_ = 1;
  num_inputs_ = y * x * t * num_input_channels_;
  desc_ = one_by_one(num_inputs_, num_output_channels_);
}
size_t FCEdge::GetParameterMemoryRequirement() { return (size_t)num_output_channels_ * (num_inputs_ + (has_no_bias_ ? 0 : 1)); }
void FCEdge::SetMemory(Matrix& p) {                          // fc_edge.cc:20-31
  p.Reshape(num_output_channels_, -1);
  p.GetSlice(weights_, 0, num_inputs_);
  weights_.SetShape4D(num_output_channels_, 1, 1, num_inputs_);
  if (!has_no_bias_) { p.GetSlice(bias_, num_inputs_, num_inputs_ + 1); bias_.Reshape(1, -1); }
}
void FCEdge::SetGradMemory(Matrix& p) {
  p.Reshape(num_output_channels_, -1);
  p.GetSlice(grad_weights_, 0, num_inputs_);
  grad_weights_.SetShape4D_like(weights_);
  if (!has_no_bias_) { p.GetSlice(grad_bias_, num_inputs_, num_inputs_ + 1); grad_bias_.Reshape(1, -1); }
}
void FCEdge::View(Matrix& in, Matrix& out) {
  in.SetShape4D(in.GetRows(), 1, 1, num_inputs_);
  out.SetShape4D(out.GetRows(), 1, 1, num_output_channels_);
}
void FCEdge::ComputeUp(Matrix& input, Matrix& output, bool overwrite, bool train) {      // fc_edge.cc:51-60
  Shape4D si = input.GetShape4D(), so = output.GetShape4D();
  View(input, output);
  const bool fused = fuse_relu_ && !has_no_bias_;
  StageForUp(input);
  if (fused) convnet_b200_fuse_next_act(bias_.GetDevData(), up_act_, nullptr);
  const bool bias_pass = !has_no_bias_ && !fused;
  if (emit_up_ && !bias_pass) convnet_b200_emit_bf16_next();
  ApplyDropoutRequest(fused);
  Matrix::ConvUp(input, weights_, output, desc_, overwrite ? 0 : 1);     // output = input * W^T
  NoteUp();
  if (bias_pass) { if (emit_up_) convnet_b200_emit_bf16_next(); output.AddRowVec(bias_); }
  input.GetShape4D() = si; output.GetShape4D() = so;
}
void FCEdge::ComputeDown(Matrix& deriv_output, Matrix& input, Matrix& output, Matrix& deriv_input, bool overwrite) {
  Shape4D si = deriv_input.GetShape4D(), so = deriv_output.GetShape4D();
  View(deriv_input, deriv_output);
  StageForBprop(deriv_output);
  if (fuse_mask_) convnet_b200_fuse_next_act(nullptr, down_act_, input.GetDevData());
  if (emit_down_) convnet_b200_emit_bf16_next();
  ApplyBiasGradRequest();
  Matrix::ConvDown(deriv_output, weights_, deriv_input, desc_, overwrite ? 0 : 1);
  NoteDown();
  deriv_input.GetShape4D() = si; deriv_output.GetShape4D() = so;
}
void FCEdge::ComputeOuter(Matrix& input, Matrix& deriv_output) {                          // fc_edge.cc:69-81
  const int batch_size = input.GetRows();
  const int scale_targets = GetNumGradsReceived() > 0 ? 1 : 0;
  Shape4D si = input.GetShape4D(), so = deriv_output.GetShape4D();
  View(input, deriv_output);
  StageForBprop(deriv_output);
  Matrix::ConvOutp(input, deriv_output, grad_weights_, desc_, 0, 0, scale_targets, scale_gradients_ / batch_size);
  NoteOuter();
  const bool bias_done = bias_grad_fused_;
  bias_grad_fused_ = false;
  if (!has_no_bias_ && !bias_done) SumBiasRows(deriv_output, scale_targets, scale_gradients_ / batch_size);
  input.GetShape4D() = si; deriv_output.GetShape4D() = so;
  IncrementNumGradsReceived();
}
double FCEdge::FlopsUp() const { return 2.0 * batch_size_ * (double)num_inputs_ * num_output_channels_; }

// ---------------------------------------------------------------- ConvOneToOneEdge (src/conv_onetoone_edge.cc)
void ConvOneToOneEdge::SetImageSize(int y, int x, int t) {
  Edge::SetImageSize(y, x, t);
  desc_ = one_by_one(num_input_channels_, num_output_channels_);
}
size_t ConvOneToOneEdge::GetParameterMemoryRequirement() {
  return (size_t)num_output_channels_ * (num_input_channels_ + (has_no_bias_ ? 0 : 1));
}
void ConvOneToOneEdge::SetMemory(Matrix& p) {
  p.Reshape(num_output_channels_, -1);
  p.GetSlice(weights_, 0, num_input_channels_);
  weights_.SetShape4D(num_output_channels_, 1, 1, num_input_channels_);
  if (!has_no_bias_) { p.GetSlice(bias_, num_input_channels_, num_input_channels_ + 1); bias_.Reshape(1, -1); }
}
void ConvOneToOneEdge::SetGradMemory(Matrix& p) {
  p.Reshape(num_output_channels_, -1);
  p.GetSlice(grad_weights_, 0, num_input_channels_);
  grad_weights_.SetShape4D_like(weights_);
  if (!has_no_bias_) { p.GetSlice(grad_bias_, num_input_channels_, num_input_channels_ + 1); grad_bias_.Reshape(1, -1); }
}
void ConvOneToOneEdge::ComputeUp(Matrix& input, Matrix& output, bool overwrite, bool train) {   // :56-73
  const int batch_size = input.GetRows();
  const bool fused = fuse_relu_ && !has_no_bias_;
  StageForUp(input);
  if (fused) convnet_b200_fuse_next_act(bias_.GetDevData(), up_act_, nullptr);
  const bool bias_pass = !has_no_bias_ && !fused;
  if (emit_up_ && !bias_pass) convnet_b200_emit_bf16_next();
  ApplyDropoutRequest(fused);
  Matrix::ConvUp(input, weights_, output, desc_, overwrite ? 0 : 1);
  NoteUp();
  if (!has_no_bias_ && !fused) {
    output.Reshape(-1, num_output_channels_);
    if (emit_up_) convnet_b200_emit_bf16_next();
    output.AddRowVec(bias_);
    output.Reshape(batch_size, -1);
  }
}
void ConvOneToOneEdge::ComputeDown(Matrix& deriv_output, Matrix& input, Matrix& output, Matrix& deriv_input,
                                   bool overwrite) {
  StageForBprop(deriv_output);
  if (fuse_mask_) convnet_b200_fuse_next_act(nullptr, down_act_, input.GetDevData());
  if (emit_down_) convnet_b200_emit_bf16_next();
  ApplyBiasGradRequest();
  Matrix::ConvDown(deriv_output, weights_, deriv_input, desc_, overwrite ? 0 : 1);
  NoteDown();
  RememberDown(deriv_output, deriv_input);
}
void ConvOneToOneEdge::PrestageDown() {
  if (!down_out_ || !down_in_) return;
  convnet_b200_prestage_next();
  Matrix::ConvDown(*down_out_, weights_, *down_in_, desc_, 0);
}
void ConvOneToOneEdge::ComputeOuter(Matrix& input, Matrix& deriv_output) {                        // :87-102
  const int batch_size = input.GetRows();
  const int scale_targets = GetNumGradsReceived() > 0 ? 1 : 0;
  StageForBprop(deriv_output);
  Matrix::ConvOutp(input, deriv_output, grad_weights_, desc_, 0, 0, scale_targets, scale_gradients_ / batch_size);
  NoteOuter();
  const bool bias_done = bias_grad_fused_;
  bias_grad_fused_ = false;
  if (!has_no_bias_ && !bias_done) {
    deriv_output.Reshape(-1, num_output_channels_);
    SumBiasRows(deriv_output, scale_targets, scale_gradients_ / batch_size);
    deriv_output.Reshape(batch_size, -1);
  }
  IncrementNumGradsReceived();
}
double ConvOneToOneEdge::FlopsUp() const {
  return 2.0 * batch_size_ * image_size_y_ * image_size_x_ * image_size_t_ * (double)num_input_channels_ * num_output_channels_;
}

// ---------------------------------------------------------------- MaxPoolEdge / AvgPoolEdge
void MaxPoolEdge::SetImageSize(int y, int x, int t) {        // maxpool_edge.cc:15-26
  Edge::SetImageSize(y, x, t);
  conv_desc_.num_input_channels = num_input_channels_;
  conv_desc_.num_output_channels = num_output_channels_;
  conv_desc_.input_channel_end = num_input_channels_;
  conv_desc_.output_channel_end = num_output_channels_;
  if (conv_desc_.kernel_size_y <= 0) conv_desc_.kernel_size_y = y;     // "global" pooling
  if (conv_desc_.kernel_size_x <= 0) conv_desc_.kernel_size_x = x;
  if (conv_desc_.kernel_size_t <= 0) conv_desc_.kernel_size_t = t;
  Edge::GetNumModules(conv_desc_, y, x, t, num_modules_y_, num_modules_x_, num_modules_t_);
}
void MaxPoolEdge::ComputeUp(Matrix& input, Matrix& output, bool overwrite, bool train) {   // :50-58
  if (!overwrite) {
    fprintf(stderr, " In MaxPoolEdge::ComputeUp() : some other layer is writing to this maxpool layer's output. Not implemented.\n");
    exit(1);
  }
  if (emit_up_) convnet_b200_emit_bf16_next();
  // training: have the kernel record which window elements equal the maximum; ComputeDown then reads those masks instead of
  // re-reading and comparing input and output (nothing between the two calls writes either tensor except through the library,
  // which drops the masks when it does)
  if (train) convnet_b200_pool_cache_next();
  Matrix::ConvMaxPool(input, output, conv_desc_);
}
void MaxPoolEdge::ComputeDown(Matrix& deriv_output, Matrix& input, Matrix& output, Matrix& deriv_input, bool overwrite) {
  if (fuse_mask_) convnet_b200_fuse_next_act(nullptr, down_act_, input.GetDevData());
  if (emit_down_) convnet_b200_emit_bf16_next();
  ApplyBiasGradRequest();
  Matrix::ConvMaxPoolUndo(input, deriv_output, output, deriv_input, conv_desc_, overwrite ? 0 : 1);
}
void AvgPoolEdge::ComputeUp(Matrix& input, Matrix& output, bool overwrite, bool train) {   // avgpool_edge.cc:50-58
  if (!overwrite) { fprintf(stderr, " In AvgPoolEdge::ComputeUp() : not implemented for non-overwrite.\n"); exit(1); }
  if (emit_up_) convnet_b200_emit_bf16_next();
  Matrix::ConvAvgPool(input, output, conv_desc_);
}
void AvgPoolEdge::ComputeDown(Matrix& deriv_output, Matrix& input, Matrix& output, Matrix& deriv_input, bool overwrite) {
  if (fuse_mask_) convnet_b200_fuse_next_act(nullptr, down_act_, input.GetDevData());
  if (emit_down_) convnet_b200_emit_bf16_next();
  ApplyBiasGradRequest();
  Matrix::ConvAvgPoolUndo(deriv_output, deriv_input, conv_desc_, overwrite ? 0 : 1);
}

// ---------------------------------------------------------------- ResponseNormEdge (src/response_norm_edge.cc)
void ResponseNormEdge::SetImageSize(int y, int x, int t) {   // :32-39
  Edge::SetImageSize(y, x, t);
  num_filters_response_norm_ = (int)(frac_of_filters_response_norm_ * num_input_channels_);
}
void ResponseNormEdge::ComputeUp(Matrix& input, Matrix& output, bool overwrite, bool train) {   // :41-51
  if (fuse_relu_ && image_size_t_ == 1) convnet_b200_fuse_next(nullptr, 1, nullptr);     // ReLU of the destination layer
  if (emit_up_) convnet_b200_emit_bf16_next();
  if (image_size_t_ == 1)
    Matrix::ConvResponseNormCrossMap(input, output, num_input_channels_, num_filters_response_norm_, add_scale_, pow_scale_, blocked_);
  else
    Matrix::ConvResponseNormCrossMap3D(input, output, num_input_channels_, num_filters_response_norm_, add_scale_, pow_scale_, blocked_, image_size_t_);
}
void ResponseNormEdge::ComputeDown(Matrix& deriv_output, Matrix& input, Matrix& output, Matrix& deriv_input,
                                   bool overwrite) {         // :53-66 (ignores `overwrite`, like the reference)
  if (emit_down_) convnet_b200_emit_bf16_next();
  if (image_size_t_ == 1)
    Matrix::ConvResponseNormCrossMapUndo(deriv_output, input, output, deriv_input, num_input_channels_, num_filters_response_norm_, add_scale_, pow_scale_, blocked_);
  else
    Matrix::ConvResponseNormCrossMapUndo3D(deriv_output, input, output, deriv_input, num_input_channels_, num_filters_response_norm_, add_scale_, pow_scale_, blocked_, image_size_t_);
}

}  // namespace cnbhost
