// edge.cc — see edge.h.  Sequencing follows the reference's src/*_edge.cc line by line where cited.
#include "edge.h"

#include <cmath>
#include <random>
#include <stdexcept>
#include <string>
#include <vector>

namespace cnbhost {

const char* const kEdgeTypeNames[RGBTOYUV + 1] = {"FC", "CONVOLUTIONAL", "MAXPOOL", "AVERAGE_POOL", "RESPONSE_NORM",
                                                 "CONV_ONETOONE", "LOCAL", "UPSAMPLE", "DOWNSAMPLE", "RGBTOYUV"};

// ---------------------------------------------------------------- Edge (src/edge.cc)
Edge::Edge(const EdgeConfig& c)
    : config_(c), name_(c.name.empty() ? c.source + ":" + c.dest : c.name), source_(nullptr), dest_(nullptr),
      num_input_channels_(0), num_output_channels_(0), image_size_y_(0), image_size_x_(0), image_size_t_(1),
      num_modules_y_(1), num_modules_x_(1), num_modules_t_(1), batch_size_(0) {}

// a chain has one edge into each layer, so every edge overwrites its output: the accumulating paths are not implemented
static void NotOverwrite(const char* what) {
  throw std::logic_error(std::string(what) + ": another edge writes this edge's output, which is not implemented");
}

Edge* Edge::ChooseEdgeClass(const EdgeConfig& c) {          // src/edge.cc:17-60
  switch (c.edge_type) {
    case FC: return new FCEdge(c);
    case CONVOLUTIONAL: return new ConvEdge(c);
    case MAXPOOL: return new MaxPoolEdge(c);
    case AVGPOOL: return new AvgPoolEdge(c);
    case RESPONSE_NORM: return new ResponseNormEdge(c);
    case CONV_ONETOONE: return new ConvOneToOneEdge(c);
    case LOCAL: return new LocalEdge(c);
    case UPSAMPLE: return new UpSampleEdge(c);
    case DOWNSAMPLE: return new DownSampleEdge(c);
    case RGBTOYUV: return new RgbToYuvEdge(c);
  }
  throw std::logic_error("Edge::ChooseEdgeClass: edge type " + std::to_string((int)c.edge_type) + " is not defined");
}

ConvDesc Edge::GetConvDesc(const EdgeConfig& c) {           // src/edge.cc:87-106
  ConvDesc d;
  d.num_input_channels = 0; d.num_output_channels = 0;
  auto pick = [](int v, int fallback) { return v != EdgeConfig::kUnset ? v : fallback; };
  d.kernel_size_y = pick(c.kernel_size_y, c.kernel_size);
  d.kernel_size_x = pick(c.kernel_size_x, c.kernel_size);
  d.kernel_size_t = c.kernel_size_t;
  d.stride_y = pick(c.stride_y, c.stride);
  d.stride_x = pick(c.stride_x, c.stride);
  d.stride_t = c.stride_t;
  d.padding_y = -pick(c.padding_y, c.padding);                      // NEGATED: kernels add it to the window start
  d.padding_x = -pick(c.padding_x, c.padding);
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

void Edge::SetImageSize(int y, int x, int t, ConvDesc& d) {
  Edge::SetImageSize(y, x, t);
  d.num_input_channels = d.input_channel_end = num_input_channels_;
  d.num_output_channels = d.output_channel_end = num_output_channels_;
  Edge::GetNumModules(d, y, x, t, num_modules_y_, num_modules_x_, num_modules_t_);
}

void Edge::ArmUp(const float* bias, bool emit) {
  if (plan_.up_act != CNB_ACT_LINEAR) convnet_b200_fuse_next_act(bias, plan_.up_act, nullptr);
  if (emit) convnet_b200_emit_bf16_next();
  if (up_req_.drop_scale != 0.f) convnet_b200_fuse_next_dropout(up_req_.drop_prob, up_req_.drop_scale, up_req_.drop_seed);
  up_req_ = UpRequest();
}
void Edge::ArmDown(const float* act_state) {
  const DownRequest& r = down_req_;
  if (plan_.down_act != CNB_ACT_LINEAR) convnet_b200_fuse_next_act(nullptr, plan_.down_act, act_state);
  if (r.emit) convnet_b200_emit_bf16_next();
  if (r.bias_grad.grad_bias) convnet_b200_fuse_next_bias_grad(r.bias_grad.grad_bias, r.bias_grad.st, r.bias_grad.so);
  if (r.scale != 1.f) convnet_b200_fuse_next_scale(r.scale);
  down_req_ = DownRequest();
}

// ---------------------------------------------------------------- EdgeWithWeight
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
void EdgeWithWeight::AddBias(Matrix& output, bool emit) {
  const int rows = output.GetRows();
  output.Reshape(-1, bias_.GetCols());
  if (emit) convnet_b200_emit_bf16_next();
  output.AddRowVec(bias_);
  output.Reshape(rows, -1);
}
void EdgeWithWeight::SumBias(Matrix& deriv_output, float scale_targets, float scale) {
  const int rows = deriv_output.GetRows();
  deriv_output.Reshape(-1, bias_.GetCols());
  cudaEventRecord(side_->ready, Matrix::Stream());            // the derivative is final on the main stream
  cudaStreamWaitEvent(side_->stream, side_->ready, 0);
  void* main_stream = convnet_b200_get_stream();
  convnet_b200_set_stream(side_->stream);
  deriv_output.SumRows(grad_bias_, scale_targets, scale);
  convnet_b200_set_stream(main_stream);
  side_->used = true;
  deriv_output.Reshape(rows, -1);
}

size_t EdgeWithWeight::GetParameterMemoryRequirement() {
  if (Tied()) return 0;                                      // it runs on its owner's slice
  return (size_t)num_output_channels_ * (WeightCols() + (has_no_bias_ ? 0 : BiasCols()));
}
void EdgeWithWeight::Carve(Matrix& p, Matrix& w, Matrix& b) {    // e.g. conv_edge.cc:80-96, 108-136
  p.Reshape(num_output_channels_, -1);
  p.GetSlice(w, 0, WeightCols());
  w.GetShape4D() = WeightShape();
  if (!has_no_bias_) {
    p.GetSlice(b, WeightCols(), WeightCols() + BiasCols());
    b.Reshape(1, -1);
  }
}

void EdgeWithWeight::ComputeUp(Matrix& input, Matrix& output, bool overwrite, bool train) {   // e.g. conv_edge.cc:138-170
  const bool bias_pass = !has_no_bias_ && plan_.up_act == CNB_ACT_LINEAR;   // else the bias rides in the epilogue
  const bool emit = up_req_.emit;
  StageForUp(input);
  ArmUp(bias_.GetDevData(), emit && !bias_pass);
  GemmUp(input, output, overwrite ? 0 : 1);
  NoteUp();
  if (bias_pass) AddBias(output, emit);
}
void EdgeWithWeight::ComputeDown(Matrix& deriv_output, Matrix& input, Matrix& output, Matrix& deriv_input,
                                 bool overwrite) {           // e.g. conv_edge.cc:172-181
  StageForBprop(deriv_output);
  ArmDown(input.GetDevData());                               // activation' of the source layer
  GemmDown(deriv_output, deriv_input, overwrite ? 0 : 1);
  NoteDown();
  if (PrestagesDown()) {
    down_out_ = bf_down_ == 1 ? &deriv_output : nullptr;
    down_in_ = bf_down_ == 1 ? &deriv_input : nullptr;
  }
}
void EdgeWithWeight::PrestageDown() {
  if (!down_out_ || !down_in_) return;
  convnet_b200_prestage_next();
  GemmDown(*down_out_, *down_in_, 0);
}
void EdgeWithWeight::ComputeOuter(Matrix& input, Matrix& deriv_output) {   // e.g. conv_edge.cc:183-245
  const int scale_targets = GetNumGradsReceived() > 0 ? 1 : 0;
  const float scale = scale_gradients_ / input.GetRows();
  StageForBprop(deriv_output);
  GemmOuter(input, deriv_output, scale_targets, scale);
  NoteOuter();
  // the reference sums the bias in two steps through a temp (conv_edge.cc:212-218); one deterministic pass here, unless
  // the edge above summed the channels while it wrote the derivative
  if (!has_no_bias_ && !bias_grad_fused_) SumBias(deriv_output, scale_targets, scale);
  bias_grad_fused_ = false;
  IncrementNumGradsReceived();
}

void EdgeWithWeight::NoteUp() { bf_up_ = convnet_b200_last_conv_path() == 2 ? 1 : 0; }
void EdgeWithWeight::NoteDown() {
  bf_down_ = convnet_b200_last_conv_path() == 2 ? 1 : 0;
  // nobody reads the bf16 weights: no edge of the tie group (just this edge when untied) has taken or may take a bf16 path
  for (const EdgeWithWeight* e : owner_->group_)
    if (e->bf_up_ != 0 || e->bf_down_ != 0) return;
  convnet_b200_bf16_invalidate(weights_.GetDevData());
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
Edge::BiasGradTarget EdgeWithWeight::HandOffBiasGrad() {
  bias_grad_fused_ = true;
  return BiasGradTarget{grad_bias_.GetDevData(), GetNumGradsReceived() > 0 ? 1.f : 0.f, scale_gradients_ / batch_size_};
}

// edge_with_weight.cc:108-143, on the host RNG: the fan-in is the weight columns (:116, :126); init_wt is taken as given
// (CONSTANT with init_wt 0 gives zeros)
std::vector<float> EdgeWithWeight::InitialWeights(unsigned seed) const {
  const size_t n = (size_t)num_output_channels_ * WeightCols();
  std::vector<float> h(n);
  std::mt19937 gen(seed);
  const int init = config_.initialization;
  const float init_wt = config_.init_wt;
  if (init == DENSE_UNIFORM || init == DENSE_UNIFORM_SQRT_FAN_IN) {
    std::uniform_real_distribution<float> u(-0.5f, 0.5f);
    const float scale = init == DENSE_UNIFORM ? 2 * init_wt : 2 * init_wt / std::sqrt(WeightCols() / 3.0f);
    for (size_t i = 0; i < n; i++) h[i] = u(gen) * scale;
  } else if (init == DENSE_GAUSSIAN || init == DENSE_GAUSSIAN_SQRT_FAN_IN) {
    std::normal_distribution<float> g(0.f, 1.f);
    const float scale = init == DENSE_GAUSSIAN ? init_wt : init_wt / std::sqrt((float)WeightCols());
    for (size_t i = 0; i < n; i++) h[i] = g(gen) * scale;
  } else {                                                   // CONSTANT (ConvNet::Refuse admits no other rule)
    for (size_t i = 0; i < n; i++) h[i] = init_wt;
  }
  return h;
}
void EdgeWithWeight::Initialize(unsigned seed) {
  // PRETRAINED: ConvNet::AllocateMemory reads it from its checkpoint; a tied edge's parameters are its owner's
  if (config_.initialization == PRETRAINED || Tied()) return;
  const std::vector<float> h = InitialWeights(seed);
  const size_t n = weights_.GetNumEls();
  weights_.CopyFromHost(h.data(), n);
  cudaStreamSynchronize(Matrix::Stream());
  if (!has_no_bias_) bias_.Set(config_.init_bias);
}

// ---------------------------------------------------------------- ConvEdge (src/conv_edge.cc)
ConvEdge::ConvEdge(const EdgeConfig& c)
    : EdgeWithWeight(c), conv_desc_(Edge::GetConvDesc(c)), partial_sum_y_(0), partial_sum_x_(0),
      shared_bias_(c.shared_bias) {}

void ConvEdge::SetImageSize(int y, int x, int t) {           // :27-38
  Edge::SetImageSize(y, x, t, conv_desc_);
  if (partial_sum_y_ == 0) partial_sum_y_ = num_modules_y_;
  if (partial_sum_x_ == 0) partial_sum_x_ = num_modules_x_;
}

int ConvEdge::WeightCols() const {                           // :72-78
  return conv_desc_.kernel_size_y * conv_desc_.kernel_size_x * conv_desc_.kernel_size_t * conv_desc_.num_input_channels;
}
Shape4D ConvEdge::WeightShape() const {                      // :80-96
  return Shape4D{{conv_desc_.num_output_channels, conv_desc_.kernel_size_x, conv_desc_.kernel_size_y,
                  conv_desc_.num_input_channels * conv_desc_.kernel_size_t}};
}

void ConvEdge::GemmUp(Matrix& input, Matrix& output, float scale_targets) {   // :138-170
  if (image_size_t_ == 1) Matrix::ConvUp(input, weights_, output, conv_desc_, scale_targets);
  else Matrix::Conv3DUp(input, weights_, output, conv_desc_, scale_targets);
}
void ConvEdge::GemmDown(Matrix& deriv_output, Matrix& deriv_input, float scale_targets) {   // :172-181
  if (image_size_t_ == 1) Matrix::ConvDown(deriv_output, weights_, deriv_input, conv_desc_, scale_targets);
  else Matrix::Conv3DDown(deriv_output, weights_, deriv_input, conv_desc_, scale_targets);
}
void ConvEdge::GemmOuter(Matrix& input, Matrix& deriv_output, float scale_targets, float scale) {   // :183-245
  if (image_size_t_ == 1)
    Matrix::ConvOutp(input, deriv_output, grad_weights_, conv_desc_, partial_sum_y_, partial_sum_x_, scale_targets, scale);
  else
    Matrix::Conv3DOutp(input, deriv_output, grad_weights_, conv_desc_, scale_targets, scale);
}

// 3-D: one bias per channel added to each output frame (:157-164); unshared: one per output column.  Neither takes the emit
// request, and both gradients are summed on the main stream
void ConvEdge::AddBias(Matrix& output, bool emit) {
  if (shared_bias_ && image_size_t_ == 1) return EdgeWithWeight::AddBias(output, emit);
  if (!shared_bias_) return output.AddRowVec(bias_);
  const int rows = output.GetRows(), c = conv_desc_.num_output_channels;
  output.Reshape(-1, c * num_modules_t_);
  for (int m = 0; m < num_modules_t_; m++) {
    Matrix slice;
    output.GetSlice(slice, m * c, (m + 1) * c);
    slice.AddRowVec(bias_);
  }
  output.Reshape(rows, -1);
}
void ConvEdge::SumBias(Matrix& deriv_output, float scale_targets, float scale) {
  if (shared_bias_ && image_size_t_ == 1) return EdgeWithWeight::SumBias(deriv_output, scale_targets, scale);
  if (!shared_bias_) return deriv_output.SumRows(grad_bias_, scale_targets, scale);
  const int rows = deriv_output.GetRows(), c = conv_desc_.num_output_channels;
  deriv_output.Reshape(-1, c * num_modules_t_);
  for (int m = 0; m < num_modules_t_; m++) {
    Matrix slice;
    deriv_output.GetSlice(slice, m * c, (m + 1) * c);
    slice.SumRows(grad_bias_, (m == 0) ? scale_targets : 1, scale);
  }
  deriv_output.Reshape(rows, -1);
}

double ConvEdge::FlopsUp() const {
  return 2.0 * batch_size_ * num_modules_y_ * num_modules_x_ * num_modules_t_ * conv_desc_.num_output_channels * WeightCols();
}

// ---------------------------------------------------------------- LocalEdge (src/local_edge.cc)
void LocalEdge::SetImageSize(int y, int x, int t) { Edge::SetImageSize(y, x, t, conv_desc_); }   // :20-33
Shape4D LocalEdge::WeightShape() const {                      // :59-72
  return Shape4D{{num_output_channels_, conv_desc_.kernel_size_x, conv_desc_.kernel_size_y,
                  conv_desc_.num_input_channels * Modules()}};
}
void LocalEdge::GemmUp(Matrix& input, Matrix& output, float scale_targets) {   // :103-119
  Matrix::LocalUp(input, weights_, output, conv_desc_, scale_targets);
}
void LocalEdge::GemmDown(Matrix& deriv_output, Matrix& deriv_input, float scale_targets) {   // :121-126
  Matrix::LocalDown(deriv_output, weights_, deriv_input, conv_desc_, scale_targets);
}
void LocalEdge::GemmOuter(Matrix& input, Matrix& deriv_output, float scale_targets, float scale) {   // :128-139
  Matrix::LocalOutp(input, deriv_output, grad_weights_, conv_desc_, scale_targets, scale);
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
// [images x features] seen by the conv entry points as images of 1x1 pixels and `features` channels, for one call
struct FlatView {
  Matrix& m;
  Shape4D saved;
  FlatView(Matrix& x, int features) : m(x), saved(x.GetShape4D()) { x.SetShape4D(x.GetRows(), 1, 1, features); }
  ~FlatView() { m.GetShape4D() = saved; }
};
void FCEdge::GemmUp(Matrix& input, Matrix& output, float scale_targets) {      // fc_edge.cc:51-60: output = input * W^T
  FlatView i(input, num_inputs_), o(output, num_output_channels_);
  Matrix::ConvUp(input, weights_, output, desc_, scale_targets);
}
void FCEdge::GemmDown(Matrix& deriv_output, Matrix& deriv_input, float scale_targets) {
  FlatView i(deriv_input, num_inputs_), o(deriv_output, num_output_channels_);
  Matrix::ConvDown(deriv_output, weights_, deriv_input, desc_, scale_targets);
}
void FCEdge::GemmOuter(Matrix& input, Matrix& deriv_output, float scale_targets, float scale) {   // fc_edge.cc:69-81
  FlatView i(input, num_inputs_), o(deriv_output, num_output_channels_);
  Matrix::ConvOutp(input, deriv_output, grad_weights_, desc_, 0, 0, scale_targets, scale);
}
double FCEdge::FlopsUp() const { return 2.0 * batch_size_ * (double)num_inputs_ * num_output_channels_; }

// ---------------------------------------------------------------- ConvOneToOneEdge (src/conv_onetoone_edge.cc)
void ConvOneToOneEdge::SetImageSize(int y, int x, int t) {
  Edge::SetImageSize(y, x, t);
  desc_ = one_by_one(num_input_channels_, num_output_channels_);
}
void ConvOneToOneEdge::GemmUp(Matrix& input, Matrix& output, float scale_targets) {   // :56-73
  Matrix::ConvUp(input, weights_, output, desc_, scale_targets);
}
void ConvOneToOneEdge::GemmDown(Matrix& deriv_output, Matrix& deriv_input, float scale_targets) {
  Matrix::ConvDown(deriv_output, weights_, deriv_input, desc_, scale_targets);
}
void ConvOneToOneEdge::GemmOuter(Matrix& input, Matrix& deriv_output, float scale_targets, float scale) {   // :87-102
  Matrix::ConvOutp(input, deriv_output, grad_weights_, desc_, 0, 0, scale_targets, scale);
}
double ConvOneToOneEdge::FlopsUp() const {
  return 2.0 * batch_size_ * image_size_y_ * image_size_x_ * image_size_t_ * (double)num_input_channels_ * num_output_channels_;
}

// ---------------------------------------------------------------- MaxPoolEdge / AvgPoolEdge
void MaxPoolEdge::SetImageSize(int y, int x, int t) {        // maxpool_edge.cc:15-26
  if (conv_desc_.kernel_size_y <= 0) conv_desc_.kernel_size_y = y;     // "global" pooling
  if (conv_desc_.kernel_size_x <= 0) conv_desc_.kernel_size_x = x;
  if (conv_desc_.kernel_size_t <= 0) conv_desc_.kernel_size_t = t;
  Edge::SetImageSize(y, x, t, conv_desc_);
}
void MaxPoolEdge::ComputeUp(Matrix& input, Matrix& output, bool overwrite, bool train) {   // :50-58
  if (!overwrite) NotOverwrite("MaxPoolEdge::ComputeUp()");
  ArmUp(nullptr, up_req_.emit);
  // training: have the kernel record which window elements equal the maximum; ComputeDown then reads those masks instead of
  // re-reading and comparing input and output (nothing between the two calls writes either tensor except through the library,
  // which drops the masks when it does)
  if (train) convnet_b200_pool_cache_next();
  Matrix::ConvMaxPool(input, output, conv_desc_);
}
void MaxPoolEdge::ComputeDown(Matrix& deriv_output, Matrix& input, Matrix& output, Matrix& deriv_input, bool overwrite) {
  ArmDown(input.GetDevData());
  Matrix::ConvMaxPoolUndo(input, deriv_output, output, deriv_input, conv_desc_, overwrite ? 0 : 1);
}
void AvgPoolEdge::ComputeUp(Matrix& input, Matrix& output, bool overwrite, bool train) {   // avgpool_edge.cc:50-58
  if (!overwrite) NotOverwrite("AvgPoolEdge::ComputeUp()");
  ArmUp(nullptr, up_req_.emit);
  Matrix::ConvAvgPool(input, output, conv_desc_);
}
void AvgPoolEdge::ComputeDown(Matrix& deriv_output, Matrix& input, Matrix& output, Matrix& deriv_input, bool overwrite) {
  ArmDown(input.GetDevData());
  Matrix::ConvAvgPoolUndo(deriv_output, deriv_input, conv_desc_, overwrite ? 0 : 1);
}

// ---------------------------------------------------------------- ResponseNormEdge (src/response_norm_edge.cc)
void ResponseNormEdge::SetImageSize(int y, int x, int t) {   // :32-39
  Edge::SetImageSize(y, x, t);
  num_filters_response_norm_ = (int)(frac_of_filters_response_norm_ * num_input_channels_);
}
void ResponseNormEdge::ComputeUp(Matrix& input, Matrix& output, bool overwrite, bool train) {   // :41-51
  ArmUp(nullptr, up_req_.emit);                              // (ReLU of the destination layer)
  if (image_size_t_ == 1)
    Matrix::ConvResponseNormCrossMap(input, output, num_input_channels_, num_filters_response_norm_, add_scale_, pow_scale_, blocked_);
  else
    Matrix::ConvResponseNormCrossMap3D(input, output, num_input_channels_, num_filters_response_norm_, add_scale_, pow_scale_, blocked_, image_size_t_);
}
void ResponseNormEdge::ComputeDown(Matrix& deriv_output, Matrix& input, Matrix& output, Matrix& deriv_input,
                                   bool overwrite) {         // :53-66 (ignores `overwrite`, like the reference)
  ArmDown(nullptr);
  if (image_size_t_ == 1)
    Matrix::ConvResponseNormCrossMapUndo(deriv_output, input, output, deriv_input, num_input_channels_, num_filters_response_norm_, add_scale_, pow_scale_, blocked_);
  else
    Matrix::ConvResponseNormCrossMapUndo3D(deriv_output, input, output, deriv_input, num_input_channels_, num_filters_response_norm_, add_scale_, pow_scale_, blocked_, image_size_t_);
}

// ---------------------------------------------------------------- UpSampleEdge / DownSampleEdge / RgbToYuvEdge
ConvDesc SampleEdge::Desc() const {
  ConvDesc d = Edge::GetConvDesc(config_);
  d.kernel_size_y = d.kernel_size_x = d.stride_y = d.stride_x = factor_;
  d.kernel_size_t = d.stride_t = 1;
  d.padding_y = d.padding_x = d.padding_t = 0;
  d.num_input_channels = d.num_output_channels = d.input_channel_end = d.output_channel_end = num_input_channels_ * image_size_t_;
  return d;
}

void UpSampleEdge::SetImageSize(int y, int x, int t) {        // upsample_edge.cc:17-22
  Edge::SetImageSize(y, x, t);
  num_modules_y_ = y * factor_;
  num_modules_x_ = x * factor_;
}
void UpSampleEdge::ComputeUp(Matrix& input, Matrix& output, bool overwrite, bool train) {
  ArmUp(nullptr, up_req_.emit);
  UpSampleGemm(input.GetMat(), output.GetMat(), &input.GetShape4D(), &output.GetShape4D(), factor_, overwrite ? 0 : 1);
}
// the derivative of replication: the sum over each f x f block
void UpSampleEdge::ComputeDown(Matrix& deriv_output, Matrix& input, Matrix& output, Matrix& deriv_input, bool overwrite) {
  if (!overwrite) NotOverwrite("UpSampleEdge::ComputeDown()");
  ArmDown(input.GetDevData());
  AvgPoolGemm(deriv_output.GetMat(), deriv_input.GetMat(), &deriv_output.GetShape4D(), &deriv_input.GetShape4D(), Desc(), 0,
              (float)(factor_ * factor_));
}

void DownSampleEdge::SetImageSize(int y, int x, int t) {      // (the reference multiplies here, DESIGN.md §5)
  Edge::SetImageSize(y, x, t);
  num_modules_y_ = factor_ > 0 ? y / factor_ : 0;            // (a factor below 1 is refused: SampleEdgeError)
  num_modules_x_ = factor_ > 0 ? x / factor_ : 0;
}
void DownSampleEdge::ComputeUp(Matrix& input, Matrix& output, bool overwrite, bool train) {
  if (!overwrite) NotOverwrite("DownSampleEdge::ComputeUp()");
  ArmUp(nullptr, up_req_.emit);
  DownSampleGemm(input.GetMat(), output.GetMat(), &input.GetShape4D(), &output.GetShape4D(), factor_);
}
// the derivative of the block mean: d / f^2 to every element of the block, AvgPoolEdge's call
void DownSampleEdge::ComputeDown(Matrix& deriv_output, Matrix& input, Matrix& output, Matrix& deriv_input, bool overwrite) {
  ArmDown(input.GetDevData());
  Matrix::ConvAvgPoolUndo(deriv_output, deriv_input, Desc(), overwrite ? 0 : 1);
}

void RgbToYuvEdge::ComputeUp(Matrix& input, Matrix& output, bool overwrite, bool train) {   // rgbtoyuv_edge.cc
  if (!overwrite) NotOverwrite("RgbToYuvEdge::ComputeUp()");
  ArmUp(nullptr, up_req_.emit);
  Matrix::ConvRGBToYUV(input, output);
}
void RgbToYuvEdge::ComputeDown(Matrix&, Matrix&, Matrix&, Matrix&, bool) {
  throw std::logic_error("RgbToYuvEdge::ComputeDown: RGBTOYUV has no backward pass");
}

}  // namespace cnbhost
