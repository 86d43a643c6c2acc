// edge.h — the Edge operator API of the reference (src/edge.h:20-190, src/edge_with_weight.h:10-58)
// and the six edge types on the BASELINE configs' path, on top of the host Matrix facade.
//
//   ConvEdge            src/conv_edge.{h,cc}            conv -> shared bias ; wgrad -> bias grad
//   MaxPoolEdge         src/maxpool_edge.{h,cc}
//   AvgPoolEdge         src/avgpool_edge.{h,cc}
//   ResponseNormEdge    src/response_norm_edge.{h,cc}
//   FCEdge              src/fc_edge.{h,cc}              (reference: Matrix::Dot / cublasSgemm)
//   ConvOneToOneEdge    src/conv_onetoone_edge.{h,cc}   (reference: Matrix::Dot / cublasSgemm)
//   LocalEdge           src/local_edge.{h,cc}           untied conv -> per-feature bias ; wgrad -> bias grad
// FC and 1x1 edges run on the same implicit-GEMM conv kernels (a 1x1 convolution IS that GEMM),
// SURVEY.md §8(f) rank 1.  The protobuf `config::Edge` is replaced by the plain EdgeConfig struct
// (protobuf is not in the image); field names follow proto/convnet_config.proto:120-221.
#pragma once
#include <string>
#include <vector>

#include "matrix.h"

namespace cnbhost {

class Layer;

enum EdgeType { FC, CONVOLUTIONAL, MAXPOOL, AVGPOOL, RESPONSE_NORM, CONV_ONETOONE, LOCAL };

// proto/convnet_config.proto:64-113 Optimizer, the fields of the SGD, Adagrad and RMSProp paths (src/optimizer.cc:174-279),
// with the proto's names, numbers and defaults.  Plain C layout: the C API (capi.cc) and net.py's ctypes mirror pass it as is.
enum EpsilonDecay { DECAY_NONE = 0, INVERSE_T = 1, EXPONENTIAL = 2, LINEAR_DECAY = 3, EXPONENTIAL_STEP = 4 };
enum OptimizerType { STOCHASTIC_GRADIENT_DESCENT = 0, LBFGS = 1, ADAGRAD_SGD = 2, RMSPROP_SGD = 3 };
struct OptimizerConfig {
  float epsilon = 0.f;
  int epsilon_decay = DECAY_NONE;
  int epsilon_decay_timescale = 0;
  float minimum_epsilon = 0.f;
  float decay_factor = 1.f;                  // EXPONENTIAL_STEP
  float initial_momentum = 0.f;
  float final_momentum = 0.f;                // the momentum when momentum_transition_timescale is 0
  int momentum_transition_timescale = 0;
  float l2_decay = 0.f;
  float gradient_clip = -1.f;                // <= 0: no clipping
  int start_optimization_after = 0;
  float weight_norm_limit = 0.f;             // per-row (output unit) norm cap, 0: none
  float weight_norm_constraint = 0.f;        // per-row norm set to this value, 0: none (wins over the limit)
  int optimizer_type = STOCHASTIC_GRADIENT_DESCENT;
  float adagrad_delta = 1.f;                 // ADAGRAD_SGD: the state starts here
  float rms_prop_factor = 0.f;               // RMSPROP_SGD: running-average factor of the squared gradient, in [0, 1]
};
// nullptr if `c` can run, else why not (GetDecayedEpsilon exits on a timescale without a decay rule; LBFGS is not supported)
const char* OptimizerConfigError(const OptimizerConfig& c);
// ADAGRAD_SGD / RMSPROP_SGD: the optimizer keeps one state float per parameter
inline bool IsAdaptive(const OptimizerConfig& c) { return c.optimizer_type == ADAGRAD_SGD || c.optimizer_type == RMSPROP_SGD; }
// the state a tensor under `c` starts from (adagrad_delta or 1), into `state` (no-op for SGD or an empty slice)
void InitAdaptiveState(const OptimizerConfig& c, Matrix& state);
// (epsilon, momentum) of the update after `step` earlier ones: GetDecayedEpsilon / GetMomentum, optimizer.cc:83-104,158-165
void OptimizerSchedule(const OptimizerConfig& c, long long step, float* epsilon, float* momentum);
// one tensor's update under optimizer `o` (SGD / Adagrad / RMSProp ::Optimize, optimizer.cc:174-279), appended to `out`
// unless the optimizer is still before start_optimization_after (an Adagrad tensor is then appended for its state
// alone); advances `step` either way.  `rows`: the norm groups of the tensor; `state`: its adaptive state (adaptive rules)
void AppendOptTensor(const OptimizerConfig& o, long long& step, float* w, float* hist, const float* grad, float* state,
                     long long n, int rows, std::vector<CnbOptTensorEx>& out);

struct EdgeConfig {
  std::string name, source, dest;
  EdgeType edge_type = FC;
  int kernel_size = 1, stride = 1, padding = 0;
  int kernel_size_y = 0, kernel_size_x = 0, stride_y = 0, stride_x = 0, padding_y = -1, padding_x = -1;   // 0/-1: unset
  int kernel_size_t = 1, stride_t = 1, padding_t = 0;
  bool shared_bias = true, has_no_bias = false;
  float add_scale = 0.0005f, pow_scale = 0.75f, frac_of_filters_response_norm = 0.25f;
  bool response_norm_in_blocks = false;
  float scale_gradients = 1.f;
  float init_wt = 0.f;               // 0: DENSE_UNIFORM_SQRT_FAN_IN (edge_with_weight.cc:120-128)
  OptimizerConfig weight_optimizer, bias_optimizer;
  bool grad_check = false;
  int grad_check_num_params = 10;
  std::vector<float> grad_check_epsilon;
};

class Edge {
 public:
  explicit Edge(const EdgeConfig& c);
  virtual ~Edge() {}
  static Edge* ChooseEdgeClass(const EdgeConfig& c);                     // src/edge.cc:17-60
  static ConvDesc GetConvDesc(const EdgeConfig& c);                      // src/edge.cc:87-106 (negates padding)
  static void GetNumModules(const ConvDesc d, int image_size_y, int image_size_x, int image_size_t,
                            int& num_modules_y, int& num_modules_x, int& num_modules_t);   // src/edge.cc:108-114

  virtual void ComputeUp(Matrix& input, Matrix& output, bool overwrite, bool train) = 0;
  virtual void ComputeDown(Matrix& deriv_output, Matrix& input, Matrix& output, Matrix& deriv_input,
                           bool overwrite) = 0;
  virtual void ComputeOuter(Matrix& input, Matrix& deriv_output) {}
  virtual void UpdateWeights() {}
  virtual void SetMemory(Matrix& p) {}
  virtual void SetGradMemory(Matrix& p) {}
  virtual void SetHistoryMemory(Matrix& p) {}
  virtual size_t GetParameterMemoryRequirement() { return 0; }
  virtual void Initialize(unsigned seed) {}
  virtual bool HasNoParameters() const { return true; }
  virtual void SetImageSize(int image_size_y, int image_size_x, int image_size_t);
  virtual double FlopsUp() const { return 0; }                           // 2*MACs per batch (BASELINE.md §2c)

  int GetNumModulesY() const { return num_modules_y_; }
  int GetNumModulesX() const { return num_modules_x_; }
  int GetNumModulesT() const { return num_modules_t_; }
  void SetInputChannels(int a) { num_input_channels_ = a; }
  void SetOutputChannels(int a) { num_output_channels_ = a; }
  int GetNumOutputChannels() const { return num_output_channels_; }
  const std::string& GetName() const { return name_; }
  const EdgeConfig& Config() const { return config_; }
  Layer* GetSource() { return source_; }
  Layer* GetDest() { return dest_; }
  void SetSource(Layer* l) { source_ = l; }
  void SetDest(Layer* l) { dest_ = l; }
  void SetBatchSize(int n) { batch_size_ = n; }
  // Epilogue fusion (convnet_b200_fuse_next): the ReLU of the destination layer rides in ComputeUp's conv epilogue
  // (together with the shared bias), the ReLU derivative of the source layer in ComputeDown's. ConvNet decides.
  // The activation is that of the layer (CNB_ACT_*: ReLU or logistic): `up` the destination's, `down` the source's.  Where
  // CanFuseReLU / CanFuseMask hold, the ReLU rides in the epilogue; the logistic unit only where CanFuseLogistic holds too
  virtual bool CanFuseReLU() const { return false; }
  virtual bool CanFuseMask() const { return false; }
  virtual bool CanFuseLogistic() const { return false; }
  void SetFuseActs(int up, int down) { up_act_ = up; down_act_ = down; }
  void SetFuseReLU(bool v) { fuse_relu_ = v; }
  void SetFuseMask(bool v) { fuse_mask_ = v; }
  bool WantsFuseReLU() const { return fuse_relu_; }
  bool WantsFuseMask() const { return fuse_mask_; }
  // bf16 mode: the kernel that writes a tensor LAST also leaves its bf16 copy for the conv edge that reads it next
  // (convnet_b200_emit_bf16_next) instead of that edge running a conversion pass.  ConvNet sets these before each call:
  // emit_up: ComputeUp is the last writer of the destination state and the next edge multiplies in bf16;
  // emit_down: ComputeDown is the last writer of the source layer's derivative and the edge below multiplies in bf16.
  void SetEmitUp(bool v) { emit_up_ = v; }
  void SetEmitDown(bool v) { emit_down_ = v; }
  // Fused bias gradient: the edge ABOVE writes this edge's output derivative last, and its kernel can sum the channels
  // while it stores them (convnet_b200_fuse_next_bias_grad).  ConvNet asks the lower edge for its target (which makes that
  // edge skip its own SumRows in ComputeOuter) and hands it to the upper edge's ComputeDown.
  struct BiasGradTarget { float* grad_bias = nullptr; float st = 0.f, so = 1.f; };
  virtual bool OfferFusedBiasGrad(BiasGradTarget*) { return false; }
  void SetBiasGradRequest(const BiasGradTarget& t) { bg_request_ = t; }
  // ComputeDown multiplies the derivative it writes by this factor (1 = none): the dropout derivative of a ReLU layer folded
  // into the dgrad epilogue (convnet_b200_fuse_next_scale); only edges whose ComputeDown is a conv dgrad with the mask fused
  void SetDerivScale(float s) { deriv_scale_ = s; }
  virtual bool CanScaleDeriv() const { return false; }
  // The dropout of the destination layer rides in ComputeUp's conv epilogue behind the fused bias + ReLU
  // (convnet_b200_fuse_next_dropout: no mask tensor — ConvNet asks only when the backward pass folds the dropout derivative
  // into the dgrad above, see ConvNet::DropoutFolds).  One-shot: the next ComputeUp consumes it.
  virtual bool CanFuseDropout() const { return false; }
  void SetDropoutRequest(float prob, float scale, unsigned long long seed) { drop_prob_ = prob; drop_scale_ = scale; drop_seed_ = seed; }
  virtual bool CanProduceBiasGrad() const { return false; }   // ComputeDown kernels that take the request
  virtual bool WantsBf16Input() const { return false; }      // this edge reads its input (fprop / wgrad) as bf16
  virtual bool WantsBf16Deriv() const { return false; }      // this edge reads its output derivative (wgrad / dgrad) as bf16

 protected:
  EdgeConfig config_;
  std::string name_;
  Layer *source_, *dest_;
  int num_input_channels_, num_output_channels_;
  int image_size_y_, image_size_x_, image_size_t_;
  int num_modules_y_, num_modules_x_, num_modules_t_;
  int batch_size_;
  bool fuse_relu_ = false, fuse_mask_ = false;      // the activation / its derivative is fused (whichever it is)
  int up_act_ = CNB_ACT_RELU, down_act_ = CNB_ACT_RELU;
  bool emit_up_ = false, emit_down_ = false;
  BiasGradTarget bg_request_;
  float deriv_scale_ = 1.f;
  float drop_prob_ = 0.f, drop_scale_ = 0.f;
  unsigned long long drop_seed_ = 0;
  void ApplyDropoutRequest(bool fused_epilogue) {   // call right before the ComputeUp kernel (after convnet_b200_fuse_next)
    if (drop_scale_ != 0.f && fused_epilogue) convnet_b200_fuse_next_dropout(drop_prob_, drop_scale_, drop_seed_);
    drop_scale_ = 0.f;
  }
  void ApplyBiasGradRequest() {            // call right before the ComputeDown kernel
    if (bg_request_.grad_bias) convnet_b200_fuse_next_bias_grad(bg_request_.grad_bias, bg_request_.st, bg_request_.so);
    bg_request_ = BiasGradTarget();
    if (deriv_scale_ != 1.f) convnet_b200_fuse_next_scale(deriv_scale_);
    deriv_scale_ = 1.f;
  }
};

// The side stream of ConvNet::TrainOneBatch (all-reduce + optimizer, see convnet.h): bias-gradient column sums are
// memory-bound passes over a derivative that is already final, so they run there, beside the tensor-bound wgrad / dgrad
// kernels of the main stream.  ConvNet::AllocateMemory gives every weighted edge the lane together with its gradient memory.
struct SideLane { cudaStream_t stream = nullptr; cudaEvent_t ready = nullptr; bool used = false; };

class EdgeWithWeight : public Edge {
 public:
  void SetSideLane(SideLane* s) { side_ = s; }
  // after this edge's optimizer step, on the optimizer's stream: rebuild what the next ComputeDown derives from the
  // weights alone (convnet_b200_prestage_next), off the next step's critical path.  Default: nothing to prepare.
  virtual void PrestageDown() {}
  explicit EdgeWithWeight(const EdgeConfig& c)
      : Edge(c), has_no_bias_(c.has_no_bias), scale_gradients_(c.scale_gradients), num_grads_received_(0),
        weight_opt_(c.weight_optimizer), bias_opt_(c.bias_optimizer) {}
  bool HasNoParameters() const override { return false; }
  void UpdateWeights() override;                                         // src/edge_with_weight.cc:96-118
  void SetHistoryMemory(Matrix& p) override;
  void SetStateMemory(Matrix& p);          // the adaptive optimizer state, carved like the history
  void InitState(int which);               // the state of the weights (0) or the bias (1) back to its optimizer's start
  void Initialize(unsigned seed) override;
  Matrix& GetWeight() { return weights_; }
  Matrix& GetGradWeight() { return grad_weights_; }
  Matrix& GetBias() { return bias_; }
  Matrix& GetGradBias() { return grad_bias_; }
  int GetNumGradsReceived() const { return num_grads_received_; }
  void IncrementNumGradsReceived() { num_grads_received_++; }
  void NotifyStart() { num_grads_received_ = 0; }
  virtual int FanIn() const = 0;
  // bf16 mode (convnet_b200_set_conv_precision(2)): each tensor this edge feeds to two conv calls of a step has ONE bf16
  // copy — the input (fprop + wgrad), the output derivative (wgrad + dgrad) and the weights (fprop + dgrad).  The copy is
  // normally written by the kernel that produced the tensor (emit_up / emit_down of the neighbouring edges, the dropout
  // and SGD kernels); convnet_b200_bf16_ensure converts only when no valid copy exists.  Which calls really run in bf16 is
  // learnt from convnet_b200_last_conv_path() during the first step (FC-shaped calls stay on tf32 and are not staged).
  bool WantsBf16Input() const override { return bf_up_ == 1 || bf_outer_ == 1; }
  bool WantsBf16Deriv() const override { return bf_outer_ == 1 || bf_down_ == 1; }
  // weights (+ bias) of this edge for one multi-tensor update with this update's (epsilon, momentum); advances both
  // optimizers' step counts (a tensor whose optimizer is still before start_optimization_after is left out)
  void AppendSgdTensors(std::vector<CnbOptTensorEx>& out);
  // the optimizer of the weights (which = 0) or of the bias (1): its settings, and how many updates it has counted
  OptimizerConfig& Optimizer(int which) { return which ? bias_opt_ : weight_opt_; }
  long long OptimizerStep(int which) const { return which ? bias_step_ : weight_step_; }
  void ReduceLearningRate(float factor) { weight_opt_.epsilon *= factor; bias_opt_.epsilon *= factor; }   // edge_with_weight.cc:90-93
  bool OfferFusedBiasGrad(BiasGradTarget* t) override;
  virtual bool BiasIsPerChannel2D() const { return !has_no_bias_; }       // one bias per output channel, 2-D layer
  // (a conv dgrad would only run the column-sum pass inside the library call, on the main stream; leaving it to the edge
  //  below puts it on the side lane instead — so only the pooling edges, whose kernels really fuse it, take the request)
  bool CanScaleDeriv() const override { return fuse_mask_; }               // (3-D ConvEdge: fuse_mask_ is off, CanFuseMask)
  // sigma and sigma' ride in the conv epilogues exactly where max(., 0) and the ReLU' mask do
  bool CanFuseLogistic() const override { return true; }

 protected:
  void StageForUp(Matrix& input);
  void StageForBprop(Matrix& deriv_output);
  void SumBiasRows(Matrix& deriv_output, float scale_targets, float scale);      // SumRows on the side lane
  SideLane* side_ = nullptr;
  void NoteUp();
  void NoteDown();
  void NoteOuter();
  Matrix weights_, grad_weights_, bias_, grad_bias_, hist_weights_, hist_bias_, state_weights_, state_bias_;
  bool has_no_bias_;
  float scale_gradients_;
  int num_grads_received_;
  OptimizerConfig weight_opt_, bias_opt_;
  long long weight_step_ = 0, bias_step_ = 0;             // the reference's per-optimizer step_ (optimizer.cc:199)
  int bf_up_ = -1, bf_down_ = -1, bf_outer_ = -1;        // -1 unknown, 0 tf32 / fp32 path, 1 bf16 path
  // the tensors of the last ComputeDown that took the bf16 path (layer-owned, stable): PrestageDown re-describes that call
  Matrix* down_out_ = nullptr;
  Matrix* down_in_ = nullptr;
  void RememberDown(Matrix& deriv_output, Matrix& deriv_input) {
    down_out_ = bf_down_ == 1 ? &deriv_output : nullptr;
    down_in_ = bf_down_ == 1 ? &deriv_input : nullptr;
  }
  bool bias_grad_fused_ = false;                         // this step's bias gradient comes from the edge above (ComputeOuter skips SumRows)
};

class ConvEdge : public EdgeWithWeight {
 public:
  explicit ConvEdge(const EdgeConfig& c);
  void SetImageSize(int y, int x, int t) override;
  size_t GetParameterMemoryRequirement() override;
  void SetMemory(Matrix& p) override;
  void SetGradMemory(Matrix& p) override;
  void ComputeUp(Matrix& input, Matrix& output, bool overwrite, bool train) override;
  void ComputeDown(Matrix& deriv_output, Matrix& input, Matrix& output, Matrix& deriv_input, bool overwrite) override;
  void PrestageDown() override;
  void ComputeOuter(Matrix& input, Matrix& deriv_output) override;
  double FlopsUp() const override;
  int FanIn() const override;
  ConvDesc GetConvDesc() const { return conv_desc_; }
  bool CanFuseReLU() const override { return !has_no_bias_ && shared_bias_ && image_size_t_ == 1; }
  bool CanFuseDropout() const override { return fuse_relu_ && CanFuseReLU(); }
  bool CanFuseMask() const override { return image_size_t_ == 1; }
  bool BiasIsPerChannel2D() const override { return !has_no_bias_ && shared_bias_ && image_size_t_ == 1; }

 private:
  ConvDesc conv_desc_;
  int partial_sum_y_, partial_sum_x_;
  bool shared_bias_;
};

// Locally connected ("untied") layer, src/local_edge.{h,cc}: a conv whose filter bank differs per output position.
// Parameters [Cout x (K*modules + modules)]: the banks of all modules (Shape4D (Cout, kx, ky, Cin*modules)), then one
// bias per output feature (column m + modules*o of the output).  2-D only (ConvNet refuses it on 3-D layers).
class LocalEdge : public EdgeWithWeight {
 public:
  explicit LocalEdge(const EdgeConfig& c) : EdgeWithWeight(c), conv_desc_(Edge::GetConvDesc(c)) {}
  void SetImageSize(int y, int x, int t) override;
  size_t GetParameterMemoryRequirement() override;
  void SetMemory(Matrix& p) override;
  void SetGradMemory(Matrix& p) override;
  void ComputeUp(Matrix& input, Matrix& output, bool overwrite, bool train) override;
  void ComputeDown(Matrix& deriv_output, Matrix& input, Matrix& output, Matrix& deriv_input, bool overwrite) override;
  void ComputeOuter(Matrix& input, Matrix& deriv_output) override;
  double FlopsUp() const override;
  // the reference's initialisation scale: weights_.GetCols() = K * modules (edge_with_weight.cc:126)
  int FanIn() const override { return KernelSize() * Modules(); }
  bool CanFuseReLU() const override { return !has_no_bias_; }                  // per-feature bias in the epilogue
  bool CanFuseDropout() const override { return fuse_relu_ && CanFuseReLU(); }
  bool CanFuseMask() const override { return true; }
  bool BiasIsPerChannel2D() const override { return false; }

 private:
  int KernelSize() const { return conv_desc_.kernel_size_y * conv_desc_.kernel_size_x * conv_desc_.num_input_channels; }
  int Modules() const { return num_modules_y_ * num_modules_x_; }
  ConvDesc conv_desc_;
};

class FCEdge : public EdgeWithWeight {          // weights [Cout x K] column-major, like a conv filter bank
 public:
  explicit FCEdge(const EdgeConfig& c) : EdgeWithWeight(c) {}
  void SetImageSize(int y, int x, int t) override;
  size_t GetParameterMemoryRequirement() override;
  void SetMemory(Matrix& p) override;
  void SetGradMemory(Matrix& p) override;
  void ComputeUp(Matrix& input, Matrix& output, bool overwrite, bool train) override;
  void ComputeDown(Matrix& deriv_output, Matrix& input, Matrix& output, Matrix& deriv_input, bool overwrite) override;
  void ComputeOuter(Matrix& input, Matrix& deriv_output) override;
  double FlopsUp() const override;
  int FanIn() const override { return num_inputs_; }
  bool CanFuseReLU() const override { return !has_no_bias_; }
  bool CanFuseDropout() const override { return fuse_relu_ && CanFuseReLU(); }
  bool CanFuseMask() const override { return true; }


 private:
  void View(Matrix& in, Matrix& out);
  int num_inputs_ = 0;
  ConvDesc desc_;
};

class ConvOneToOneEdge : public EdgeWithWeight {
 public:
  explicit ConvOneToOneEdge(const EdgeConfig& c) : EdgeWithWeight(c) {}
  void SetImageSize(int y, int x, int t) override;
  size_t GetParameterMemoryRequirement() override;
  void SetMemory(Matrix& p) override;
  void SetGradMemory(Matrix& p) override;
  void ComputeUp(Matrix& input, Matrix& output, bool overwrite, bool train) override;
  void ComputeDown(Matrix& deriv_output, Matrix& input, Matrix& output, Matrix& deriv_input, bool overwrite) override;
  void PrestageDown() override;
  void ComputeOuter(Matrix& input, Matrix& deriv_output) override;
  double FlopsUp() const override;
  int FanIn() const override { return num_input_channels_; }
  bool CanFuseReLU() const override { return !has_no_bias_; }
  bool CanFuseDropout() const override { return fuse_relu_ && CanFuseReLU(); }
  bool CanFuseMask() const override { return true; }

 private:
  ConvDesc desc_;
};

class MaxPoolEdge : public Edge {
 public:
  explicit MaxPoolEdge(const EdgeConfig& c) : Edge(c), conv_desc_(Edge::GetConvDesc(c)) {}
  void SetImageSize(int y, int x, int t) override;
  void ComputeUp(Matrix& input, Matrix& output, bool overwrite, bool train) override;
  void ComputeDown(Matrix& deriv_output, Matrix& input, Matrix& output, Matrix& deriv_input, bool overwrite) override;
  bool CanFuseMask() const override { return true; }
  bool CanProduceBiasGrad() const override { return image_size_t_ == 1; }

 protected:
  ConvDesc conv_desc_;
};

class AvgPoolEdge : public MaxPoolEdge {
 public:
  explicit AvgPoolEdge(const EdgeConfig& c) : MaxPoolEdge(c) {}
  void ComputeUp(Matrix& input, Matrix& output, bool overwrite, bool train) override;
  void ComputeDown(Matrix& deriv_output, Matrix& input, Matrix& output, Matrix& deriv_input, bool overwrite) override;
};

class ResponseNormEdge : public Edge {
 public:
  bool CanFuseReLU() const override { return image_size_t_ == 1; }      // max(., 0) rides in the rnorm kernel's store
  explicit ResponseNormEdge(const EdgeConfig& c)
      : Edge(c), num_filters_response_norm_(0), blocked_(c.response_norm_in_blocks), add_scale_(c.add_scale),
        pow_scale_(c.pow_scale), frac_of_filters_response_norm_(c.frac_of_filters_response_norm) {}
  void SetImageSize(int y, int x, int t) override;
  void ComputeUp(Matrix& input, Matrix& output, bool overwrite, bool train) override;
  void ComputeDown(Matrix& deriv_output, Matrix& input, Matrix& output, Matrix& deriv_input, bool overwrite) override;

 private:
  int num_filters_response_norm_;
  bool blocked_;
  float add_scale_, pow_scale_, frac_of_filters_response_norm_;
};

}  // namespace cnbhost
