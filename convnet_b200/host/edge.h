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
//   UpSampleEdge        src/upsample_edge.{h,cc}        UpSampleGemm ; dgrad: the block sum (DESIGN.md §5)
//   DownSampleEdge      src/downsample_edge.{h,cc}      DownSampleGemm ; dgrad: AvgPoolUndoGemm
//   RgbToYuvEdge        src/rgbtoyuv_edge.{h,cc}        RGBToYUV ; no backward pass (input layer only)
// FC and 1x1 edges run on the same implicit-GEMM conv kernels (a 1x1 convolution IS that GEMM),
// SURVEY.md §8(f) rank 1.  The protobuf `config::Edge` is replaced by the plain EdgeConfig struct
// (protobuf is not in the image); field names follow proto/convnet_config.proto:120-221.
#pragma once
#include <string>
#include <vector>

#include "matrix.h"

namespace cnbhost {

class Layer;

enum EdgeType { FC, CONVOLUTIONAL, MAXPOOL, AVGPOOL, RESPONSE_NORM, CONV_ONETOONE, LOCAL, UPSAMPLE, DOWNSAMPLE, RGBTOYUV };
// the proto value name of each EdgeType (model files, messages)
extern const char* const kEdgeTypeNames[RGBTOYUV + 1];

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

// proto/convnet_config.proto:142-150 Initialization, same numbers.  SPARSE_GAUSSIAN is not implemented (a model file that
// asks for it is refused); PRETRAINED reads the edge from a checkpoint file (ConvNet::AllocateMemory, checkpoint.cc)
enum Initialization {
  DENSE_GAUSSIAN = 0, SPARSE_GAUSSIAN = 1, CONSTANT = 2, DENSE_GAUSSIAN_SQRT_FAN_IN = 3, PRETRAINED = 4, DENSE_UNIFORM = 5,
  DENSE_UNIFORM_SQRT_FAN_IN = 6
};

struct EdgeConfig {
  std::string name, source, dest;
  EdgeType edge_type = FC;
  int kernel_size = 1, stride = 1, padding = 0;
  // kUnset: take kernel_size / stride / padding (Edge::GetConvDesc); any other value is used as given, as the reference
  // does for a field that is present (an explicit kernel_size_y: 0 on a pooling edge pools globally in y)
  static constexpr int kUnset = -2147483647 - 1;
  int kernel_size_y = kUnset, kernel_size_x = kUnset, stride_y = kUnset, stride_x = kUnset, padding_y = kUnset,
      padding_x = kUnset;
  int kernel_size_t = 1, stride_t = 1, padding_t = 0;
  bool shared_bias = true, has_no_bias = false;
  float add_scale = 0.0005f, pow_scale = 0.75f, frac_of_filters_response_norm = 0.25f;
  bool response_norm_in_blocks = false;
  float scale_gradients = 1.f;
  int sample_factor = 1;                     // UPSAMPLE / DOWNSAMPLE: the factor per spatial axis
  // EdgeWithWeight::Initialize (edge_with_weight.cc:108-143).  The model reader applies the proto's defaults
  // (DENSE_GAUSSIAN_SQRT_FAN_IN, init_wt 1, init_bias 0) to model files and built-in models alike; the built-in texts ask
  // for DENSE_UNIFORM_SQRT_FAN_IN
  int initialization = DENSE_UNIFORM_SQRT_FAN_IN;
  float init_wt = 1.f;
  float init_bias = 0.f;
  // PRETRAINED: the checkpoint file, used as given, and the edge whose records it takes ("" = this edge's source:dest,
  // edge_with_weight.cc:18-19)
  std::string pretrained_model, pretrained_edge_name;
  OptimizerConfig weight_optimizer, bias_optimizer;
  bool grad_check = false;
  int grad_check_num_params = 10;
  std::vector<float> grad_check_epsilon;
  // the name of the edge whose weights and bias this edge runs with and trains ("" = its own; src/edge.cc:131-180).  A tied
  // edge has no parameters of its own: its optimizers, initialisation and pretrained_* fields are not used (TieError)
  std::string tied_to;
  // no derivative passes through this edge (proto field 13): it and every edge below it are frozen (FrozenEdges)
  bool block_backprop = false;
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
  virtual void SetMemory(Matrix& p) {}
  virtual void SetGradMemory(Matrix& p) {}
  virtual size_t GetParameterMemoryRequirement() { return 0; }
  virtual void Initialize(unsigned seed) {}
  virtual bool HasNoParameters() const { return true; }
  virtual void SetImageSize(int image_size_y, int image_size_x, int image_size_t);
  virtual double FlopsUp() const { return 0; }                           // 2*MACs per batch (BASELINE.md §2c)

  int GetNumModulesY() const { return num_modules_y_; }
  int GetNumModulesX() const { return num_modules_x_; }
  int GetNumModulesT() const { return num_modules_t_; }
  int GetImageSizeY() const { return image_size_y_; }
  int GetImageSizeX() const { return image_size_x_; }
  int GetImageSizeT() const { return image_size_t_; }
  void SetInputChannels(int a) { num_input_channels_ = a; }
  void SetOutputChannels(int a) { num_output_channels_ = a; }
  int GetNumOutputChannels() const { return num_output_channels_; }
  const std::string& GetName() const { return name_; }
  const EdgeConfig& Config() const { return config_; }
  bool IsBackPropBlocked() const { return config_.block_backprop; }
  Layer* GetSource() { return source_; }
  Layer* GetDest() { return dest_; }
  void SetSource(Layer* l) { source_ = l; }
  void SetDest(Layer* l) { dest_ = l; }
  void SetBatchSize(int n) { batch_size_ = n; }

  // Epilogue fusion: passes of the neighbouring layers that ride in this edge's kernels (SURVEY.md 8(f) rank 2).
  // What the kernels of this edge can absorb, once SetImageSize has fixed its shapes:
  struct Absorbs {
    bool act_up = false;           // ComputeUp: the destination's ReLU (after the bias, where there is one)
    bool act_down = false;         // ComputeDown: the source's ReLU' mask
    bool logistic = false;         // sigma / sigma' too, wherever the two above hold
    bool dropout = false;          // behind a fused activation: the destination's dropout (ComputeUp), the source's
                                   // dropout derivative as a scale (ComputeDown)
    bool sums_bias_below = false;  // ComputeDown can sum the channels of the derivative it writes
    bool per_channel_bias = false; // the bias gradient is that channel sum of this edge's output derivative
  };
  virtual Absorbs CanAbsorb() const { return Absorbs(); }
  // What ConvNet::PlanFusion decided for this edge, fixed for the life of the net
  struct FusionPlan {
    int up_act = CNB_ACT_LINEAR;    // CNB_ACT_* that ComputeUp applies in its epilogue
    int down_act = CNB_ACT_LINEAR;  // CNB_ACT_* whose derivative ComputeDown applies
    bool dropout_up = false;        // the destination's dropout may ride in ComputeUp (UpRequest)
    bool scale_down = false;        // the source's dropout derivative may fold into ComputeDown (DownRequest::scale)
    bool sums_bias_below = false;   // ComputeDown may take the bias gradient of the edge below (DownRequest::bias_grad)
    bool offers_bias_grad = false;  // the edge above may sum this edge's bias gradient
  };
  void SetFusionPlan(const FusionPlan& p) { plan_ = p; }
  const FusionPlan& Plan() const { return plan_; }
  // One-shot requests ConvNet makes before each ComputeUp / ComputeDown; the call consumes them.
  // emit (bf16 mode): the call writes the tensor LAST and the next conv edge multiplies it in bf16, so the kernel leaves
  // the bf16 copy too (convnet_b200_emit_bf16_next) instead of that edge running a conversion pass.
  // Dropout (scale != 0): convnet_b200_fuse_next_dropout, no mask tensor (only where ConvNet::DropoutFolds).
  // scale: the dropout derivative of the source layer folded into the dgrad (convnet_b200_fuse_next_scale).
  // bias_grad: the edge below's bias gradient, summed while the derivative is stored (convnet_b200_fuse_next_bias_grad).
  struct UpRequest { bool emit = false; float drop_prob = 0.f, drop_scale = 0.f; unsigned long long drop_seed = 0; };
  struct BiasGradTarget { float* grad_bias = nullptr; float st = 0.f, so = 1.f; };
  struct DownRequest { bool emit = false; float scale = 1.f; BiasGradTarget bias_grad; };
  void Request(const UpRequest& r) { up_req_ = r; }
  void Request(const DownRequest& r) { down_req_ = r; }
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
  // SetImageSize of an edge with a conv descriptor: its channels, then its output size (src/edge.cc:108-114)
  void SetImageSize(int y, int x, int t, ConvDesc& d);
  FusionPlan plan_;
  UpRequest up_req_;
  DownRequest down_req_;
  // right before the ComputeUp / ComputeDown kernel: the plan's fused activation and the pending request as ABI calls.
  // `emit`: this kernel is the one that writes the output last
  void ArmUp(const float* bias, bool emit);
  void ArmDown(const float* act_state);
};

// The side stream of ConvNet::TrainOneBatch (all-reduce + optimizer, see convnet.h): bias-gradient column sums are
// memory-bound passes over a derivative that is already final, so they run there, beside the tensor-bound wgrad / dgrad
// kernels of the main stream.  ConvNet::AllocateMemory gives every weighted edge the lane together with its gradient memory.
struct SideLane { cudaStream_t stream = nullptr; cudaEvent_t ready = nullptr; bool used = false; };

// The call sequence of every edge with weights: ComputeUp / ComputeDown / ComputeOuter stage the bf16 operands, arm the
// requests, run the edge type's GEMM, note the path it took and add the bias (or sum its gradient).  A subclass supplies
// its three GEMM calls, its parameter sizes and whether it prestages dgrad banks.
class EdgeWithWeight : public Edge {
 public:
  void SetSideLane(SideLane* s) { side_ = s; }
  // after this edge's optimizer step, on the optimizer's stream: rebuild what the next ComputeDown derives from the
  // weights alone (convnet_b200_prestage_next), off the next step's critical path (edges where PrestagesDown holds)
  void PrestageDown();
  explicit EdgeWithWeight(const EdgeConfig& c)
      : Edge(c), has_no_bias_(c.has_no_bias), scale_gradients_(c.scale_gradients), num_grads_received_(0) {}
  bool HasNoParameters() const override { return false; }
  void ComputeUp(Matrix& input, Matrix& output, bool overwrite, bool train) override;
  void ComputeDown(Matrix& deriv_output, Matrix& input, Matrix& output, Matrix& deriv_input, bool overwrite) override;
  void ComputeOuter(Matrix& input, Matrix& deriv_output) override;
  // parameters [Cout x (WeightCols + BiasCols)]: the weights (Shape4D WeightShape), then the bias columns; the gradient
  // is carved the same way
  size_t GetParameterMemoryRequirement() override;
  // tied edges (EdgeConfig::tied_to): ConvNet hands this edge the owner's parameter and gradient slices, and the group
  // shares the owner's gradient counter, so the first contribution of a step overwrites and the others accumulate
  // (edge_with_weight.cc:150-188)
  bool Tied() const { return !config_.tied_to.empty(); }
  void TieTo(EdgeWithWeight* owner) { owner_ = owner; owner->group_.push_back(this); }
  Shape4D GetWeightShape() const { return WeightShape(); }
  int GetBiasCols() const { return has_no_bias_ ? 0 : BiasCols(); }
  void SetMemory(Matrix& p) override { Carve(p, weights_, bias_); }
  void SetGradMemory(Matrix& p) override { Carve(p, grad_weights_, grad_bias_); }
  void Initialize(unsigned seed) override;
  // the initial weights Initialize(seed) writes (host only: valid once SetImageSize has fixed the shapes); the bias
  // starts at init_bias
  std::vector<float> InitialWeights(unsigned seed) const;
  Matrix& GetWeight() { return weights_; }
  Matrix& GetGradWeight() { return grad_weights_; }
  Matrix& GetBias() { return bias_; }
  Matrix& GetGradBias() { return grad_bias_; }
  int GetNumGradsReceived() const { return owner_->num_grads_received_; }
  void IncrementNumGradsReceived() { owner_->num_grads_received_++; }
  void NotifyStart() { owner_->num_grads_received_ = 0; }     // the optimizer has taken this step's gradients
  // bf16 mode (convnet_b200_set_conv_precision(2)): each tensor this edge feeds to two conv calls of a step has ONE bf16
  // copy — the input (fprop + wgrad), the output derivative (wgrad + dgrad) and the weights (fprop + dgrad).  The copy is
  // normally written by the kernel that produced the tensor (the emit requests of the neighbouring edges, the dropout
  // and SGD kernels); convnet_b200_bf16_ensure converts only when no valid copy exists.  Which calls really run in bf16 is
  // learnt from convnet_b200_last_conv_path() during the first step (FC-shaped calls stay on tf32 and are not staged).
  bool WantsBf16Input() const override { return bf_up_ == 1 || bf_outer_ == 1; }
  bool WantsBf16Deriv() const override { return bf_outer_ == 1 || bf_down_ == 1; }
  // floats of the weights and of the bias (0 under has_no_bias) in the edge's parameter slice, weights first
  long long WeightCount() const { return (long long)num_output_channels_ * WeightCols(); }
  long long BiasCount() const { return has_no_bias_ ? 0 : (long long)num_output_channels_ * BiasCols(); }
  // the target of this step's bias gradient for the edge above (Plan().offers_bias_grad): ComputeOuter then skips its sum
  BiasGradTarget HandOffBiasGrad();
  // sigma and sigma' ride in the conv epilogues exactly where max(., 0) and the ReLU' mask do; so does the dropout.
  // (A conv dgrad would only run the bias-gradient column sum inside the library call, on the main stream; leaving it to
  // the edge below puts it on the side lane instead — so only the pooling edges, whose kernels really fuse it, take it.)
  Absorbs CanAbsorb() const override {
    Absorbs a;
    a.act_up = a.per_channel_bias = !has_no_bias_;
    a.act_down = a.logistic = a.dropout = true;
    return a;
  }

 protected:
  virtual void GemmUp(Matrix& input, Matrix& output, float scale_targets) = 0;
  virtual void GemmDown(Matrix& deriv_output, Matrix& deriv_input, float scale_targets) = 0;
  virtual void GemmOuter(Matrix& input, Matrix& deriv_output, float scale_targets, float scale) = 0;
  virtual int WeightCols() const = 0;      // per output channel; also the fan-in of the initialisation (edge_with_weight.cc:126)
  virtual int BiasCols() const { return 1; }
  virtual Shape4D WeightShape() const = 0;
  virtual bool PrestagesDown() const { return false; }
  void Carve(Matrix& p, Matrix& w, Matrix& b);
  // bias_ (1 x B) added to every B columns of the output, reshaped to [rows x B] (cnb_add_channel_bias); its gradient the
  // column sum of the output derivative in that shape, on the side lane
  virtual void AddBias(Matrix& output, bool emit);
  virtual void SumBias(Matrix& deriv_output, float scale_targets, float scale);
  void StageForUp(Matrix& input);
  void StageForBprop(Matrix& deriv_output);
  SideLane* side_ = nullptr;
  void NoteUp();
  void NoteDown();
  void NoteOuter();
  Matrix weights_, grad_weights_, bias_, grad_bias_;
  bool has_no_bias_;
  float scale_gradients_;
  int num_grads_received_;
  EdgeWithWeight* owner_ = this;                         // whose parameters and gradient counter this edge uses
  std::vector<EdgeWithWeight*> group_{this};             // the owner's: every edge that uses its parameters, itself first
  int bf_up_ = -1, bf_down_ = -1, bf_outer_ = -1;        // -1 unknown, 0 tf32 / fp32 path, 1 bf16 path
  // the tensors of the last ComputeDown that took the bf16 path (layer-owned, stable): PrestageDown re-describes that call
  Matrix* down_out_ = nullptr;
  Matrix* down_in_ = nullptr;
  bool bias_grad_fused_ = false;                         // this step's bias gradient comes from the edge above (ComputeOuter skips SumRows)
};

class ConvEdge : public EdgeWithWeight {
 public:
  explicit ConvEdge(const EdgeConfig& c);
  void SetImageSize(int y, int x, int t) override;
  double FlopsUp() const override;
  ConvDesc GetConvDesc() const { return conv_desc_; }
  Absorbs CanAbsorb() const override {                   // the 3-D kernels fuse nothing; only a shared bias rides along
    Absorbs a = EdgeWithWeight::CanAbsorb();
    a.act_up = a.per_channel_bias = !has_no_bias_ && shared_bias_ && image_size_t_ == 1;
    a.act_down = image_size_t_ == 1;
    return a;
  }

 protected:
  void GemmUp(Matrix& input, Matrix& output, float scale_targets) override;
  void GemmDown(Matrix& deriv_output, Matrix& deriv_input, float scale_targets) override;
  void GemmOuter(Matrix& input, Matrix& deriv_output, float scale_targets, float scale) override;
  int WeightCols() const override;
  int BiasCols() const override { return shared_bias_ ? 1 : num_modules_y_ * num_modules_x_ * num_modules_t_; }
  Shape4D WeightShape() const override;
  bool PrestagesDown() const override { return image_size_t_ == 1; }
  void AddBias(Matrix& output, bool emit) override;
  void SumBias(Matrix& deriv_output, float scale_targets, float scale) override;

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
  double FlopsUp() const override;
  Absorbs CanAbsorb() const override {                   // the bias is per output feature, not per channel
    Absorbs a = EdgeWithWeight::CanAbsorb();
    a.per_channel_bias = false;
    return a;
  }

 protected:
  void GemmUp(Matrix& input, Matrix& output, float scale_targets) override;
  void GemmDown(Matrix& deriv_output, Matrix& deriv_input, float scale_targets) override;
  void GemmOuter(Matrix& input, Matrix& deriv_output, float scale_targets, float scale) override;
  // the reference's initialisation scale: weights_.GetCols() = K * modules (edge_with_weight.cc:126)
  int WeightCols() const override { return KernelSize() * Modules(); }
  int BiasCols() const override { return Modules(); }
  Shape4D WeightShape() const override;

 private:
  int KernelSize() const { return conv_desc_.kernel_size_y * conv_desc_.kernel_size_x * conv_desc_.num_input_channels; }
  int Modules() const { return num_modules_y_ * num_modules_x_; }
  ConvDesc conv_desc_;
};

class FCEdge : public EdgeWithWeight {          // weights [Cout x K] column-major, like a conv filter bank
 public:
  explicit FCEdge(const EdgeConfig& c) : EdgeWithWeight(c) {}
  void SetImageSize(int y, int x, int t) override;
  double FlopsUp() const override;

 protected:
  void GemmUp(Matrix& input, Matrix& output, float scale_targets) override;
  void GemmDown(Matrix& deriv_output, Matrix& deriv_input, float scale_targets) override;
  void GemmOuter(Matrix& input, Matrix& deriv_output, float scale_targets, float scale) override;
  int WeightCols() const override { return num_inputs_; }
  Shape4D WeightShape() const override { return Shape4D{{num_output_channels_, 1, 1, num_inputs_}}; }

 private:
  int num_inputs_ = 0;
  ConvDesc desc_;
};

class ConvOneToOneEdge : public EdgeWithWeight {
 public:
  explicit ConvOneToOneEdge(const EdgeConfig& c) : EdgeWithWeight(c) {}
  void SetImageSize(int y, int x, int t) override;
  double FlopsUp() const override;

 protected:
  void GemmUp(Matrix& input, Matrix& output, float scale_targets) override;
  void GemmDown(Matrix& deriv_output, Matrix& deriv_input, float scale_targets) override;
  void GemmOuter(Matrix& input, Matrix& deriv_output, float scale_targets, float scale) override;
  int WeightCols() const override { return num_input_channels_; }
  Shape4D WeightShape() const override { return Shape4D{{num_output_channels_, 1, 1, num_input_channels_}}; }
  bool PrestagesDown() const override { return true; }

 private:
  ConvDesc desc_;
};

class MaxPoolEdge : public Edge {
 public:
  explicit MaxPoolEdge(const EdgeConfig& c) : Edge(c), conv_desc_(Edge::GetConvDesc(c)) {}
  void SetImageSize(int y, int x, int t) override;
  void ComputeUp(Matrix& input, Matrix& output, bool overwrite, bool train) override;
  void ComputeDown(Matrix& deriv_output, Matrix& input, Matrix& output, Matrix& deriv_input, bool overwrite) override;
  Absorbs CanAbsorb() const override {
    Absorbs a;
    a.act_down = true;
    a.sums_bias_below = image_size_t_ == 1;
    return a;
  }

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
  Absorbs CanAbsorb() const override {                  // max(., 0) rides in the rnorm kernel's store
    Absorbs a;
    a.act_up = image_size_t_ == 1;
    return a;
  }
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

// UPSAMPLE and DOWNSAMPLE: every pixel replicated into an f x f block, and the mean of each f x f block.  Channels and
// frames are kept; on a 3-D layer the frames are folded into the Shape4D planes (C * T), so the 2-D calls apply as they
// are.  The derivatives are the true ones (DESIGN.md §5): the block sum (AvgPoolGemm with scaleOutput f^2) and the mean's
// derivative d / f^2 (AvgPoolUndoGemm) — the reference's calls are f^2 too small and f^2 too large.
class SampleEdge : public Edge {
 public:
  explicit SampleEdge(const EdgeConfig& c) : Edge(c), factor_(c.sample_factor) {}
  int Factor() const { return factor_; }
  Absorbs CanAbsorb() const override {                   // ReLU / ReLU' in the kernels, sigma / sigma' as passes in the call
    Absorbs a;
    a.act_up = a.act_down = a.dropout = true;
    a.sums_bias_below = image_size_t_ == 1;
    return a;
  }

 protected:
  int factor_;
  ConvDesc Desc() const;                                  // the f x f window with stride f over the C * T planes
};
class UpSampleEdge : public SampleEdge {
 public:
  explicit UpSampleEdge(const EdgeConfig& c) : SampleEdge(c) {}
  void SetImageSize(int y, int x, int t) override;
  void ComputeUp(Matrix& input, Matrix& output, bool overwrite, bool train) override;
  void ComputeDown(Matrix& deriv_output, Matrix& input, Matrix& output, Matrix& deriv_input, bool overwrite) override;
};
class DownSampleEdge : public SampleEdge {
 public:
  explicit DownSampleEdge(const EdgeConfig& c) : SampleEdge(c) {}
  void SetImageSize(int y, int x, int t) override;
  void ComputeUp(Matrix& input, Matrix& output, bool overwrite, bool train) override;
  void ComputeDown(Matrix& deriv_output, Matrix& input, Matrix& output, Matrix& deriv_input, bool overwrite) override;
};
// RGB -> YUV of the input layer (3 -> 3 channels, 2-D).  The reference has no backward pass for it, so its destination
// layer receives no derivative (ConvNet: Layer::ReceivesDeriv) and ComputeDown is never called
class RgbToYuvEdge : public Edge {
 public:
  explicit RgbToYuvEdge(const EdgeConfig& c) : Edge(c) {}
  void ComputeUp(Matrix& input, Matrix& output, bool overwrite, bool train) override;
  void ComputeDown(Matrix& deriv_output, Matrix& input, Matrix& output, Matrix& deriv_input, bool overwrite) override;
};

}  // namespace cnbhost
