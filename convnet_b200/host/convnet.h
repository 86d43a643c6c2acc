// convnet.h — the slice of the reference's ConvNet that sequences the hot path
// (src/convnet.{h,cc}: BuildNet :150, AllocateEdgeMemory :272-298, Fprop :377, Bprop :390,
// UpdateWeights :440-450, TrainOneBatch :475-485), its GradChecker (src/grad_check.cc) and the
// data-parallel gradient sync that replaces the reference's host-staged MPI
// Accumulate + Broadcast (src/convnet.cc:407-438) with in-place NCCL all-reduce over NVLink.
//
// Layers form a chain (every BASELINE net is one: Appendix B of SURVEY.md).  The model comes
// from a ModelConfig struct that model_file.cc reads from the reference's config::Model text proto:
// a net.pbtxt file, or the text of a built-in model, which models.cc holds by name.
#pragma once
#include <map>
#include <memory>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "data.h"
#include "edge.h"

namespace cnbhost {

enum Activation { LINEAR, RECTIFIED_LINEAR, SOFTMAX, LOGISTIC, SOFTMAX_DIST };
// proto/convnet_config.proto:34-44 LossFunction, same numbers (the CNB_LOSS_* codes of the kernels)
enum LossFunction {
  SQUARED_ERROR = 0, LINEAR_ERROR = 1, CROSS_ENTROPY_MULTINOMIAL = 2, CROSS_ENTROPY_BINARY = 3,
  CROSS_ENTROPY_MULTINOMIAL_DISTRIBUTED = 4, CLASSIFICATION_MULTINOMIAL = 5, CLASSIFICATION_BINARY = 6,
  HINGE_LINEAR = 7, HINGE_QUADRATIC = 8
};
// the kernel code of a fused or stand-alone activation (CNB_ACT_*): 0 for LINEAR and the softmaxes
inline int ActCode(Activation a) { return a == RECTIFIED_LINEAR ? CNB_ACT_RELU : (a == LOGISTIC ? CNB_ACT_LOGISTIC : CNB_ACT_LINEAR); }
// an output layer of this activation is trained on integer labels (SOFTMAX); every other one on a float target per feature
inline bool TakesLabels(Activation a) { return a == SOFTMAX; }
// a loss function or performance metric that reads labels (the others read per-feature targets)
inline bool ReadsLabels(int f) { return f == CROSS_ENTROPY_MULTINOMIAL || f == CLASSIFICATION_MULTINOMIAL; }

struct LayerConfig {
  std::string name;
  int num_channels = 0;
  bool is_input = false, is_output = false;
  Activation activation = LINEAR;
  // output layers (proto/convnet_config.proto:46-48)
  int loss_function = CROSS_ENTROPY_MULTINOMIAL;
  int performance_metric = CLASSIFICATION_MULTINOMIAL;
  float loss_function_weight = 1.f;
  int image_size_y = 0, image_size_x = 0, image_size_t = 1;   // input layer only
  float dropprob = 0.f;
  // batch normalisation between the incoming edge and the activation (proto/convnet_config.proto:56-61)
  bool batch_normalize = false;
  float bn_f = 0.98f;                      // running averages: mu = bn_f*mu + (1-bn_f)*batch mean (likewise sigma)
  float bn_epsilon = 1e-5f;                // sigma = sqrt(biased variance + bn_epsilon)
  OptimizerConfig gamma_optimizer, beta_optimizer;
};

// nullptr if `c` can train gamma or beta, else why not: OptimizerConfigError, or a norm rule (refused, DESIGN.md §5)
const char* BnOptimizerConfigError(const OptimizerConfig& c);
// Fine-tuning (EdgeConfig::block_backprop): an edge is frozen if it is blocked or lies below a blocked edge, so the frozen
// edges of a chain are [0, FrozenEdges).  They run their forward pass only: no weight gradient, no derivative into their
// source, no optimizer step.  The hidden layers they write receive no derivative (the output layer keeps the one its
// loss writes)
int FrozenEdges(const std::vector<EdgeConfig>& edges);

// What ConvNet's constructor throws for a model it cannot run.  what() names the layer or edge and says why; `edge` and
// `index` say which layer or edge of the chain holds what it objects to, and `fields` which of its fields, in order of
// preference (none: the layer or edge as a whole).  The model-file reader reports the refusal at that field's line
struct ModelRefused : std::invalid_argument {
  ModelRefused(const std::string& what, bool edge, size_t index, std::vector<std::string> fields)
      : std::invalid_argument(what), edge(edge), index(index), fields(std::move(fields)) {}
  bool edge;
  size_t index;
  std::vector<std::string> fields;
};

struct ModelConfig {
  std::string name;
  std::vector<LayerConfig> layer;
  std::vector<EdgeConfig> edge;
  unsigned seed = 42;
  // Polyak averaging (proto Model fields, same defaults): on when polyak_after and polyak_queue_size are both > 0; its
  // insertion rule (PolyakDue) also reads validate_after and save_after
  int polyak_after = 0, polyak_queue_size = 0, validate_after = -1, save_after = -1;
  // the rest of the training schedule ConvNet::Train runs (TrainSchedule; proto Model fields, same defaults).  ModelText
  // writes none of them, nor validate_after / save_after without Polyak: a checkpoint's __model__ carries no schedule
  int max_iter = -1, print_after = -1, reduce_lr_num_steps = 0, reduce_lr_max = 0;
  float reduce_lr_factor = 1.f, reduce_lr_threshold = 0.f;
  bool smaller_is_better = false;
  std::string reduce_lr_layer_name, checkpoint_dir;
  // train_dataset / valid_dataset: the batch order and, from the data stream of the input layer, its crop (gpu_image_size
  // 0: the whole image) and jitter
  struct Dataset {
    bool present = false;
    DatasetOrder order;
    int translate = 0, flip = 0, gpu_image_size_y = 0, gpu_image_size_x = 0;
  };
  Dataset train_dataset, valid_dataset;
};
inline bool PolyakOn(const ModelConfig& m) { return m.polyak_after > 0 && m.polyak_queue_size > 0; }
// checkpoint.cc: whether the reference's training loop inserts the parameters into the Polyak queue after TrainOneBatch call
// number `iteration` (src/convnet.cc:881-883, 965-967 with i + 1 = iteration; C++'s truncating %).  False with Polyak off
bool PolyakDue(const ModelConfig& m, long long iteration);

// train.cc: the reference's CheckReduceLearningRate (src/convnet.cc:788-818): false while `history` holds fewer than
// num_steps values; else the float running means of the first num_steps / 2 and of the other values among the last
// num_steps, and true when (smaller_is_better ? first - second : second - first) < threshold
bool ReduceLrDue(const std::vector<float>& history, int num_steps, float threshold, bool smaller_is_better);

// train.cc: the schedule of the reference's Train loop (src/convnet.cc:921-1006) without a net, so that a dry run and
// ConvNet::Train take their decisions from the same code.  Periods are C++'s truncating %: an action with period p runs
// after TrainOneBatch call `iteration` when iteration % p == 0, so p = -1 (the proto default of print_after and
// save_after) runs it after every call, and -p acts as p.  The constructor refuses (std::invalid_argument naming the
// field) what the reference divides by zero or exits on: print_after or save_after 0, and a reduce_lr_layer_name that
// is not the output layer's
class TrainSchedule {
 public:
  TrainSchedule(const ModelConfig& m, int lr_reduce_counter);
  enum Action { PRINT = 1, INSERT = 2, VALIDATE = 4, SAVE = 8 };
  // the actions after TrainOneBatch call `iteration` (i + 1 in the reference's loop), in the order they run;
  // VALIDATE only when there is a validation set
  int Actions(long long iteration, bool validation_set) const;
  bool FinalSave() const { return m_.max_iter % m_.save_after != 0; }       // :1003, after the last step
  // :978-994 for a new validation value: true when the learning rate is to be reduced now (the counters have moved)
  bool Validated(float value);
  int LrReduceCounter() const { return lr_reduce_counter_; }
  const ModelConfig& Model() const { return m_; }

 private:
  ModelConfig m_;
  std::vector<float> history_;
  int lr_reduce_counter_, dont_reduce_lr_ = 0;
};

// one line of ConvNet::Train's log: the training metric of a print (TRAIN) or a validation value (VALID)
struct TrainEvent {
  enum Kind { TRAIN, VALID };
  long long iteration;
  Kind kind;
  float value;
  bool lr_reduced = false;        // VALID: the learning rate was reduced after it
  bool polyak = false;            // VALID: measured on the Polyak average (false: on the current weights)
};

// checkpoint.cc: a checkpoint file (DESIGN.md §5 "Checkpoints"): an 8-byte magic, a u32 version, then records until EOF,
// each a u32 name length, the name, a u8 type, a u64 element count and the payload, little-endian.  The constructor reads
// the record headers and checks that every payload is there; std::invalid_argument names the file and what is wrong
class CheckpointFile {
 public:
  enum Type { FLOAT32 = 0, INT64 = 1, TEXT = 2 };
  explicit CheckpointFile(const std::string& path);
  const std::string& Path() const { return path_; }
  const std::vector<std::string>& Names() const { return names_; }        // in file order
  bool Has(const std::string& name) const { return records_.count(name) != 0; }
  // "" if record `name` exists with this type and element count (count < 0: any), else why not (the file, the record and
  // both sizes where they apply)
  std::string Check(const std::string& name, int type, long long count) const;
  std::vector<char> Read(const std::string& name) const;                   // the payload bytes (std::runtime_error: I/O)
 private:
  struct Record { int type; long long count, offset; };
  std::string path_;
  std::vector<std::string> names_;
  std::map<std::string, Record> records_;
};
// the weights a PRETRAINED edge `c` of `n` weights takes from its checkpoint (record <pretrained_edge_name>:weight)
std::vector<float> PretrainedWeights(const EdgeConfig& c, long long n);

// One trained tensor of a net, with its optimizer: an edge's weights or bias, or a batch-normalised layer's gamma or beta
// (ConvNet::PlanParameters, in flat-buffer order).  The bias of a has_no_bias edge keeps a record of zero floats, so that
// its optimizer can still be read and set; updates and checkpoints skip it.
struct TrainedTensor {
  enum Kind { WEIGHTS, BIAS, GAMMA, BETA };
  Kind kind;
  std::string name;        // the checkpoint record prefix: <edge>:weight, <edge>:bias, <layer>:gamma, <layer>:beta
  int edge;                // the edge whose bucket carries it (for gamma / beta: the edge that writes the layer; for a tie
                           // group's weights and bias: the group's lowest edge)
  size_t offset;           // into the flat parameter, gradient, history and adaptive state buffers
  long long n;             // floats
  int rows;                // norm groups: the output units of the weights; one for the others
  OptimizerConfig opt;     // the settings in force
  long long step = 0;      // updates counted so far, the reference's per-optimizer step_ (optimizer.cc:199)
  int owner = -1;          // weights / bias: the edge whose tensors they are and whose config gives their optimizer
  // ReduceLearningRate scales the edges' tensors only: gamma / beta keep their rate, as in the reference
  bool OnEdge() const { return kind == WEIGHTS || kind == BIAS; }
  // nullptr if `c` can train this tensor, else why not
  const char* ConfigError(const OptimizerConfig& c) const { return OnEdge() ? OptimizerConfigError(c) : BnOptimizerConfigError(c); }
};
// the optimizer block of `m` that configures `t`
OptimizerConfig& ModelOptimizer(ModelConfig& m, const TrainedTensor& t);

// one record of a net's checkpoint: a float32 tensor at `offset` of the parameters, the momentum history or the adaptive
// state, a layer's running statistic (RUNNING, at `running`), or (STEP) the step count of trained tensor `tensor`
struct CheckpointEntry {
  enum Buffer { PARAMS, HISTORY, STATE, RUNNING, STEP };
  std::string name;
  Buffer buffer;
  size_t offset;
  long long n;
  size_t tensor;
  float* running;
};

class Layer {                                   // src/layer.{h,cc}, reduced to state/deriv + activation
 public:
  explicit Layer(const LayerConfig& c) : config_(c), image_size_y_(0), image_size_x_(0), image_size_t_(1) {}
  void SetSize(int y, int x, int t) { image_size_y_ = y; image_size_x_ = x; image_size_t_ = t; }
  void AllocateMemory(int batch_size);
  void ApplyActivation(bool emit_bf16 = false);               // layer.cc:545-560
  void ApplyDerivativeOfActivation(bool emit_bf16 = false);   // layer.cc:562-580
  void ApplyDropout(bool train, unsigned long long step, unsigned long long salt, bool emit_bf16 = false);   // layer.cc:  mask = rand > dropprob ; state *= mask
  void ApplyDerivativeofDropout(bool emit_bf16 = false);        // unless ConvNet::DropoutFolds: the dgrad above scales instead
  bool HasDropout() const { return config_.dropprob > 0 && !config_.is_input; }
  float DropoutScale() const { return 1.0f / (1.0f - config_.dropprob); }
  float DropoutProb() const { return config_.dropprob; }
  unsigned long long DropoutSeed(unsigned long long step, unsigned long long salt) const;
  bool HasSeparateActivationPass() const { return ActCode(config_.activation) != CNB_ACT_LINEAR && !activation_fused_; }
  bool HasSeparateDerivPass() const { return ReceivesDeriv() && ActCode(config_.activation) != CNB_ACT_LINEAR && !deriv_fused_; }
  // output layer: deriv = loss_function_weight * dLoss/dstate and the per-image loss (unweighted), layer.cc:426-437
  void ComputeDeriv();
  void ComputePerformanceMetric();              // the per-image performance metric (GetPerformanceMetric, layer.cc:422)
  Matrix& GetState() { return state_; }
  Matrix& GetDeriv() { return deriv_; }
  int* GetLabels() { return labels_; }
  // the float targets of an output layer that does not take labels ([images x state columns]); empty otherwise
  Matrix& GetTargets() { return targets_; }
  float* GetLossPerImage() { return loss_per_image_.GetDevData(); }
  float* GetMetricPerImage() { return metric_per_image_.GetDevData(); }
  float LossWeight() const { return config_.loss_function_weight; }
  bool IsInput() const { return config_.is_input; }
  // back-propagation writes a derivative for this layer: not the input layer, nor the layer an RGBTOYUV edge writes (it
  // has no backward pass), nor a hidden layer a frozen edge writes (SetNoDeriv).  A layer without one has no derivative
  // buffer and runs no derivative pass
  bool ReceivesDeriv() const { return !config_.is_input && !no_deriv_; }
  void SetNoDeriv() { no_deriv_ = true; }
  bool IsOutput() const { return config_.is_output; }
  int GetNumChannels() const { return config_.num_channels; }
  int GetSizeY() const { return image_size_y_; }
  int GetSizeX() const { return image_size_x_; }
  int GetSizeT() const { return image_size_t_; }
  const std::string& GetName() const { return config_.name; }
  Activation GetActivation() const { return config_.activation; }
  void SetActivationFused(bool v) { activation_fused_ = v; }      // the incoming edge applies the ReLU in its epilogue
  void SetDerivFused(bool v) { deriv_fused_ = v; }                // the outgoing edge applies ReLU' in its epilogue
  ~Layer();

  // ---- batch normalisation (layer.cc:452-510).  The incoming edge writes the pre-normalisation input x into its own
  // buffer (GetPreBN); the forward pass (statistics, then gamma/beta and the activation) writes the state from it.  The
  // backward pass reads x, not the state: the state has been through the ReLU and the dropout.
  bool BatchNormalize() const { return config_.batch_normalize; }
  Matrix& GetPreBN() { return pre_bn_; }
  // gamma | beta: 2 * channels floats of the flat parameter and gradient buffers (ConvNet::PlanParameters)
  void SetBnMemory(Matrix& params, Matrix& grads);
  void InitializeBn();                                          // gamma = 1, beta = 0, mu = 0, sigma = 1 (layer.cc:271-278)
  void ApplyBatchNormalization(bool train, bool emit_bf16);     // activation included (its own pass is switched off)
  void ApplyDerivativeofBatchNormalization(bool emit_bf16);     // of the transform the last ApplyBatchNormalization applied
  // device vectors of `channels` floats: 0 running mean, 1 running sigma, 2 batch mean, 3 batch sigma
  float* BnStat(int which) { return bn_stats_.GetDevData() + (size_t)which * config_.num_channels; }
  long long BnPixels() const { return (long long)image_size_y_ * image_size_x_; }

 private:
  LayerConfig config_;
  int image_size_y_, image_size_x_, image_size_t_;
  Matrix state_, deriv_, loss_per_image_, metric_per_image_, targets_, dropout_mask_;
  Matrix pre_bn_, bn_stats_, gamma_, beta_, grad_gamma_, grad_beta_;
  bool bn_train_ = false;                       // the last ApplyBatchNormalization used the batch statistics
  int* labels_ = nullptr;
  bool activation_fused_ = false, deriv_fused_ = false;
  bool no_deriv_ = false;
};

// NCCL all-reduce of the flat gradient buffer, bucketed along edge boundaries and launched on a side
// stream as soon as the gradients of a bucket are final, so the exchange hides under back-propagation.
class DataParallelSync {
 public:
  DataParallelSync();
  ~DataParallelSync();
  static void GetUniqueId(char out[128]);                       // rank 0; bytes are broadcast by the launcher
  void Init(int rank, int world, const char id[128]);
  int world() const { return world_; }
  int rank() const { return rank_; }
  void Broadcast(float* buf, size_t count);                     // initial parameters from rank 0 (convnet.cc:300-309)
  // average buf[offset, offset+count) over ranks on `comm` (the caller orders `comm` after the producers of the gradients)
  void AllReduceAverageAsync(float* buf, size_t offset, size_t count, cudaStream_t comm);
  int reserved_sms() const { return nccl_ctas_; }               // SMs the collective's CTAs need while it is in flight
 private:
  void* comm_ = nullptr;
  cudaStream_t comm_stream_ = nullptr;                          // broadcast only; the all-reduces ride on ConvNet's side stream
  cudaEvent_t ready_ = nullptr, done_ = nullptr;
  int rank_ = 0, world_ = 1, nccl_ctas_ = 0;
};

// Gradient buckets: the unit of the overlapped all-reduce AND of the optimizer step.  Back-propagation finalises edge
// gradients from the LAST edge to the first, and edge slices are adjacent in the flat buffer (128-float padded), so a
// bucket is the contiguous range [lo, hi) — the edges [trigger, last] — that becomes final when edge `trigger` has run
// ComputeOuter.  Buckets are closed once they hold >= bucket_floats; the FIRST weighted edge of the net always gets a
// bucket of its own (its gradient is the last to appear: only that small exchange stays exposed at the end of the step);
// every parameter belongs to exactly one bucket.  (ConvNet passes frozen edges as empty: the buckets cover the trained
// edges only, and the first of them travels alone.)
struct Bucket { size_t lo, hi; int trigger, last; };
std::vector<Bucket> PlanBuckets(const std::vector<size_t>& edge_offset, const std::vector<size_t>& edge_size,
                                size_t bucket_floats);

class ConvNet {
 public:
  ConvNet(const ModelConfig& model, int batch_size);            // ModelRefused: a model this class cannot run
  virtual ~ConvNet();
  // the layout of the flat parameter buffer (host only): each edge's slice padded to 128 floats, followed by the
  // [gamma | beta] slice, also padded, of the layer the edge writes when that layer is batch-normalised; and the table of
  // trained tensors in that order, each with the optimizer the model gives it
  void PlanParameters();
  void AllocateMemory();                                        // convnet.cc:272-298: ONE flat parameter / gradient buffer
  virtual void Fprop(bool train);                               // convnet.cc:377-388
  virtual void Bprop();                                         // convnet.cc:390-405
  virtual void UpdateWeights();                                 // convnet.cc:440-450
  void ReduceLearningRate(float factor);                        // base epsilon of every weight and bias optimizer *= factor
  std::vector<TrainedTensor>& Tensors() { return tensors_; }
  // replace the settings of one trained tensor's optimizer; the step count and momentum history stay.  An adaptive
  // optimizer allocates the net's state buffer if it has none, and the tensor's state restarts (adagrad_delta or 1) when
  // optimizer_type or adagrad_delta changes.  The caller has validated `c` (TrainedTensor::ConfigError)
  void SetOptimizer(TrainedTensor& t, const OptimizerConfig& c);
  // the adaptive optimizer state: one float per parameter, laid out like the parameters; nullptr until some optimizer of
  // the net is ADAGRAD_SGD or RMSPROP_SGD
  float* AdaptiveState() { return state_.GetDevData(); }
  void ComputeDeriv();
  void TrainOneBatch(float* loss_out);                          // convnet.cc:475-485
  float GetLoss();                                              // loss_function_weight * the batch's loss (synchronises)
  float GetPerformanceMetric();                                 // sum of the per-image performance metric (synchronises)
  // the same sum into device float `dst`, on the main stream, without a host wait
  void SumPerformanceMetric(float* dst);

  // ---- the reference's Validate and Train (train.cc)
  // src/convnet.cc:571-589: Seek(0), then dataset_size / batch_size batches (the rest is dropped) of GetBatch, Fprop(false)
  // and the output layer's metric; the float running mean total = total * k / (k + 1) + e / (batch * (k + 1)).  One host
  // wait, at the end.  std::invalid_argument: the handler's batch size is not the net's
  float Validate(DataHandler& data);
  // src/convnet.cc:866-1006 from Iteration() to max_iter (TrainSchedule).  The run is named run_name ("" : <model
  // name>_<timestamp>); under checkpoint_dir ("" : the model's, and "." if it has none; created if missing) it writes
  // <run>.pbtxt, <run>_train.log, <run>_valid.log, <run>.ckpt and, with Polyak, <run>.ckptpolyak.  Validation with
  // Polyak on runs on LoadPolyakWeights() and training continues from the average, as in the reference; where the queue
  // is still empty (the reference divides by zero) it runs on the current weights, and the log says so.
  // std::invalid_argument: the schedule (TrainSchedule), a handler of another batch size, a data-parallel net
  std::vector<TrainEvent> Train(DataHandler& train, DataHandler* valid, const std::string& checkpoint_dir,
                                const std::string& run_name);
  // reductions of the learning rate the loop has applied to this net; a checkpoint keeps it (record
  // __lr_reduce_counter__, written when it is not 0), and Load restores it without applying them again
  int LrReduceCounter() const { return lr_reduce_counter_; }
  void SetDataParallel(DataParallelSync* dp, size_t bucket_floats);
  void SetBucketFloats(size_t bucket_floats);                   // re-plan the buckets (also used without data parallelism)
  void BroadcastParameters();
  void InvalidateStaging();                                     // after any write to the parameters from outside UpdateWeights

  // ---- checkpoints and Polyak averaging (checkpoint.cc; src/convnet.cc:659-751)
  // Save: waits for every stream, writes path + "temp", flushes and fsyncs it and renames it to `path`.  Load: reads and
  // validates the whole file before it changes anything (std::invalid_argument names the record; the net is then
  // unchanged), applies the file's optimizer blocks, copies every record, takes the file's seed and iteration, and leaves
  // the staged bf16 copies and dgrad banks coherent.  std::runtime_error: an I/O failure
  void Save(const std::string& path);
  void Load(const std::string& path);
  const ModelConfig& Model() const { return model_; }           // the model the net was built from (Load: its seed)
  ModelConfig CurrentModel() const;                             // the model with the optimizer settings now in force
  unsigned long long Iteration() const { return step_; }        // TrainOneBatch calls so far (the dropout step)
  // the keep-mask seed the next training Fprop gives layer i; 0 for a layer without dropout
  unsigned long long NextDropoutSeed(size_t i) const {
    return layers_[i]->HasDropout() ? layers_[i]->DropoutSeed(step_, dropout_salt_) : 0;
  }
  // Polyak queue on the device, allocated at the first insert: polyak_queue_size slots and a backup of the parameters.
  // std::invalid_argument: Polyak is off, nothing inserted, no backup; std::runtime_error: the allocation failed
  void InsertPolyak();                                          // parameters -> next slot (device copy, no host wait)
  void LoadPolyakWeights();                                     // backup <- parameters; parameters <- the average
  void LoadCurrentWeights();                                    // parameters <- backup
  int PolyakCount() const { return polyak_full_ ? model_.polyak_queue_size : polyak_index_; }

  Layer& InputLayer() { return *layers_.front(); }
  Layer& OutputLayer() { return *layers_.back(); }
  std::vector<std::unique_ptr<Edge>>& Edges() { return edges_; }
  std::vector<std::unique_ptr<Layer>>& Layers() { return layers_; }
  Matrix& Parameters() { return parameters_; }
  Matrix& GradParameters() { return grad_parameters_; }
  Matrix& History() { return history_; }
  size_t NumParameters() const { return num_params_; }
  int BatchSize() const { return batch_size_; }
  // the frozen edges are [0, NumFrozenEdges()) (FrozenEdges); their trained tensors are the prefix [0, TrainedOffset()) of
  // the flat buffers, which no optimizer step, bucket or Polyak average touches
  int NumFrozenEdges() const { return frozen_; }
  size_t TrainedOffset() const { return frozen_ < (int)edges_.size() ? edge_offset_[frozen_] : num_params_; }
  double FlopsFprop() const;
  // fprop + wgrad + dgrad of every edge, less the dgrad into the input layer, the wgrad of each frozen edge and the dgrad
  // into each layer a frozen edge writes
  double FlopsTrainStep() const;
  // per edge position: the slice of the flat buffer placed there (a tie group's slice sits at its lowest edge; the other
  // edges of the group have an empty one)
  const std::vector<size_t>& EdgeOffsets() const { return edge_offset_; }
  const std::vector<size_t>& EdgeSizes() const { return edge_size_; }
  // where the parameters edge `i` runs with begin (its owner's slice for a tied edge)
  size_t ParamOffset(size_t i) const { return edge_offset_[owner_[i] >= 0 ? home_[i] : (int)i]; }
  const std::vector<long long>& BnOffsets() const { return bn_offset_; }     // per layer: offset of [gamma | beta], -1 none
  float* DeviceLoss() { return loss_sum_.GetDevData(); }
  // One traced TrainOneBatch: device times (ms since the step began) of the pipeline's milestones, for the scaling report:
  // {fprop_end, bprop_compute_end, step_end, n_buckets, then per bucket {MB, exchange_begin, exchange_end, sgd_end}}.
  // exchange_* are -1 on one rank.  The events cost a few microseconds; the ordinary step records none of them.
  std::vector<float> TraceStep();

 protected:
  ModelConfig model_;
  int batch_size_;
  std::vector<std::unique_ptr<Layer>> layers_;
  std::vector<std::unique_ptr<Edge>> edges_;    // edges_[i]: layers_[i] -> layers_[i+1]
  void Refuse() const;                          // throws ModelRefused if this class cannot run the model
  // which passes of the neighbouring layers ride in each edge's kernels (Edge::FusionPlan), once the shapes are known;
  // also tells each layer whether its activation / derivative pass is left to do (Layer::SetActivationFused / SetDerivFused)
  void PlanFusion();
  // tie groups (EdgeConfig::tied_to), resolved once Refuse has accepted them: per edge, owner_ is the edge whose parameters
  // it runs with (itself when untied, -1 without parameters) and home_ the group's lowest edge, where the parameters sit in
  // the flat buffer.  Back-propagation reaches that edge last, so its bucket becomes final after every contribution to
  // the shared gradients and every read of the shared weights
  std::vector<int> owner_, home_;
  int frozen_ = 0;                              // FrozenEdges(model_.edge)
  void ResolveTies();
  bool Grouped(size_t i) const;                 // edge i shares its parameters with another edge
  bool prestage_ = true;                       // rebuild the dgrad banks behind each optimizer step (PrestageDown)
  // AllocateMemory has begun: the net may own staged bf16 copies and an SM reservation, which its destructor drops.  A
  // host-only net (no AllocateMemory) leaves the library's state to the nets that run
  bool allocated_ = false;
  Matrix parameters_, grad_parameters_, history_, loss_sum_, state_;
  std::vector<TrainedTensor> tensors_;
  void AllocateAdaptiveState();                 // state_, each tensor's slice initialised for its optimizer
  void InitState(const TrainedTensor& t);       // t's slice of state_ back to its optimizer's start
  std::vector<size_t> edge_offset_, edge_size_;
  std::vector<size_t> edge_span_;               // edge slice + the [gamma | beta] slice of its destination, both padded
  std::vector<long long> bn_offset_;
  size_t num_params_ = 0;
  // Side-stream pipeline of TrainOneBatch: as soon as a bucket's gradients are final its all-reduce (data parallel) is
  // enqueued on side_, and once the bucket's edges have finished their dgrad the multi-tensor SGD step of that bucket
  // follows on the same stream — the exchange and the update of the FC layers hide under the conv back-propagation.
  void IssueBucketUpdate(const Bucket& b);
  // the update of every trained tensor that edges [first, last] carry, in table order (AppendOptTensor: advances the step
  // counts); the weighted edges among them start counting gradients again
  void AppendUpdates(int first, int last, std::vector<CnbOptTensorEx>& out);
  // layers_[i] is a ReLU or logistic layer with dropout whose derivative is written by a dgrad that applies
  // act'(state) * 1/(1-p) itself: the backward pass needs no mask tensor, and the forward pass may fuse the dropout into
  // the edge below
  bool DropoutFolds(size_t i) const;
  void WaitSide();
  DataParallelSync* dp_ = nullptr;
  std::vector<Bucket> buckets_;
  // side_: bias-gradient passes; comm_: the NCCL all-reduces only; opt_: the per-bucket SGD steps.  Three streams so that a
  // long exchange (fc6: 302 MB) never delays the column sums, and an all-reduce (which waits for the side stream's bias
  // gradients) never queues behind the optimizer step of an earlier bucket
  cudaStream_t side_ = nullptr, comm_ = nullptr, opt_ = nullptr;
  cudaEvent_t ev_main_ = nullptr, ev_side_ = nullptr, ev_comm_ = nullptr, ev_opt_ = nullptr;
  std::vector<cudaEvent_t> ev_reduced_;         // per bucket: its all-reduce has finished (comm_ -> side_ / main)
  bool comm_pending_ = false;
  SideLane lane_;                               // what the edges see of the side stream (bias-gradient passes)
  bool eager_update_ = false, side_pending_ = false, opt_pending_ = false, updated_in_bprop_ = false;
  bool dropout_active_ = false;                 // the last Fprop applied dropout (train == true): states hold relu(x) * mask
  struct Trace {
    bool on = false;
    cudaEvent_t t0 = nullptr, fwd = nullptr, bwd = nullptr, end = nullptr;
    std::vector<cudaEvent_t> c0, c1, s1;        // per bucket: exchange begin / end (comm_), optimizer step end (side_)
  } trace_;
  unsigned long long step_ = 0;
  unsigned long long dropout_salt_ = 0xD1B54A32D192ED03ULL;      // model seed and data-parallel rank, see SetDataParallel
  bool salted_ = false;                                          // SetDataParallel has set dropout_salt_ (SaltDropout)
  void SaltDropout();
  // checkpoint.cc
  // in params order; opt[k]: the optimizer of tensors_[k] (which adaptive record it has)
  std::vector<CheckpointEntry> CheckpointEntries(const std::vector<OptimizerConfig>& opt);
  float* EntryData(const CheckpointEntry& e);
  void LoadPretrained(size_t edge);                             // a PRETRAINED edge's records, after AllocateAdaptiveState
  void WaitAllStreams();                                        // host waits for the main, side, comm and optimizer streams
  void PrestageAll();                                           // every prestaging edge rebuilds its dgrad banks (main stream)
  float* polyak_ = nullptr;                                     // polyak_queue_size slots, then the backup
  int polyak_index_ = 0;
  int lr_reduce_counter_ = 0;
  void SaveWithPolyak(const std::string& path);                 // train.cc: the reference's Save() (:659-667)
  bool polyak_full_ = false, polyak_backup_ = false;
};

// src/grad_check.{h,cc}: finite-difference check of dLoss/dparam for the first k weights and biases
// of every edge flagged grad_check, through the whole net.
struct GradCheckResult {
  std::string edge;
  float epsilon;
  float mean_scaled_diff_w, mean_scaled_diff_b;     // pass if < 0.01 (grad_check.cc:61)
};
class GradChecker : public ConvNet {
 public:
  GradChecker(const ModelConfig& model, int batch_size) : ConvNet(model, batch_size) {}
  std::vector<GradCheckResult> Run(unsigned seed);
 private:
  double LossAtD(Matrix& w, size_t index, float value);
};

// models.cc: a built-in name (its model text, read by ReadModelText), a path ending in ".pbtxt" (ReadModelFile), either
// with suffixes ("+bn", "+rmsprop", ...).  std::invalid_argument: unknown name, unreadable or refused file
ModelConfig BuildModel(const std::string& name);

// model_file.cc: the reference's config::Model text proto (src/util.cc ReadPbtxt, proto/convnet_config.proto).
// ReadModelFile applies the proto's defaults and presence rules, the default optimizers (src/convnet.cc:41-62) and the
// chain order of the graph; std::invalid_argument names the file, the line and the field of what it cannot read or run.
ModelConfig ReadModelFile(const std::string& path);
// the same for model text that `where` names in messages; check_pretrained = false skips opening the checkpoints of
// PRETRAINED edges (ConvNet::Load reading a checkpoint's own __model__)
ModelConfig ReadModelText(const std::string& text, const std::string& where, bool check_pretrained);
// `m` as a config::Model text proto that ReadModelFile reads back to the same model: every field the host reads for a
// layer or edge of that kind explicit, floats printed so that they read back bit-exactly
std::string ModelText(const ModelConfig& m);

}  // namespace cnbhost
