// convnet.cc — see convnet.h.
#include "convnet.h"

#include <dlfcn.h>
#include <nccl.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <stdexcept>

#ifndef DIVUP
#define DIVUP(x, y) (((x) + (y)-1) / (y))
#endif

namespace cnbhost {

// =================================================================== Layer
Layer::~Layer() { if (labels_) cudaFree(labels_); }

const char* BnOptimizerConfigError(const OptimizerConfig& c) {
  if (const char* err = OptimizerConfigError(c)) return err;
  if (c.weight_norm_limit > 0 || c.weight_norm_constraint > 0)
    return "weight_norm_limit / weight_norm_constraint are not supported on gamma / beta";
  return nullptr;
}

void Layer::AllocateMemory(int batch_size) {               // layer.cc:228-262 (Shape4D convention :257-258)
  const int cols = image_size_y_ * image_size_x_ * image_size_t_ * config_.num_channels;
  state_.AllocateGPUMemory(batch_size, cols);
  state_.SetShape4D(batch_size, image_size_x_, image_size_y_, config_.num_channels * image_size_t_);
  if (ReceivesDeriv()) {
    deriv_.AllocateGPUMemory(batch_size, cols);
    deriv_.SetShape4D(batch_size, image_size_x_, image_size_y_, config_.num_channels * image_size_t_);
  }
  if (config_.dropprob > 0) dropout_mask_.AllocateGPUMemory(batch_size, cols);
  if (config_.batch_normalize) {
    pre_bn_.AllocateGPUMemory(batch_size, cols);
    pre_bn_.SetShape4D_like(state_);
    bn_stats_.AllocateGPUMemory(1, 4 * config_.num_channels);
  }
  if (config_.is_output) {
    CUDA_CHECK(cudaMalloc((void**)&labels_, sizeof(int) * batch_size));
    CUDA_CHECK(cudaMemset(labels_, 0, sizeof(int) * batch_size));
    loss_per_image_.AllocateGPUMemory(batch_size, 1);
    metric_per_image_.AllocateGPUMemory(batch_size, 1);
    if (!TakesLabels(config_.activation)) {                // layer.cc:530-602: data_ shaped like the state
      targets_.AllocateGPUMemory(batch_size, cols);
      targets_.Set(0);
    }
  }
}

int FrozenEdges(const std::vector<EdgeConfig>& edges) {
  int n = 0;
  for (size_t i = 0; i < edges.size(); i++)
    if (edges[i].block_backprop) n = (int)i + 1;
  return n;
}

// ---- the checks of ConvNet::Refuse.  Each returns why it refuses (empty: it does not) and the fields it objects to, in
// order of preference (ModelRefused::fields)
namespace {
struct Objection {
  std::string why;
  std::vector<std::string> fields;
};

// edge `e`, once SetImageSize has run, between layers of `source_channels` and `dest_channels`: it gives its destination at
// least one module in y, x and t, a pooling or response-norm edge keeps the channel count, and a convolution has no
// temporal padding (the 3-D kernels fold the frames into channels).  The edge as a whole
Objection EdgeShapeError(const Edge& e, int source_channels, int dest_channels) {
  const int my = e.GetNumModulesY(), mx = e.GetNumModulesX(), mt = e.GetNumModulesT();
  if (my < 1 || mx < 1 || mt < 1)
    return {"its kernel, stride and padding leave no output (" + std::to_string(my) + " x " + std::to_string(mx) + " x " +
            std::to_string(mt) + " modules in y, x, t)"};
  const EdgeType t = e.Config().edge_type;
  if ((t == MAXPOOL || t == AVGPOOL || t == RESPONSE_NORM) && source_channels != dest_channels)
    return {"pooling and response normalisation keep the channel count, but the source layer has " +
            std::to_string(source_channels) + " channels and the destination " + std::to_string(dest_channels)};
  if ((t == CONVOLUTIONAL || t == LOCAL) && e.Config().padding_t != 0)
    return {"padding_t " + std::to_string(e.Config().padding_t) + " is not supported on a convolution (the 3-D kernels "
            "fold the frames into channels)"};
  return {};
}

// an UPSAMPLE, DOWNSAMPLE or RGBTOYUV edge `e` (SetImageSize has run) between layers of `source_channels` and
// `dest_channels`, its source being the input layer when `on_input` and its destination the output layer when
// `into_output`.  A factor is at least 1, the three keep the channel count, a DOWNSAMPLE's image size is divisible by its
// factor, and RGBTOYUV maps the 3 channels of a 2-D input layer to a hidden layer (the layer it writes receives no
// derivative, and an output layer needs one for its loss).  sample_factor or edge_type
Objection SampleEdgeError(const Edge& e, int source_channels, int dest_channels, bool on_input, bool into_output) {
  const EdgeType t = e.Config().edge_type;
  if (t != UPSAMPLE && t != DOWNSAMPLE && t != RGBTOYUV) return {};
  auto refuse = [](const std::string& field, const std::string& why) {
    return Objection{"field '" + field + "': " + why, {field}};
  };
  const std::string name = kEdgeTypeNames[t], f = std::to_string(e.Config().sample_factor);
  if (t != RGBTOYUV && e.Config().sample_factor < 1) return refuse("sample_factor", f + " is below 1");
  if (source_channels != dest_channels)
    return refuse("edge_type", name + " keeps the channel count, but the source layer has " + std::to_string(source_channels) +
                  " channels and the destination " + std::to_string(dest_channels));
  const int y = e.GetImageSizeY(), x = e.GetImageSizeX();
  if (t == DOWNSAMPLE && (y % e.Config().sample_factor || x % e.Config().sample_factor))
    return refuse("sample_factor", "DOWNSAMPLE by " + f + " needs image sizes divisible by " + f +
                  ", and the source layer is " + std::to_string(y) + " x " + std::to_string(x));
  if (t == RGBTOYUV) {
    if (!on_input)
      return refuse("edge_type", "RGBTOYUV runs only on the input layer's outgoing edge (it has no backward pass)");
    if (source_channels != 3)
      return refuse("edge_type",
                    "RGBTOYUV maps 3 colour channels to 3, and the layers have " + std::to_string(source_channels));
    if (e.GetImageSizeT() != 1) return refuse("edge_type", "RGBTOYUV is not supported on 3-D layers (image_size_t > 1)");
    if (into_output)
      return refuse("edge_type", "RGBTOYUV cannot write the output layer (the layer it writes receives no derivative, and the "
                    "loss needs one)");
  }
  return {};
}

// edge `i` of a chain (every edge's SetImageSize has run), if tied, may run with and train the parameters of the edge its
// tied_to names.  The owner must exist, be another edge, be untied itself, have parameters of the same edge_type and the
// same weight and bias shapes, and sum its bias gradient on the same stream; a tied edge may not ask for grad_check (its
// owner checks the shared tensors).  tied_to
Objection TieError(const std::vector<const Edge*>& edges, size_t i) {
  const EdgeConfig& c = edges[i]->Config();
  if (c.tied_to.empty()) return {};
  auto refuse = [](const std::string& why) { return Objection{"field 'tied_to': " + why, {"tied_to"}}; };
  const std::string owner = "edge '" + c.tied_to + "'";
  size_t k = 0;
  while (k < edges.size() && edges[k]->GetName() != c.tied_to) k++;
  if (k == edges.size()) return refuse("the net has no edge '" + c.tied_to + "'");
  if (k == i) return refuse("an edge cannot be tied to itself");
  const EdgeConfig& o = edges[k]->Config();
  if (!o.tied_to.empty())
    return refuse(owner + " is itself tied (to '" + o.tied_to + "'): tie to '" + o.tied_to + "' instead");
  if (edges[k]->HasNoParameters()) return refuse(owner + " has no parameters");
  if (o.edge_type != c.edge_type)
    return refuse(owner + " is " + kEdgeTypeNames[o.edge_type] + ", this edge " + kEdgeTypeNames[c.edge_type] +
                  " (a tie joins edges of one edge_type)");
  const EdgeWithWeight *w = dynamic_cast<const EdgeWithWeight*>(edges[i]), *ow = dynamic_cast<const EdgeWithWeight*>(edges[k]);
  auto shape = [](const Shape4D& s) {
    return "(" + std::to_string(s.shape[0]) + ", " + std::to_string(s.shape[1]) + ", " + std::to_string(s.shape[2]) + ", " +
           std::to_string(s.shape[3]) + ")";
  };
  const Shape4D a = w->GetWeightShape(), b = ow->GetWeightShape();
  if (memcmp(&a, &b, sizeof(a)) != 0)
    return refuse("the weights of this edge have shape " + shape(a) + ", those of " + owner + " " + shape(b));
  auto bias = [](const EdgeWithWeight* e) {
    const EdgeConfig& x = e->Config();
    if (x.has_no_bias) return std::string("none (has_no_bias)");
    return std::to_string(e->GetNumOutputChannels()) + " x " + std::to_string(e->GetBiasCols()) +
           (x.edge_type == CONVOLUTIONAL ? (x.shared_bias ? " (shared_bias)" : " (one per output position)") : "");
  };
  if (bias(w) != bias(ow)) return refuse("the bias of this edge is " + bias(w) + ", that of " + owner + " " + bias(ow));
  // every contribution to the shared bias gradient must come from one stream: a 3-D conv sums its bias on the main stream,
  // a 2-D one on the side lane
  if (c.edge_type == CONVOLUTIONAL && (edges[i]->GetImageSizeT() == 1) != (edges[k]->GetImageSizeT() == 1))
    return refuse("a tie joins a 3-D and a 2-D convolution");
  if (c.grad_check) return refuse("grad_check on a tied edge (set it on " + owner + ", which checks the shared tensors)");
  return {};
}

// edge `i` of a chain (shapes known, ties accepted by TieError) may be frozen or trained as its block_backprop says.  A
// weighted edge below a blocked one must be blocked itself, the edges of a tie group agree, and a frozen edge may not ask
// for grad_check.  block_backprop of the blocked edge *at
Objection FrozenError(const std::vector<const Edge*>& edges, size_t i, size_t* at) {
  const Edge& e = *edges[i];
  auto refuse = [](const std::string& why) { return Objection{"field 'block_backprop': " + why, {"block_backprop"}}; };
  for (size_t k = 0; k < edges.size() && !e.Config().tied_to.empty(); k++)
    if (edges[k]->GetName() == e.Config().tied_to && edges[k]->IsBackPropBlocked() != e.IsBackPropBlocked()) {
      const Edge& blocked = e.IsBackPropBlocked() ? e : *edges[k];
      const Edge& open = e.IsBackPropBlocked() ? *edges[k] : e;
      *at = e.IsBackPropBlocked() ? i : k;
      return refuse("edge '" + blocked.GetName() + "' is blocked and edge '" + open.GetName() + "' of its tie group is not (a "
                    "tie group is frozen or trained as a whole)");
    }
  size_t above = i;                                  // the nearest blocked edge at or above this one
  while (above < edges.size() && !edges[above]->IsBackPropBlocked()) above++;
  if (above == edges.size() || e.HasNoParameters()) return {};
  *at = above;
  if (above != i)
    return refuse("this edge has weights and lies below the blocked edge '" + edges[above]->GetName() + "', so no derivative "
                  "reaches it and nothing would train it: set block_backprop on it too");
  if (e.Config().grad_check) return refuse("grad_check on a frozen edge (its parameters get no gradient)");
  return {};
}

// the activation, loss function and performance metric of `c` can run.  The loss function or performance metric that
// fails, else the activation
Objection LayerConfigError(const LayerConfig& c) {
  const bool softmax = c.activation == SOFTMAX || c.activation == SOFTMAX_DIST;
  if (!c.is_output) {
    if (softmax)
      return {"SOFTMAX / SOFTMAX_DIST is an output activation (back-propagation through a softmax is not implemented)",
              {"activation"}};
    return {};
  }
  auto name = [](int f) -> std::string {
    static const char* n[] = {"SQUARED_ERROR", "LINEAR_ERROR", "CROSS_ENTROPY_MULTINOMIAL", "CROSS_ENTROPY_BINARY",
                              "CROSS_ENTROPY_MULTINOMIAL_DISTRIBUTED", "CLASSIFICATION_MULTINOMIAL", "CLASSIFICATION_BINARY",
                              "HINGE_LINEAR", "HINGE_QUADRATIC"};
    return f >= 0 && f <= HINGE_QUADRATIC ? n[f] : "LossFunction " + std::to_string(f);
  };
  const std::string target = TakesLabels(c.activation) ? "integer labels" : "a float target per feature";
  for (int which = 0; which < 2; which++) {
    const int f = which ? c.performance_metric : c.loss_function;
    const std::string field = which ? "performance_metric" : "loss_function";
    auto refuse = [&](const std::string& why) { return Objection{field + " " + name(f) + why, {field, "activation"}}; };
    if (f < SQUARED_ERROR || f > CLASSIFICATION_BINARY) return refuse(" is not supported");
    if (!which && (f == CLASSIFICATION_MULTINOMIAL || f == CLASSIFICATION_BINARY))
      return refuse(" has no derivative to train with");
    if (ReadsLabels(f) != TakesLabels(c.activation))
      return refuse(std::string(" reads ") + (ReadsLabels(f) ? "integer labels" : "a float target per feature") +
                    ", but this output layer's activation has " + target);
  }
  return {};
}
}  // namespace

// `emit`: this call is the last writer of the tensor and the next conv edge reads it as bf16 (see LastStateWriter)
void Layer::ApplyActivation(bool emit) {
  if (activation_fused_) return;
  switch (config_.activation) {
    case LINEAR: break;
    case RECTIFIED_LINEAR:
      if (emit) convnet_b200_emit_bf16_next();
      state_.ApplyReLU();                                  // LowerBound(0), layer.cc:550
      break;
    case LOGISTIC:                                         // ApplyLogistic, layer.cc:598
      if (emit) convnet_b200_emit_bf16_next();
      cnb_logistic(state_.GetDevData(), (long long)state_.GetNumEls());
      break;
    case SOFTMAX: case SOFTMAX_DIST: state_.ApplySoftmax(); break;
  }
}
// (of the state as stored: for a layer with dropout that is act(x) * mask, the reference's order, DESIGN.md §5)
void Layer::ApplyDerivativeOfActivation(bool emit) {
  if (deriv_fused_) return;
  if (config_.activation == RECTIFIED_LINEAR) {
    if (emit) convnet_b200_emit_bf16_next();
    deriv_.ApplyDerivOfReLU(state_);
  } else if (config_.activation == LOGISTIC) {            // ApplyDerivativeOfLogistic, layer.cc:601
    if (emit) convnet_b200_emit_bf16_next();
    cnb_logistic_deriv(deriv_.GetDevData(), state_.GetDevData(), (long long)deriv_.GetNumEls());
  }
}
void Layer::ApplyDropout(bool train, unsigned long long step, unsigned long long salt, bool emit) {      // layer.cc:367-395, scale-up at train time
  if (config_.dropprob <= 0 || !train) return;
  if (emit) convnet_b200_emit_bf16_next();
  // salt = model seed and data-parallel rank (the reference seeds each process with seed + rank, convnet.cc:67-68):
  // replicas must not draw the same mask for the same local image index
  const unsigned long long seed = DropoutSeed(step, salt);
  cnb_dropout(state_.GetDevData(), dropout_mask_.GetDevData(), (long long)state_.GetNumEls(), config_.dropprob,
              1.0f / (1.0f - config_.dropprob), seed);
}
unsigned long long Layer::DropoutSeed(unsigned long long step, unsigned long long salt) const {
  return (std::hash<std::string>()(config_.name) ^ (step * 0x9E3779B97F4A7C15ULL)) ^ salt;
}
void Layer::ApplyDerivativeofDropout(bool emit) {
  if (config_.dropprob <= 0 || config_.is_input) return;
  if (emit) convnet_b200_emit_bf16_next();
  cnb_mult(deriv_.GetDevData(), dropout_mask_.GetDevData(), (long long)deriv_.GetNumEls());
}
void Layer::SetBnMemory(Matrix& params, Matrix& grads) {
  const int C = config_.num_channels;
  params.GetSlice(gamma_, 0, C); params.GetSlice(beta_, C, 2 * C);
  grads.GetSlice(grad_gamma_, 0, C); grads.GetSlice(grad_beta_, C, 2 * C);
}
void Layer::InitializeBn() {
  const int C = config_.num_channels;
  gamma_.Set(1); beta_.Set(0);
  Matrix running;
  bn_stats_.GetSlice(running, 0, C); running.Set(0);                 // mu
  bn_stats_.GetSlice(running, C, 2 * C); running.Set(1);             // sigma
}
// layer.cc:452-478 on the state reshaped to [N*pixels x channels]; the activation follows in the same pass
void Layer::ApplyBatchNormalization(bool train, bool emit) {
  const int C = config_.num_channels;
  const long long n = (long long)state_.GetRows() * BnPixels();
  float *mu = BnStat(0), *sigma = BnStat(1);
  if (train) {
    cnb_bn_stats(pre_bn_.GetDevData(), n, C, config_.bn_epsilon, config_.bn_f, BnStat(2), BnStat(3), mu, sigma);
    mu = BnStat(2); sigma = BnStat(3);
  }
  bn_train_ = train;
  const bool logistic = config_.activation == LOGISTIC;   // the BN kernel fuses max(., 0) only: sigma is a pass after it
  if (emit && !logistic) convnet_b200_emit_bf16_next();
  cnb_bn_apply(pre_bn_.GetDevData(), state_.GetDevData(), n, C, gamma_.GetDevData(), beta_.GetDevData(), mu, sigma,
               config_.activation == RECTIFIED_LINEAR);
  if (logistic) {
    if (emit) convnet_b200_emit_bf16_next();
    cnb_logistic(state_.GetDevData(), (long long)state_.GetNumEls());
  }
}
// layer.cc:480-510, with xhat from the saved input (DESIGN.md §5: the state holds relu / dropout of the output)
void Layer::ApplyDerivativeofBatchNormalization(bool emit) {
  const long long n = (long long)state_.GetRows() * BnPixels();
  const int s = bn_train_ ? 2 : 0;
  if (emit) convnet_b200_emit_bf16_next();
  cnb_bn_backward(deriv_.GetDevData(), pre_bn_.GetDevData(), n, config_.num_channels, gamma_.GetDevData(), BnStat(s),
                  BnStat(s + 1), bn_train_, grad_gamma_.GetDevData(), grad_beta_.GetDevData());
}
void Layer::ComputeDeriv() {
  cnb_loss_deriv(config_.loss_function, state_.GetDevData(), targets_.GetDevData(), labels_, deriv_.GetDevData(),
                 loss_per_image_.GetDevData(), state_.GetRows(), state_.GetCols(), config_.loss_function_weight);
}
void Layer::ComputePerformanceMetric() {
  cnb_metric(config_.performance_metric, state_.GetDevData(), targets_.GetDevData(), labels_, metric_per_image_.GetDevData(),
             state_.GetRows(), state_.GetCols());
}

// =================================================================== DataParallelSync (NCCL, loaded lazily)
namespace {
struct NcclApi {
  void* handle = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommInitRankConfig)(ncclComm_t*, int, ncclUniqueId, int, ncclConfig_t*) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Bcast)(const void*, void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  std::string error;                                         // why it cannot be used ("": it can)
};
NcclApi& nccl() {
  static NcclApi api;
  static bool tried = false;
  if (!tried) {
    tried = true;
    // torch's bundled libnccl.so.2 is already mapped when the launcher imported torch; otherwise the loader path is used
    api.handle = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!api.handle) { api.error = std::string("cannot load libnccl.so.2: ") + dlerror(); return api; }
#define LOAD(field, sym) api.field = reinterpret_cast<decltype(api.field)>(dlsym(api.handle, sym))
    LOAD(GetUniqueId, "ncclGetUniqueId"); LOAD(CommInitRank, "ncclCommInitRank"); LOAD(CommDestroy, "ncclCommDestroy");
    LOAD(CommInitRankConfig, "ncclCommInitRankConfig");
    LOAD(AllReduce, "ncclAllReduce"); LOAD(Bcast, "ncclBroadcast"); LOAD(GetErrorString, "ncclGetErrorString");
#undef LOAD
    if (!api.GetUniqueId || !api.CommInitRank || !api.AllReduce || !api.Bcast)
      api.error = "libnccl.so.2 lacks ncclGetUniqueId, ncclCommInitRank, ncclAllReduce or ncclBroadcast";
  }
  return api;
}
NcclApi& RequireNccl() {
  if (!nccl().error.empty()) throw DeviceError("NCCL is not available: " + nccl().error);
  return nccl();
}
}  // namespace

const char* NcclErrorString(int result) {
  return nccl().GetErrorString ? nccl().GetErrorString((ncclResult_t)result) : "unknown NCCL error";
}

DataParallelSync::DataParallelSync() {}
DataParallelSync::~DataParallelSync() {
  if (comm_ && nccl().CommDestroy) nccl().CommDestroy((ncclComm_t)comm_);
  if (comm_stream_) cudaStreamDestroy(comm_stream_);
  if (ready_) cudaEventDestroy(ready_);
  if (done_) cudaEventDestroy(done_);
}
void DataParallelSync::GetUniqueId(char out[128]) {
  ncclUniqueId id;
  static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");
  NCCL_CHECK(RequireNccl().GetUniqueId(&id));
  memcpy(out, &id, 128);
}
void DataParallelSync::Init(int rank, int world, const char idbytes[128]) {
  RequireNccl();
  rank_ = rank; world_ = world;
  ncclUniqueId id;
  memcpy(&id, idbytes, 128);
  // The collective's CTAs need whole SMs (registers, shared memory) beside persistent conv kernels that own every SM they
  // touch and walk their tiles with a fixed stride: a conv CTA that finds its SM taken starts late and stretches the whole
  // kernel.  So NCCL gets exactly CONVNET_B200_NCCL_CTAS CTAs — through the communicator's own config, which holds whether or
  // not the launcher (torch.distributed) initialised NCCL and its environment cache first — and the conv grids leave that
  // many SMs free while a collective is in flight (convnet_b200_reserve_sms).  0: NCCL's default width, nothing reserved.
  const char* e = getenv("CONVNET_B200_NCCL_CTAS");
  // the widths chosen to hide AlexNet's 417 MB exchange under the backward pass: 16 CTAs up to 4 ranks, 24 above (not yet
  // retuned on H100s: ConvNet::TraceStep shows each bucket's exchange window)
  nccl_ctas_ = e ? atoi(e) : (world <= 4 ? 16 : 24);
  if (nccl_ctas_ < 0) nccl_ctas_ = 0;
  ncclComm_t c;
  if (nccl_ctas_ > 0 && nccl().CommInitRankConfig) {
    ncclConfig_t cfg = NCCL_CONFIG_INITIALIZER;
    cfg.minCTAs = nccl_ctas_;
    cfg.maxCTAs = nccl_ctas_;
    NCCL_CHECK(nccl().CommInitRankConfig(&c, world, id, rank, &cfg));
  } else {
    if (nccl_ctas_ > 0 && !getenv("NCCL_MAX_CTAS")) {          // older NCCL: the environment, effective only if nothing read it yet
      char buf[16]; snprintf(buf, sizeof(buf), "%d", nccl_ctas_);
      setenv("NCCL_MAX_CTAS", buf, 1);
    }
    NCCL_CHECK(nccl().CommInitRank(&c, world, id, rank));
  }
  comm_ = c;
  CUDA_CHECK(cudaStreamCreateWithFlags(&comm_stream_, cudaStreamNonBlocking));
  CUDA_CHECK(cudaEventCreateWithFlags(&ready_, cudaEventDisableTiming));
  CUDA_CHECK(cudaEventCreateWithFlags(&done_, cudaEventDisableTiming));
}
void DataParallelSync::Broadcast(float* buf, size_t count) {
  if (world_ <= 1) return;
  CUDA_CHECK(cudaEventRecord(ready_, Matrix::Stream()));
  CUDA_CHECK(cudaStreamWaitEvent(comm_stream_, ready_, 0));
  NCCL_CHECK(nccl().Bcast(buf, buf, count, ncclFloat, 0, (ncclComm_t)comm_, comm_stream_));
  CUDA_CHECK(cudaEventRecord(done_, comm_stream_));
  CUDA_CHECK(cudaStreamWaitEvent(Matrix::Stream(), done_, 0));
}
void DataParallelSync::AllReduceAverageAsync(float* buf, size_t offset, size_t count, cudaStream_t comm) {
  if (world_ <= 1 || count == 0) return;
  NCCL_CHECK(nccl().AllReduce(buf + offset, buf + offset, count, ncclFloat, ncclAvg, (ncclComm_t)comm_, comm));
}

// =================================================================== ConvNet
ConvNet::ConvNet(const ModelConfig& model, int batch_size) : model_(model), batch_size_(batch_size) {
  // BuildNet (convnet.cc:150-270), restricted to chains: edge i connects layer i to layer i+1
  if (model.layer.size() != model.edge.size() + 1)
    throw std::invalid_argument("ConvNet: the model must be a chain (" + std::to_string(model.layer.size()) + " layers, " +
                                std::to_string(model.edge.size()) + " edges)");
  for (const LayerConfig& lc : model.layer) layers_.emplace_back(new Layer(lc));
  for (size_t i = 0; i < model.edge.size(); i++) {
    edges_.emplace_back(Edge::ChooseEdgeClass(model.edge[i]));
    Edge* e = edges_.back().get();
    e->SetSource(layers_[i].get()); e->SetDest(layers_[i + 1].get());
    e->SetInputChannels(layers_[i]->GetNumChannels());
    e->SetOutputChannels(layers_[i + 1]->GetNumChannels());
    e->SetBatchSize(batch_size);
  }
  // SetImageSize propagation (convnet.cc:226-268)
  const LayerConfig& in = model.layer.front();
  layers_[0]->SetSize(in.image_size_y, in.image_size_x, in.image_size_t);
  for (size_t i = 0; i < edges_.size(); i++) {
    edges_[i]->SetImageSize(layers_[i]->GetSizeY(), layers_[i]->GetSizeX(), layers_[i]->GetSizeT());
    layers_[i + 1]->SetSize(edges_[i]->GetNumModulesY(), edges_[i]->GetNumModulesX(), edges_[i]->GetNumModulesT());
  }
  Refuse();
  frozen_ = FrozenEdges(model.edge);
  for (size_t i = 0; i < edges_.size(); i++)
    if (model.edge[i].edge_type == RGBTOYUV || ((int)i < frozen_ && !layers_[i + 1]->IsOutput())) layers_[i + 1]->SetNoDeriv();
  ResolveTies();
  PlanFusion();
}

void ConvNet::ResolveTies() {
  const int n = (int)edges_.size();
  owner_.assign(n, -1);
  home_.assign(n, -1);
  for (int i = 0; i < n; i++) {
    if (edges_[i]->HasNoParameters()) continue;
    owner_[i] = i;
    for (int k = 0; k < n; k++)
      if (edges_[k]->GetName() == model_.edge[i].tied_to) owner_[i] = k;
  }
  for (int i = n - 1; i >= 0; i--)                   // from the top down: the group's lowest edge is written last
    if (owner_[i] >= 0) home_[owner_[i]] = i;
  for (int i = 0; i < n; i++) {
    if (owner_[i] < 0) continue;
    home_[i] = home_[owner_[i]];
    if (owner_[i] != i)
      static_cast<EdgeWithWeight*>(edges_[i].get())->TieTo(static_cast<EdgeWithWeight*>(edges_[owner_[i]].get()));
  }
}
bool ConvNet::Grouped(size_t i) const {
  return owner_[i] >= 0 && std::count(owner_.begin(), owner_.end(), owner_[i]) > 1;
}

void ConvNet::Refuse() const {
  // `o`, if it objects, as the refusal of layer or edge `at`, its message after `where`
  auto check = [](const std::string& where, bool edge, size_t at, const Objection& o) {
    if (!o.why.empty()) throw ModelRefused(where + ": " + o.why, edge, at, o.fields);
  };
  for (size_t i = 0; i < layers_.size(); i++)        // activations, loss functions and metrics this class cannot run
    check("layer '" + layers_[i]->GetName() + "'", false, i, LayerConfigError(model_.layer[i]));
  std::vector<const Edge*> chain;
  for (const auto& e : edges_) chain.push_back(e.get());
  for (size_t i = 0; i < edges_.size(); i++) {
    const std::string where = "edge '" + edges_[i]->GetName() + "'";
    const int from = layers_[i]->GetNumChannels(), to = layers_[i + 1]->GetNumChannels();
    check(where, true, i, SampleEdgeError(*edges_[i], from, to, layers_[i]->IsInput(), layers_[i + 1]->IsOutput()));
    check(where, true, i, EdgeShapeError(*edges_[i], from, to));
    check(where, true, i, TieError(chain, i));
    size_t at = i;
    const Objection frozen = FrozenError(chain, i, &at);
    check(where, true, at, frozen);
    if (model_.edge[i].edge_type == LOCAL && layers_[i]->GetSizeT() != 1)     // the untied conv kernels are 2-D only
      check(where, true, i, {"LOCAL is not supported on 3-D layers (image_size_t > 1)", {"edge_type"}});
    const int init = model_.edge[i].initialization;
    if (!model_.edge[i].tied_to.empty()) continue;                          // (its initialisation is never used)
    if (!edges_[i]->HasNoParameters() && init != DENSE_GAUSSIAN && init != DENSE_GAUSSIAN_SQRT_FAN_IN &&
        init != DENSE_UNIFORM && init != DENSE_UNIFORM_SQRT_FAN_IN && init != CONSTANT && init != PRETRAINED)
      check(where, true, i, {"initialization " + std::to_string(init) + " is not implemented", {"initialization"}});
  }
  for (size_t i = 0; i < layers_.size(); i++) {      // what the batch-norm passes cannot run
    const Layer* l = layers_[i].get();
    if (!l->BatchNormalize()) continue;
    const std::string where = "layer '" + l->GetName() + "'";
    std::string why;
    if (l->IsInput() || l->IsOutput()) why = "batch_normalize is not supported on the input or output layer";
    else if (model_.edge[i - 1].edge_type == RGBTOYUV)
      why = "field 'batch_normalize': not supported on the layer RGBTOYUV writes (it receives no derivative)";
    else if (l->GetSizeT() > 1) why = "batch_normalize is not supported on 3-D layers (image_size_t > 1)";
    check(where, false, i, {why, {"batch_normalize"}});
    const LayerConfig& c = model_.layer[i];
    for (const auto& [f, o] :
         {std::pair{"gamma_optimizer", &c.gamma_optimizer}, std::pair{"beta_optimizer", &c.beta_optimizer}})
      if (const char* err = BnOptimizerConfigError(*o))
        check(where, false, i, {std::string("batch_normalize ") + f + ": " + err, {f, "batch_normalize"}});
  }
}

// Epilogue fusion of the layers' activation (ReLU, logistic), its derivative and the dropout into the neighbouring
// edges (SURVEY.md 8(f) rank 2)
void ConvNet::PlanFusion() {
  // CONVNET_B200_NO_FUSED_DROPOUT=1, _NO_DROPOUT_FOLD=1, _NO_PRESTAGE=1: the separate passes these fusions replace (the
  // reference run of tests/test_gpu_staging.py).  Read once per process
  auto on = [](const char* name) { const char* v = getenv(name); return !(v && v[0] == '1'); };
  static const bool fused_dropout = on("CONVNET_B200_NO_FUSED_DROPOUT"), dropout_fold = on("CONVNET_B200_NO_DROPOUT_FOLD"),
                    prestage = on("CONVNET_B200_NO_PRESTAGE");
  prestage_ = prestage;
  for (size_t i = 0; i < edges_.size(); i++) {
    Edge* e = edges_[i].get();
    Layer *src = layers_[i].get(), *dst = layers_[i + 1].get();
    const Edge::Absorbs a = e->CanAbsorb();
    // the activation of a layer rides where the kernel applies ReLU, and sigma only where it can apply sigma too
    auto fused = [&a](int act, bool can) { return act != CNB_ACT_LINEAR && can && (act == CNB_ACT_RELU || a.logistic); };
    const int up = ActCode(dst->GetActivation()), down = src->ReceivesDeriv() ? ActCode(src->GetActivation()) : CNB_ACT_LINEAR;
    Edge::FusionPlan p;
    // a batch-normalised layer: the edge writes the pre-normalisation input, the BN pass applies the activation
    if (!dst->BatchNormalize() && fused(up, a.act_up)) p.up_act = up;
    if (fused(down, a.act_down)) p.down_act = down;
    p.dropout_up = a.dropout && p.up_act != CNB_ACT_LINEAR && fused_dropout;
    p.scale_down = a.dropout && p.down_act != CNB_ACT_LINEAR && dropout_fold;
    p.sums_bias_below = a.sums_bias_below;
    // a pool-undo sums the handed-off bias gradient on the main stream, the other edges of a tie group sum theirs into the
    // same bias on the side lane: a tie group keeps every contribution on the side lane, in back-propagation order
    p.offers_bias_grad = a.per_channel_bias && !Grouped(i);
    e->SetFusionPlan(p);
    dst->SetActivationFused(p.up_act != CNB_ACT_LINEAR || dst->BatchNormalize());
    src->SetDerivFused(p.down_act != CNB_ACT_LINEAR);
  }
}

// Parameters (or activations) were, or may have been, written by something the library cannot see (cudaMemcpy, the
// caller's own kernels): forget every staged bf16 copy.  Writes made through the library keep the copies coherent themselves.
void ConvNet::InvalidateStaging() { convnet_b200_bf16_invalidate(nullptr); }

ConvNet::~ConvNet() {
  if (comm_) { cudaStreamSynchronize(comm_); cudaStreamDestroy(comm_); }
  if (side_) { cudaStreamSynchronize(side_); cudaStreamDestroy(side_); }
  if (opt_) { cudaStreamSynchronize(opt_); cudaStreamDestroy(opt_); }
  if (ev_opt_) cudaEventDestroy(ev_opt_);
  if (ev_comm_) cudaEventDestroy(ev_comm_);
  for (cudaEvent_t e : ev_reduced_) cudaEventDestroy(e);
  if (ev_main_) cudaEventDestroy(ev_main_);
  if (ev_side_) cudaEventDestroy(ev_side_);
  if (lane_.ready) cudaEventDestroy(lane_.ready);
  for (cudaEvent_t e : {trace_.t0, trace_.fwd, trace_.bwd, trace_.end}) if (e) cudaEventDestroy(e);
  for (std::vector<cudaEvent_t>* v : {&trace_.c0, &trace_.c1, &trace_.s1}) for (cudaEvent_t e : *v) cudaEventDestroy(e);
  if (polyak_) cudaFree(polyak_);
  if (allocated_) {
    convnet_b200_reserve_sms(0);
    convnet_b200_bf16_invalidate(nullptr);                   // the buffers go away; a later net may get the same addresses
  }
}

// AllocateEdgeMemory (convnet.cc:272-298): one flat buffer, each edge's slice padded to 128 floats.  The [gamma | beta]
// slice of a batch-normalised layer follows the slice of the edge that writes it: both gradients are final once that edge
// has run ComputeOuter, so the bucket that carries the edge carries them too (edge_span_ is what PlanBuckets sees)
OptimizerConfig& ModelOptimizer(ModelConfig& m, const TrainedTensor& t) {
  switch (t.kind) {
    case TrainedTensor::WEIGHTS: return m.edge[t.owner].weight_optimizer;
    case TrainedTensor::BIAS: return m.edge[t.owner].bias_optimizer;
    case TrainedTensor::GAMMA: return m.layer[t.edge + 1].gamma_optimizer;
    default: return m.layer[t.edge + 1].beta_optimizer;
  }
}

void ConvNet::PlanParameters() {
  edge_offset_.clear(); edge_size_.clear(); edge_span_.clear(); tensors_.clear();
  bn_offset_.assign(layers_.size(), -1);
  size_t total = 0;
  auto add = [&](TrainedTensor::Kind kind, const std::string& owner, int edge, size_t offset, long long n, int rows, int of) {
    static const char* const suffix[] = {":weight", ":bias", ":gamma", ":beta"};
    TrainedTensor t{kind, owner + suffix[kind], edge, offset, n, rows};
    t.owner = of;
    t.opt = ModelOptimizer(model_, t);
    tensors_.push_back(t);
  };
  for (size_t i = 0; i < edges_.size(); i++) {
    // the slice at edge i: the parameters of the owner whose tie group starts here (edge i's own when untied), else none
    const int o = owner_[i] >= 0 && home_[i] == (int)i ? owner_[i] : -1;
    const size_t req = o >= 0 ? edges_[o]->GetParameterMemoryRequirement() : 0;
    edge_offset_.push_back(total);
    edge_size_.push_back(req);
    // the rows of the weights are the output units; the bias is ONE row (fc_edge.cc:29-32)
    if (o >= 0) {
      const EdgeWithWeight* w = static_cast<const EdgeWithWeight*>(edges_[o].get());
      add(TrainedTensor::WEIGHTS, w->GetName(), (int)i, total, w->WeightCount(), w->GetNumOutputChannels(), o);
      add(TrainedTensor::BIAS, w->GetName(), (int)i, total + (size_t)w->WeightCount(), w->BiasCount(), 1, o);
    }
    total += DIVUP(req, (size_t)128) * 128;
    Layer* l = layers_[i + 1].get();
    if (l->BatchNormalize()) {
      const int C = l->GetNumChannels();
      bn_offset_[i + 1] = (long long)total;
      add(TrainedTensor::GAMMA, l->GetName(), (int)i, total, C, 1, (int)i);
      add(TrainedTensor::BETA, l->GetName(), (int)i, total + C, C, 1, (int)i);
      total += DIVUP(2 * (size_t)C, (size_t)128) * 128;
    }
    edge_span_.push_back(total - edge_offset_.back());
  }
  num_params_ = total;
}

void ConvNet::AllocateMemory() {
  allocated_ = true;
  for (auto& l : layers_) l->AllocateMemory(batch_size_);
  PlanParameters();
  size_t total = num_params_;
  if (total == 0) total = 128;
  parameters_.AllocateGPUMemory(1, (int)total);
  grad_parameters_.AllocateGPUMemory(1, (int)total);
  history_.AllocateGPUMemory(1, (int)total);
  loss_sum_.AllocateGPUMemory(1, 2);                           // the loss, the performance metric
  for (size_t i = 0; i < edges_.size(); i++) {
    if (owner_[i] < 0) continue;
    const int h = home_[i];                                    // every edge of a tie group is carved from the one slice
    Matrix p, g;
    parameters_.GetSlice(p, (int)edge_offset_[h], (int)(edge_offset_[h] + edge_size_[h]));
    grad_parameters_.GetSlice(g, (int)edge_offset_[h], (int)(edge_offset_[h] + edge_size_[h]));
    edges_[i]->SetMemory(p);
    edges_[i]->SetGradMemory(g);
    edges_[i]->Initialize(model_.seed + 17 * (unsigned)i);     // (a tied edge initialises nothing)
  }
  for (size_t i = 0; i < layers_.size(); i++) {
    if (bn_offset_[i] < 0) continue;
    const int lo = (int)bn_offset_[i], hi = lo + 2 * layers_[i]->GetNumChannels();
    Matrix p, g;
    parameters_.GetSlice(p, lo, hi);
    grad_parameters_.GetSlice(g, lo, hi);
    layers_[i]->SetBnMemory(p, g);
    layers_[i]->InitializeBn();
  }
  if (std::any_of(tensors_.begin(), tensors_.end(), [](const TrainedTensor& t) { return IsAdaptive(t.opt); }))
    AllocateAdaptiveState();
  // the reference allocates the optimizers before Initialize reads a PRETRAINED edge (fc_edge.cc:42, convnet.cc:286-303),
  // so the edge takes the history, the step and the adaptive state from the file too
  for (size_t i = 0; i < edges_.size(); i++)
    if (owner_[i] == (int)i && model_.edge[i].initialization == PRETRAINED) LoadPretrained(i);
  CUDA_CHECK(cudaStreamSynchronize(Matrix::Stream()));
  InvalidateStaging();
  CUDA_CHECK(cudaStreamCreateWithFlags(&side_, cudaStreamNonBlocking));
  CUDA_CHECK(cudaStreamCreateWithFlags(&opt_, cudaStreamNonBlocking));
  CUDA_CHECK(cudaEventCreateWithFlags(&ev_opt_, cudaEventDisableTiming));
  CUDA_CHECK(cudaStreamCreateWithFlags(&comm_, cudaStreamNonBlocking));
  CUDA_CHECK(cudaEventCreateWithFlags(&ev_comm_, cudaEventDisableTiming));
  CUDA_CHECK(cudaEventCreateWithFlags(&ev_main_, cudaEventDisableTiming));
  CUDA_CHECK(cudaEventCreateWithFlags(&ev_side_, cudaEventDisableTiming));
  SetBucketFloats((size_t)8 << 20);
  lane_.stream = side_;
  CUDA_CHECK(cudaEventCreateWithFlags(&lane_.ready, cudaEventDisableTiming));
  for (auto& e : edges_)
    if (EdgeWithWeight* w = dynamic_cast<EdgeWithWeight*>(e.get())) w->SetSideLane(&lane_);
}

void ConvNet::AllocateAdaptiveState() {
  state_.AllocateGPUMemory(1, parameters_.GetCols());
  for (const TrainedTensor& t : tensors_) InitState(t);
}
void ConvNet::InitState(const TrainedTensor& t) {
  Matrix s;
  state_.GetSlice(s, (int)t.offset, (int)(t.offset + t.n));
  InitAdaptiveState(t.opt, s);
}
void ConvNet::SetOptimizer(TrainedTensor& t, const OptimizerConfig& c) {
  const bool restart = c.optimizer_type != t.opt.optimizer_type || c.adagrad_delta != t.opt.adagrad_delta;
  t.opt = c;
  if (!IsAdaptive(c)) return;
  if (!AdaptiveState()) AllocateAdaptiveState();               // initialises every slice, this one included
  else if (restart) InitState(t);
}

// The pass that writes a layer's state last in Fprop, or its derivative last in Bprop.  In bf16 mode it also writes the bf16
// copy the next conv edge multiplies with (emit); a dgrad that writes a derivative last can also sum its channels, which
// is the bias gradient of the edge below.
enum class Writer { EDGE, BN, ACTIVATION, DROPOUT };
// Fprop runs the edge (into the pre-normalisation input of a batch-normalised layer), BN apply (with the activation), the
// activation pass, the dropout pass
static Writer LastStateWriter(const Layer& l, bool dropout_pass) {
  if (dropout_pass) return Writer::DROPOUT;
  if (l.HasSeparateActivationPass()) return Writer::ACTIVATION;
  if (l.BatchNormalize()) return Writer::BN;
  return Writer::EDGE;
}
// Bprop runs the edge above, the dropout pass, the activation' pass, BN backward
static Writer LastDerivWriter(const Layer& l, bool dropout_pass) {
  if (l.BatchNormalize()) return Writer::BN;
  if (l.HasSeparateDerivPass()) return Writer::ACTIVATION;
  if (dropout_pass) return Writer::DROPOUT;
  return Writer::EDGE;
}

void ConvNet::Fprop(bool train) {                            // convnet.cc:377-388
  const bool bf16 = convnet_b200_get_conv_precision() == 2;
  dropout_active_ = train;
  for (size_t i = 1; i < layers_.size(); i++) {
    Layer* l = layers_[i].get();
    Edge* e = edges_[i - 1].get();
    const bool want = bf16 && i < edges_.size() && edges_[i]->WantsBf16Input();
    // dropout inside the edge's epilogue (no mask tensor) when the backward pass will not need the mask either
    const bool fuse_drop = train && DropoutFolds(i) && e->Plan().dropout_up;
    const bool drop = train && l->HasDropout() && !fuse_drop;
    const Writer last = LastStateWriter(*l, drop);
    Edge::UpRequest r;
    r.emit = want && last == Writer::EDGE;
    if (fuse_drop) { r.drop_prob = l->DropoutProb(); r.drop_scale = l->DropoutScale(); r.drop_seed = l->DropoutSeed(step_, dropout_salt_); }
    e->Request(r);
    e->ComputeUp(layers_[i - 1]->GetState(), l->BatchNormalize() ? l->GetPreBN() : l->GetState(), /*overwrite=*/true, train);
    if (l->BatchNormalize()) l->ApplyBatchNormalization(train, want && last == Writer::BN);
    l->ApplyActivation(want && last == Writer::ACTIVATION);
    if (drop) l->ApplyDropout(train, step_, dropout_salt_, want && last == Writer::DROPOUT);
  }
}

bool ConvNet::DropoutFolds(size_t i) const {
  // edges_[i]: the edge whose ComputeDown writes layers_[i]'s derivative.  Where the mask drops a unit of a ReLU or logistic
  // layer its state is 0, and so is the derivative of the activation there
  return i >= 1 && i < edges_.size() && layers_[i]->HasDropout() && edges_[i]->Plan().scale_down;
}

void ConvNet::ComputeDeriv() { OutputLayer().ComputeDeriv(); }

float ConvNet::GetLoss() {                                   // Layer::GetLoss: the weighted sum over the batch (layer.cc:435-437)
  Layer& out = OutputLayer();
  out.ComputeDeriv();
  cnb_sum(out.GetLossPerImage(), loss_sum_.GetDevData(), batch_size_);
  return out.LossWeight() * loss_sum_.ReadValue(0);
}
float ConvNet::GetPerformanceMetric() {
  SumPerformanceMetric(loss_sum_.GetDevData() + 1);
  return loss_sum_.ReadValue(1);
}
void ConvNet::SumPerformanceMetric(float* dst) {
  Layer& out = OutputLayer();
  out.ComputePerformanceMetric();
  cnb_sum(out.GetMetricPerImage(), dst, batch_size_);
}

void ConvNet::Bprop() {                                      // convnet.cc:390-405 + 362-375
  const bool bf16 = convnet_b200_get_conv_precision() == 2;
  // a layer's dropout derivative is one factor on the kept units, which the fused act' of the dgrad above already selects:
  // that dgrad scales by it when the last Fprop applied dropout; otherwise a pass multiplies by the mask
  auto folds = [this](int k) { return dropout_active_ && DropoutFolds((size_t)k); };
  auto dropout_pass = [&](int k) { return layers_[k]->HasDropout() && !folds(k); };
  // edge i - 1 writes layer i: the frozen edges below the first trained one run no backward pass (the reference's
  // ConvNet::Bprop returns at a blocked edge, convnet.cc:363)
  for (int i = (int)layers_.size() - 1; i > frozen_; i--) {
    Layer* out = layers_[i].get();
    Layer* in = layers_[i - 1].get();
    Edge* e = edges_[i - 1].get();
    // the derivative of `out` is final once its passes have run (the reference runs them at the top of the NEXT loop
    // iteration, i.e. before this layer's edges); batch normalisation also produces the gamma / beta gradients before the
    // ComputeOuter below, which makes this edge's bucket final
    if (!out->IsOutput() && out->ReceivesDeriv()) {
      const bool want = bf16 && e->WantsBf16Deriv();
      const bool drop = dropout_pass(i);
      const Writer last = LastDerivWriter(*out, drop);
      if (drop) out->ApplyDerivativeofDropout(want && last == Writer::DROPOUT);
      out->ApplyDerivativeOfActivation(want && last == Writer::ACTIVATION);
      if (out->BatchNormalize()) out->ApplyDerivativeofBatchNormalization(want && last == Writer::BN);
    }
    e->ComputeOuter(in->GetState(), out->GetDeriv());
    // data parallel: ship every bucket whose last gradient just became final (side stream, overlaps the rest of bprop)
    if (dp_ && dp_->world() > 1)
      for (size_t bi = 0; bi < buckets_.size(); bi++) {
        const Bucket& b = buckets_[bi];
        if (b.trigger != i - 1) continue;
        if (!comm_pending_) convnet_b200_reserve_sms(dp_->reserved_sms());
        // the bucket's gradients: weight gradients on the main stream, bias gradients (column sums) on the side stream
        CUDA_CHECK(cudaEventRecord(ev_main_, Matrix::Stream()));
        CUDA_CHECK(cudaStreamWaitEvent(comm_, ev_main_, 0));
        CUDA_CHECK(cudaEventRecord(ev_side_, side_));
        CUDA_CHECK(cudaStreamWaitEvent(comm_, ev_side_, 0));
        if (trace_.on) CUDA_CHECK(cudaEventRecord(trace_.c0[bi], comm_));
        dp_->AllReduceAverageAsync(grad_parameters_.GetDevData(), b.lo, b.hi - b.lo, comm_);
        CUDA_CHECK(cudaEventRecord(ev_reduced_[bi], comm_));
        if (trace_.on) CUDA_CHECK(cudaEventRecord(trace_.c1[bi], comm_));
        comm_pending_ = true;
      }
    if (in->ReceivesDeriv()) {
      const bool last = LastDerivWriter(*in, dropout_pass(i - 1)) == Writer::EDGE;
      EdgeWithWeight* below = i >= 2 ? dynamic_cast<EdgeWithWeight*>(edges_[i - 2].get()) : nullptr;
      Edge::DownRequest r;
      r.emit = bf16 && i >= 2 && edges_[i - 2]->WantsBf16Deriv() && last;
      if (folds(i - 1)) r.scale = in->DropoutScale();
      if (last && below && e->Plan().sums_bias_below && below->Plan().offers_bias_grad) r.bias_grad = below->HandOffBiasGrad();
      e->Request(r);
      e->ComputeDown(out->GetDeriv(), in->GetState(), out->GetState(), in->GetDeriv(), /*overwrite=*/true);
    }
    // the optimizer step of a bucket follows its all-reduce on the side stream once its edges are done with the weights
    if (eager_update_)
      for (size_t bi = 0; bi < buckets_.size(); bi++)
        if (buckets_[bi].trigger == i - 1) {
          if (dp_ && dp_->world() > 1) CUDA_CHECK(cudaStreamWaitEvent(opt_, ev_reduced_[bi], 0));        // SGD after its all-reduce
          IssueBucketUpdate(buckets_[bi]);
          if (trace_.on) CUDA_CHECK(cudaEventRecord(trace_.s1[bi], opt_));
        }
  }
  if (!eager_update_ && !(dp_ && dp_->world() > 1)) WaitSide();   // stand-alone Bprop: the gradients are complete on return
}

// the SGD step of one bucket on the optimizer stream, after (events) that bucket's all-reduce, the bias-gradient sums
// queued on the side stream so far, and the compute stream's last read of the bucket's weights in this step.  Its own
// stream: an all-reduce waits for the side stream's bias gradients, and must not queue behind an earlier bucket's SGD step
void ConvNet::IssueBucketUpdate(const Bucket& b) {
  std::vector<CnbOptTensorEx> tensors;
  AppendUpdates(b.trigger, b.last, tensors);
  if (tensors.empty()) return;
  CUDA_CHECK(cudaEventRecord(ev_main_, Matrix::Stream()));
  CUDA_CHECK(cudaStreamWaitEvent(opt_, ev_main_, 0));
  CUDA_CHECK(cudaEventRecord(ev_side_, side_));
  CUDA_CHECK(cudaStreamWaitEvent(opt_, ev_side_, 0));
  void* main_stream = convnet_b200_get_stream();
  convnet_b200_set_stream(opt_);
  // the update, and the rescale of the rows of norm-limited tensors: both before the banks below are rebuilt from the weights
  // (PlanBuckets splits at edge boundaries, so every row of a tensor is updated in this one call)
  cnb_opt_update_multi(tensors.data(), (int)tensors.size());
  // what the next step's dgrad derives from these weights alone (bf16 filter banks): rebuilt here, behind the update
  // (a tie group's weights are updated in the bucket of its lowest edge: every edge of the group rebuilds its banks here)
  if (prestage_)
    for (int i = b.trigger; i <= b.last; i++)
      if (owner_[i] >= 0 && home_[i] == i)
        for (size_t k = 0; k < edges_.size(); k++)
          if (owner_[k] == owner_[i]) static_cast<EdgeWithWeight*>(edges_[k].get())->PrestageDown();
  convnet_b200_set_stream(main_stream);
  opt_pending_ = true;
}
void ConvNet::WaitSide() {
  if (lane_.used) { side_pending_ = true; lane_.used = false; }
  if (comm_pending_) {                                       // every all-reduce of the step (the SGD steps on side_ wait for theirs too)
    CUDA_CHECK(cudaEventRecord(ev_comm_, comm_));
    CUDA_CHECK(cudaStreamWaitEvent(Matrix::Stream(), ev_comm_, 0));
    comm_pending_ = false;
    convnet_b200_reserve_sms(0);
  }
  if (opt_pending_) {
    CUDA_CHECK(cudaEventRecord(ev_opt_, opt_));
    CUDA_CHECK(cudaStreamWaitEvent(Matrix::Stream(), ev_opt_, 0));
    opt_pending_ = false;
  }
  if (!side_pending_) return;
  CUDA_CHECK(cudaEventRecord(ev_side_, side_));
  CUDA_CHECK(cudaStreamWaitEvent(Matrix::Stream(), ev_side_, 0));
  side_pending_ = false;
}

void ConvNet::UpdateWeights() {                              // convnet.cc:440-450
  WaitSide();                                                // replaces Accumulate + Broadcast (MPI through host memory)
  if (updated_in_bprop_) { updated_in_bprop_ = false; return; }        // TrainOneBatch: every bucket was updated on the side stream
  // one multi-tensor launch for every trained weight and bias matrix of the net (the reference loops the edges that are
  // not blocked: optimizer.cc:174-279, convnet.cc:445)
  std::vector<CnbOptTensorEx> tensors;
  AppendUpdates(frozen_, (int)edges_.size() - 1, tensors);
  cnb_opt_update_multi(tensors.data(), (int)tensors.size());
}

void ConvNet::AppendUpdates(int first, int last, std::vector<CnbOptTensorEx>& out) {
  for (int i = first; i <= last; i++)                          // one gradient counter per tie group, reset with its update
    if (owner_[i] >= 0 && home_[i] == i) static_cast<EdgeWithWeight*>(edges_[owner_[i]].get())->NotifyStart();
  float *p = parameters_.GetDevData(), *h = history_.GetDevData(), *g = grad_parameters_.GetDevData(), *s = AdaptiveState();
  for (TrainedTensor& t : tensors_)
    if (t.edge >= first && t.edge <= last && t.n > 0)
      AppendOptTensor(t.opt, t.step, p + t.offset, h + t.offset, g + t.offset, s ? s + t.offset : nullptr, t.n, t.rows, out);
}

void ConvNet::ReduceLearningRate(float factor) {             // convnet.cc:820-825, edge_with_weight.cc:90-93
  for (TrainedTensor& t : tensors_)
    if (t.OnEdge()) t.opt.epsilon *= factor;
}

void ConvNet::TrainOneBatch(float* loss_out) {               // convnet.cc:475-485 (GetBatch is the caller's H2D copy)
  if (trace_.on) CUDA_CHECK(cudaEventRecord(trace_.t0, Matrix::Stream()));
  Fprop(true);
  ComputeDeriv();
  if (trace_.on) CUDA_CHECK(cudaEventRecord(trace_.fwd, Matrix::Stream()));
  if (loss_out) {                                            // GetLoss: one scalar D2H per step, like the reference
    cnb_sum(OutputLayer().GetLossPerImage(), loss_sum_.GetDevData(), batch_size_);
  }
  eager_update_ = true;
  Bprop();
  if (trace_.on) CUDA_CHECK(cudaEventRecord(trace_.bwd, Matrix::Stream()));
  updated_in_bprop_ = true;
  eager_update_ = false;
  UpdateWeights();
  if (trace_.on) CUDA_CHECK(cudaEventRecord(trace_.end, Matrix::Stream()));
  if (loss_out) *loss_out = OutputLayer().LossWeight() * loss_sum_.ReadValue(0);
  step_++;
}

std::vector<float> ConvNet::TraceStep() {
  auto make = [](cudaEvent_t* e) { if (!*e) CUDA_CHECK(cudaEventCreate(e)); };
  make(&trace_.t0); make(&trace_.fwd); make(&trace_.bwd); make(&trace_.end);
  for (std::vector<cudaEvent_t>* v : {&trace_.c0, &trace_.c1, &trace_.s1})
    while (v->size() < buckets_.size()) { cudaEvent_t e = nullptr; make(&e); v->push_back(e); }
  CUDA_CHECK(cudaStreamSynchronize(Matrix::Stream()));
  trace_.on = true;
  TrainOneBatch(nullptr);
  trace_.on = false;
  CUDA_CHECK(cudaStreamSynchronize(Matrix::Stream()));
  CUDA_CHECK(cudaStreamSynchronize(side_));
  CUDA_CHECK(cudaStreamSynchronize(opt_));
  CUDA_CHECK(cudaStreamSynchronize(comm_));
  auto since = [&](cudaEvent_t e) { float ms = -1.f; return cudaEventElapsedTime(&ms, trace_.t0, e) == cudaSuccess ? ms : -1.f; };
  std::vector<float> out = {since(trace_.fwd), since(trace_.bwd), since(trace_.end), (float)buckets_.size()};
  const bool multi = dp_ && dp_->world() > 1;
  for (size_t bi = 0; bi < buckets_.size(); bi++) {
    out.push_back((float)((buckets_[bi].hi - buckets_[bi].lo) * 4.0 / 1e6));
    out.push_back(multi ? since(trace_.c0[bi]) : -1.f);
    out.push_back(multi ? since(trace_.c1[bi]) : -1.f);
    out.push_back(since(trace_.s1[bi]));
  }
  cudaGetLastError();
  return out;
}

std::vector<Bucket> PlanBuckets(const std::vector<size_t>& edge_offset, const std::vector<size_t>& edge_size,
                                size_t bucket_floats) {
  std::vector<Bucket> out;
  int first_weighted = -1;
  for (int i = 0; i < (int)edge_size.size(); i++) if (edge_size[i] != 0) { first_weighted = i; break; }
  size_t lo = 0, hi = 0;
  bool open = false;
  int last_weighted = -1, top = -1;
  for (int i = (int)edge_size.size() - 1; i >= 0; i--) {
    if (edge_size[i] == 0) continue;
    const size_t e_lo = edge_offset[i], e_hi = e_lo + DIVUP(edge_size[i], (size_t)128) * 128;
    if (open && i == first_weighted) { out.push_back({lo, hi, last_weighted, top}); open = false; }   // the first edge travels alone
    if (!open) { hi = e_hi; open = true; top = i; }
    lo = e_lo;
    last_weighted = i;
    if (hi - lo >= bucket_floats) { out.push_back({lo, hi, i, top}); open = false; }
  }
  if (open) out.push_back({lo, hi, last_weighted, top});
  return out;
}

void ConvNet::SetDataParallel(DataParallelSync* dp, size_t bucket_floats) {
  dp_ = dp;
  SaltDropout();
  SetBucketFloats(bucket_floats);
}
void ConvNet::SaltDropout() {
  salted_ = true;
  dropout_salt_ = ((unsigned long long)model_.seed * 0xA24BAED4963EE407ULL) ^
                  ((unsigned long long)((dp_ ? dp_->rank() : 0) + 1) * 0xD1B54A32D192ED03ULL);
}
void ConvNet::SetBucketFloats(size_t bucket_floats) {
  std::vector<size_t> trained = edge_span_;            // no bucket carries a frozen edge
  std::fill(trained.begin(), trained.begin() + frozen_, 0);
  buckets_ = PlanBuckets(edge_offset_, trained, bucket_floats);
  while (ev_reduced_.size() < buckets_.size()) {
    cudaEvent_t e;
    CUDA_CHECK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    ev_reduced_.push_back(e);
  }
}
void ConvNet::BroadcastParameters() {
  if (dp_) dp_->Broadcast(parameters_.GetDevData(), parameters_.GetNumEls());
  InvalidateStaging();
}

double ConvNet::FlopsFprop() const {
  double f = 0;
  for (const auto& e : edges_) f += e->FlopsUp();
  return f;
}
double ConvNet::FlopsTrainStep() const {                     // BASELINE.md §2c: 3x fprop minus the dgrad into the input layer
  double f = 0;
  // edge i: fprop; wgrad unless frozen; dgrad unless layer i is the input or frozen (i <= frozen_)
  for (int i = 0; i < (int)edges_.size(); i++) f += edges_[i]->FlopsUp() * (1 + (i >= frozen_) + (i > frozen_));
  return f;
}

// =================================================================== GradChecker (src/grad_check.cc)
double GradChecker::LossAtD(Matrix& w, size_t index, float value) {
  w.WriteValue(index, value);
  InvalidateStaging();
  Fprop(false);
  // per-image cross-entropy on the device, summed in double on the host: the finite difference of two ~O(batch)
  // losses must not lose the 1e-3-sized signal to fp32 summation noise
  Layer& out = OutputLayer();
  out.ComputeDeriv();
  std::vector<float> h(batch_size_);
  CUDA_CHECK(cudaMemcpyAsync(h.data(), out.GetLossPerImage(), sizeof(float) * batch_size_, cudaMemcpyDeviceToHost, Matrix::Stream()));
  CUDA_CHECK(cudaStreamSynchronize(Matrix::Stream()));
  double s = 0;
  for (float v : h) s += v;
  return (double)out.LossWeight() * s;
}

std::vector<GradCheckResult> GradChecker::Run(unsigned seed) {
  // random inputs / labels (grad_check.cc:82-90)
  std::mt19937 gen(seed);
  std::normal_distribution<float> nd(0.f, 1.f);
  Matrix& x = InputLayer().GetState();
  std::vector<float> hx(x.GetNumEls());
  for (float& v : hx) v = nd(gen);
  x.CopyFromHost(hx.data(), hx.size());
  std::vector<int> hl(batch_size_);
  const int classes = OutputLayer().GetState().GetCols();
  for (int& v : hl) v = (int)(gen() % classes);
  CUDA_CHECK(cudaMemcpy(OutputLayer().GetLabels(), hl.data(), sizeof(int) * batch_size_, cudaMemcpyHostToDevice));
  Matrix& t = OutputLayer().GetTargets();                     // a per-feature target: one the loss function accepts
  if (t.GetNumEls()) {
    const int rows = t.GetRows(), cols = t.GetCols();
    std::vector<float> ht(t.GetNumEls());
    std::uniform_real_distribution<float> ud(0.f, 1.f);
    for (int n = 0; n < rows; n++) {
      float total = 0.f;
      for (int c = 0; c < cols; c++) {
        float& v = ht[n + (size_t)rows * c];
        switch (model_.layer.back().loss_function) {
          case CROSS_ENTROPY_BINARY: v = c % 4 == 3 ? -1.f : (float)(gen() % 2); break;       // every 4th: don't care
          case CROSS_ENTROPY_MULTINOMIAL_DISTRIBUTED: v = ud(gen) + 0.05f; total += v; break;  // normalised below
          default: v = nd(gen); break;
        }
      }
      if (total > 0.f) for (int c = 0; c < cols; c++) ht[n + (size_t)rows * c] /= total;
    }
    t.CopyFromHost(ht.data(), ht.size());
  }

  Fprop(false);
  ComputeDeriv();
  Bprop();                                                    // analytical gradients now in grad_weights of each edge

  std::vector<GradCheckResult> results;
  for (auto& ed : edges_) {
    if (!ed->Config().grad_check) continue;
    EdgeWithWeight* e = dynamic_cast<EdgeWithWeight*>(ed.get());
    if (!e) continue;
    std::vector<float> eps = ed->Config().grad_check_epsilon;
    if (eps.empty()) eps = {1e-2f, 1e-3f, 1e-4f};
    auto check = [&](Matrix& w, Matrix& gw, float epsilon) -> float {     // grad_check.cc:20-61
      int n = std::min<int>(ed->Config().grad_check_num_params, (int)w.GetNumEls());
      std::vector<float> analytical(gw.GetNumEls());
      gw.CopyToHost(analytical.data(), analytical.size());
      float diff_sum = 0; int non_zero = 0;
      for (int i = 0; i < n; i++) {
        const float val = w.ReadValue(i);
        const double e1 = LossAtD(w, i, val + epsilon);
        const double e2 = LossAtD(w, i, val - epsilon);
        w.WriteValue(i, val);
        InvalidateStaging();
        const float numeric = (float)((e1 - e2) / (batch_size_ * 2.0 * epsilon));
        const float diff = analytical[i] - numeric, scale = (analytical[i] + numeric) / 2;
        if (!(scale == 0 && diff == 0)) { diff_sum += std::fabs(diff / scale); non_zero++; }
        if (getenv("CNB_GRADCHECK_VERBOSE"))      // the reference prints this table (grad_check.cc:45-57)
          printf("%s eps %g  analytical %.9f  numerical %.9f  diff %.3e  scaled %.3e\n", e->GetName().c_str(), epsilon,
                 analytical[i], numeric, diff, scale != 0 ? std::fabs(diff / scale) : 0.f);
      }
      return non_zero ? diff_sum / non_zero : 0.f;
    };
    GradCheckResult best{e->GetName(), 0.f, 1e30f, 1e30f};
    for (float ep : eps) {                                     // first epsilon that passes wins (grad_check.cc:43-66)
      GradCheckResult r{e->GetName(), ep, check(e->GetWeight(), e->GetGradWeight(), ep), 0.f};
      r.mean_scaled_diff_b = e->GetBias().GetNumEls() ? check(e->GetBias(), e->GetGradBias(), ep) : 0.f;
      if (std::max(r.mean_scaled_diff_w, r.mean_scaled_diff_b) < std::max(best.mean_scaled_diff_w, best.mean_scaled_diff_b)) best = r;
      if (r.mean_scaled_diff_w < 0.01f && r.mean_scaled_diff_b < 0.01f) break;
    }
    results.push_back(best);
  }
  return results;
}

}  // namespace cnbhost
