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

#ifndef DIVUP
#define DIVUP(x, y) (((x) + (y)-1) / (y))
#endif

namespace cnbhost {

#define HOST_CUDA_CHECK(expr)                                                                         \
  do {                                                                                                \
    cudaError_t _e = (expr);                                                                          \
    if (_e != cudaSuccess) {                                                                          \
      fprintf(stderr, "%s(%d) : CUDA error : %s : %s\n", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      exit(EXIT_FAILURE);                                                                             \
    }                                                                                                 \
  } while (0)

// =================================================================== Layer
Layer::~Layer() { if (labels_) cudaFree(labels_); }

void Layer::AllocateMemory(int batch_size) {               // layer.cc:228-262 (Shape4D convention :257-258)
  const int cols = image_size_y_ * image_size_x_ * image_size_t_ * config_.num_channels;
  state_.AllocateGPUMemory(batch_size, cols);
  state_.SetShape4D(batch_size, image_size_x_, image_size_y_, config_.num_channels * image_size_t_);
  if (!config_.is_input) {
    deriv_.AllocateGPUMemory(batch_size, cols);
    deriv_.SetShape4D(batch_size, image_size_x_, image_size_y_, config_.num_channels * image_size_t_);
  }
  if (config_.dropprob > 0) dropout_mask_.AllocateGPUMemory(batch_size, cols);
  if (config_.is_output) {
    HOST_CUDA_CHECK(cudaMalloc((void**)&labels_, sizeof(int) * batch_size));
    HOST_CUDA_CHECK(cudaMemset(labels_, 0, sizeof(int) * batch_size));
    loss_per_image_.AllocateGPUMemory(batch_size, 1);
  }
}

// `emit`: this call is the last writer of the tensor and the next conv edge reads it as bf16 (see Edge::SetEmitUp)
void Layer::ApplyActivation(bool emit) {
  if (activation_fused_) return;
  switch (config_.activation) {
    case LINEAR: break;
    case RECTIFIED_LINEAR:
      if (emit) convnet_b200_emit_bf16_next();
      state_.ApplyReLU();                                  // LowerBound(0), layer.cc:550
      break;
    case SOFTMAX: state_.ApplySoftmax(); break;
  }
}
void Layer::ApplyDerivativeOfActivation(bool emit) {
  if (deriv_fused_) return;
  if (config_.activation == RECTIFIED_LINEAR) {
    if (emit) convnet_b200_emit_bf16_next();
    deriv_.ApplyDerivOfReLU(state_);
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
  if (dropout_deriv_folded_) { dropout_deriv_folded_ = false; return; }    // the dgrad above already applied 1/(1-p) * [state > 0]
  if (emit) convnet_b200_emit_bf16_next();
  cnb_mult(deriv_.GetDevData(), dropout_mask_.GetDevData(), (long long)deriv_.GetNumEls());
}
void Layer::ComputeDeriv() {
  cnb_softmax_ce_deriv(state_.GetDevData(), labels_, deriv_.GetDevData(), loss_per_image_.GetDevData(),
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
  bool ok = false;
};
NcclApi& nccl() {
  static NcclApi api;
  static bool tried = false;
  if (!tried) {
    tried = true;
    // torch's bundled libnccl.so.2 is already mapped when the launcher imported torch; otherwise the loader path is used
    api.handle = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!api.handle) { fprintf(stderr, "convnet_b200 host: cannot load libnccl.so.2: %s\n", dlerror()); return api; }
#define LOAD(field, sym) api.field = reinterpret_cast<decltype(api.field)>(dlsym(api.handle, sym))
    LOAD(GetUniqueId, "ncclGetUniqueId"); LOAD(CommInitRank, "ncclCommInitRank"); LOAD(CommDestroy, "ncclCommDestroy");
    LOAD(CommInitRankConfig, "ncclCommInitRankConfig");
    LOAD(AllReduce, "ncclAllReduce"); LOAD(Bcast, "ncclBroadcast"); LOAD(GetErrorString, "ncclGetErrorString");
#undef LOAD
    api.ok = api.GetUniqueId && api.CommInitRank && api.AllReduce && api.Bcast;
  }
  return api;
}
#define NCCL_CHECK(expr)                                                                               \
  do {                                                                                                 \
    ncclResult_t _r = (expr);                                                                          \
    if (_r != ncclSuccess) {                                                                           \
      fprintf(stderr, "%s(%d) : NCCL error : %s : %s\n", __FILE__, __LINE__, #expr,                    \
              nccl().GetErrorString ? nccl().GetErrorString(_r) : "?");                                \
      exit(EXIT_FAILURE);                                                                              \
    }                                                                                                  \
  } while (0)
}  // namespace

DataParallelSync::DataParallelSync() {}
DataParallelSync::~DataParallelSync() {
  if (comm_ && nccl().CommDestroy) nccl().CommDestroy((ncclComm_t)comm_);
  if (comm_stream_) cudaStreamDestroy(comm_stream_);
  if (ready_) cudaEventDestroy(ready_);
  if (done_) cudaEventDestroy(done_);
}
bool DataParallelSync::GetUniqueId(char out[128]) {
  if (!nccl().ok) return false;
  ncclUniqueId id;
  static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");
  NCCL_CHECK(nccl().GetUniqueId(&id));
  memcpy(out, &id, 128);
  return true;
}
bool DataParallelSync::Init(int rank, int world, const char idbytes[128]) {
  if (!nccl().ok) return false;
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
  HOST_CUDA_CHECK(cudaStreamCreateWithFlags(&comm_stream_, cudaStreamNonBlocking));
  HOST_CUDA_CHECK(cudaEventCreateWithFlags(&ready_, cudaEventDisableTiming));
  HOST_CUDA_CHECK(cudaEventCreateWithFlags(&done_, cudaEventDisableTiming));
  return true;
}
void DataParallelSync::Broadcast(float* buf, size_t count) {
  if (world_ <= 1) return;
  HOST_CUDA_CHECK(cudaEventRecord(ready_, Matrix::Stream()));
  HOST_CUDA_CHECK(cudaStreamWaitEvent(comm_stream_, ready_, 0));
  NCCL_CHECK(nccl().Bcast(buf, buf, count, ncclFloat, 0, (ncclComm_t)comm_, comm_stream_));
  HOST_CUDA_CHECK(cudaEventRecord(done_, comm_stream_));
  HOST_CUDA_CHECK(cudaStreamWaitEvent(Matrix::Stream(), done_, 0));
}
void DataParallelSync::AllReduceAverageAsync(float* buf, size_t offset, size_t count, cudaStream_t comm) {
  if (world_ <= 1 || count == 0) return;
  NCCL_CHECK(nccl().AllReduce(buf + offset, buf + offset, count, ncclFloat, ncclAvg, (ncclComm_t)comm_, comm));
}

// =================================================================== ConvNet
ConvNet::ConvNet(const ModelConfig& model, int batch_size) : model_(model), batch_size_(batch_size) {
  // BuildNet (convnet.cc:150-270), restricted to chains: edge i connects layer i to layer i+1
  if (model.layer.size() != model.edge.size() + 1) { fprintf(stderr, "ConvNet: model must be a chain\n"); exit(1); }
  for (const LayerConfig& lc : model.layer) layers_.push_back(new Layer(lc));
  for (size_t i = 0; i < model.edge.size(); i++) {
    Edge* e = Edge::ChooseEdgeClass(model.edge[i]);
    e->SetSource(layers_[i]); e->SetDest(layers_[i + 1]);
    e->SetInputChannels(layers_[i]->GetNumChannels());
    e->SetOutputChannels(layers_[i + 1]->GetNumChannels());
    e->SetBatchSize(batch_size);
    edges_.push_back(e);
  }
  // epilogue fusion of the Layer-side ReLU / ReLU' into the neighbouring edges (SURVEY.md 8(f) rank 2)
  const char* nf = getenv("CONVNET_B200_NO_FUSE");
  if (!(nf && nf[0] == '1')) {
    for (size_t i = 0; i < edges_.size(); i++) {
      Layer *src = layers_[i], *dst = layers_[i + 1];
      if (dst->GetActivation() == RECTIFIED_LINEAR) {
        edges_[i]->SetFuseReLU(true);              // honoured only where CanFuseReLU() (checked after SetImageSize below)
      }
      if (!src->IsInput() && src->GetActivation() == RECTIFIED_LINEAR) edges_[i]->SetFuseMask(true);
    }
  }
  // SetImageSize propagation (convnet.cc:226-268)
  const LayerConfig& in = model.layer.front();
  layers_[0]->SetSize(in.image_size_y, in.image_size_x, in.image_size_t);
  for (size_t i = 0; i < edges_.size(); i++) {
    edges_[i]->SetImageSize(layers_[i]->GetSizeY(), layers_[i]->GetSizeX(), layers_[i]->GetSizeT());
    layers_[i + 1]->SetSize(edges_[i]->GetNumModulesY(), edges_[i]->GetNumModulesX(), edges_[i]->GetNumModulesT());
  }
  for (size_t i = 0; i < edges_.size(); i++) {       // settle the fusion flags now that shapes are known
    Edge* e = edges_[i];
    const bool relu = layers_[i + 1]->GetActivation() == RECTIFIED_LINEAR && e->CanFuseReLU() && e->WantsFuseReLU();
    e->SetFuseReLU(relu);
    layers_[i + 1]->SetActivationFused(relu);
    const bool mask = e->CanFuseMask() && e->WantsFuseMask();
    e->SetFuseMask(mask);
    layers_[i]->SetDerivFused(mask);
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
  convnet_b200_reserve_sms(0);
  convnet_b200_bf16_invalidate(nullptr);                     // the buffers go away; a later net may get the same addresses
  for (Edge* e : edges_) delete e;
  for (Layer* l : layers_) delete l;
}

void ConvNet::AllocateMemory() {
  for (Layer* l : layers_) l->AllocateMemory(batch_size_);
  // AllocateEdgeMemory (convnet.cc:272-298): one flat buffer, each edge's slice padded to 128 floats
  size_t total = 0;
  for (Edge* e : edges_) {
    size_t req = e->GetParameterMemoryRequirement();
    edge_offset_.push_back(total);
    edge_size_.push_back(req);
    total += DIVUP(req, (size_t)128) * 128;
  }
  num_params_ = total;
  if (total == 0) total = 128;
  parameters_.AllocateGPUMemory(1, (int)total);
  grad_parameters_.AllocateGPUMemory(1, (int)total);
  history_.AllocateGPUMemory(1, (int)total);
  loss_sum_.AllocateGPUMemory(1, 1);
  for (size_t i = 0; i < edges_.size(); i++) {
    if (edge_size_[i] == 0) continue;
    Matrix p, g, h;
    parameters_.GetSlice(p, (int)edge_offset_[i], (int)(edge_offset_[i] + edge_size_[i]));
    grad_parameters_.GetSlice(g, (int)edge_offset_[i], (int)(edge_offset_[i] + edge_size_[i]));
    history_.GetSlice(h, (int)edge_offset_[i], (int)(edge_offset_[i] + edge_size_[i]));
    edges_[i]->SetMemory(p);
    edges_[i]->SetGradMemory(g);
    edges_[i]->SetHistoryMemory(h);
    edges_[i]->Initialize(model_.seed + 17 * (unsigned)i);
  }
  HOST_CUDA_CHECK(cudaStreamSynchronize(Matrix::Stream()));
  InvalidateStaging();
  HOST_CUDA_CHECK(cudaStreamCreateWithFlags(&side_, cudaStreamNonBlocking));
  HOST_CUDA_CHECK(cudaStreamCreateWithFlags(&opt_, cudaStreamNonBlocking));
  HOST_CUDA_CHECK(cudaEventCreateWithFlags(&ev_opt_, cudaEventDisableTiming));
  HOST_CUDA_CHECK(cudaStreamCreateWithFlags(&comm_, cudaStreamNonBlocking));
  HOST_CUDA_CHECK(cudaEventCreateWithFlags(&ev_comm_, cudaEventDisableTiming));
  HOST_CUDA_CHECK(cudaEventCreateWithFlags(&ev_main_, cudaEventDisableTiming));
  HOST_CUDA_CHECK(cudaEventCreateWithFlags(&ev_side_, cudaEventDisableTiming));
  SetBucketFloats((size_t)8 << 20);
  static const bool no_lane = getenv("CONVNET_B200_NO_SIDE_BIAS_GRAD") && getenv("CONVNET_B200_NO_SIDE_BIAS_GRAD")[0] == '1';
  if (!no_lane) {
    lane_.stream = side_;
    HOST_CUDA_CHECK(cudaEventCreateWithFlags(&lane_.ready, cudaEventDisableTiming));
    for (Edge* e : edges_)
      if (EdgeWithWeight* w = dynamic_cast<EdgeWithWeight*>(e)) w->SetSideLane(&lane_);
  }
}

void ConvNet::Fprop(bool train) {                            // convnet.cc:377-388
  const bool bf16 = convnet_b200_get_conv_precision() == 2;
  dropout_active_ = train;
  for (size_t i = 1; i < layers_.size(); i++) {
    Layer* l = layers_[i];
    Edge* e = edges_[i - 1];
    // bf16 mode: whoever writes this layer's state LAST (dropout, else a separate activation pass, else the edge's own
    // kernel) also writes the bf16 copy the next conv edge multiplies with
    const bool want = bf16 && i < edges_.size() && edges_[i]->WantsBf16Input();
    const bool act_pass = l->HasSeparateActivationPass();
    // dropout inside the edge's epilogue (no mask tensor) when the backward pass will not need the mask either
    static const bool no_fuse_drop = getenv("CONVNET_B200_NO_FUSED_DROPOUT") && getenv("CONVNET_B200_NO_FUSED_DROPOUT")[0] == '1';
    const bool fuse_drop = train && l->HasDropout() && !no_fuse_drop && !act_pass && e->CanFuseDropout() && DropoutFolds(i);
    if (fuse_drop) e->SetDropoutRequest(l->DropoutProb(), l->DropoutScale(), l->DropoutSeed(step_, dropout_salt_));
    const bool drop = train && l->HasDropout() && !fuse_drop;
    e->SetEmitUp(want && !drop && !act_pass);
    e->ComputeUp(layers_[i - 1]->GetState(), l->GetState(), /*overwrite=*/true, train);
    l->ApplyActivation(want && !drop && act_pass);
    if (!fuse_drop) l->ApplyDropout(train, step_, dropout_salt_, want && drop);
  }
}

bool ConvNet::DropoutFolds(size_t i) const {
  static const bool no_fold = getenv("CONVNET_B200_NO_DROPOUT_FOLD") && getenv("CONVNET_B200_NO_DROPOUT_FOLD")[0] == '1';
  if (no_fold || i == 0 || i >= edges_.size()) return false;        // edges_[i]: the edge whose ComputeDown writes layers_[i]'s derivative
  const Layer* l = layers_[i];
  return l->HasDropout() && l->GetActivation() == RECTIFIED_LINEAR && !l->HasSeparateDerivPass() && edges_[i]->CanScaleDeriv();
}

void ConvNet::ComputeDeriv() { OutputLayer().ComputeDeriv(); }

float ConvNet::GetLoss() {                                   // CrossEntropyMultinomial::GetLoss: sum over the batch
  Layer& out = OutputLayer();
  cnb_softmax_ce_deriv(out.GetState().GetDevData(), out.GetLabels(), out.GetDeriv().GetDevData(),
                       out.GetLossPerImage(), batch_size_, out.GetState().GetCols());
  cnb_sum(out.GetLossPerImage(), loss_sum_.GetDevData(), batch_size_);
  return loss_sum_.ReadValue(0);
}

void ConvNet::Bprop() {                                      // convnet.cc:390-405 + 362-375
  const bool bf16 = convnet_b200_get_conv_precision() == 2;
  for (int i = (int)layers_.size() - 1; i >= 1; i--) {
    Layer* out = layers_[i];
    Layer* in = layers_[i - 1];
    Edge* e = edges_[i - 1];
    // bf16 mode: the last writer of a derivative tensor (ReLU' pass, else dropout mask, else the ComputeDown of the edge
    // above) leaves the bf16 copy the edge below reads in its wgrad and dgrad
    // (the reference runs these two at the top of the NEXT loop iteration, i.e. before this layer's edges)
    if (!out->IsOutput()) {
      const bool want_out = bf16 && e->WantsBf16Deriv();
      const bool act_pass = out->HasSeparateDerivPass();
      out->ApplyDerivativeofDropout(want_out && !act_pass);
      out->ApplyDerivativeOfActivation(want_out && act_pass);
    }
    e->ComputeOuter(in->GetState(), out->GetDeriv());
    // data parallel: ship every bucket whose last gradient just became final (side stream, overlaps the rest of bprop)
    if (dp_ && dp_->world() > 1)
      for (size_t bi = 0; bi < buckets_.size(); bi++) {
        const Bucket& b = buckets_[bi];
        if (b.trigger != i - 1) continue;
        if (!comm_pending_) convnet_b200_reserve_sms(dp_->reserved_sms());
        // the bucket's gradients: weight gradients on the main stream, bias gradients (column sums) on the side stream
        HOST_CUDA_CHECK(cudaEventRecord(ev_main_, Matrix::Stream()));
        HOST_CUDA_CHECK(cudaStreamWaitEvent(comm_, ev_main_, 0));
        HOST_CUDA_CHECK(cudaEventRecord(ev_side_, side_));
        HOST_CUDA_CHECK(cudaStreamWaitEvent(comm_, ev_side_, 0));
        if (trace_.on) HOST_CUDA_CHECK(cudaEventRecord(trace_.c0[bi], comm_));
        dp_->AllReduceAverageAsync(grad_parameters_.GetDevData(), b.lo, b.hi - b.lo, comm_);
        HOST_CUDA_CHECK(cudaEventRecord(ev_reduced_[bi], comm_));
        if (trace_.on) HOST_CUDA_CHECK(cudaEventRecord(trace_.c1[bi], comm_));
        comm_pending_ = true;
      }
    if (!in->IsInput()) {
      const bool want_in = bf16 && i >= 2 && edges_[i - 2]->WantsBf16Deriv();
      // dropout derivative of a ReLU layer = one factor on the kept units, which the fused mask already selects
      const bool fold = dropout_active_ && in->HasDropout() && DropoutFolds((size_t)i - 1);
      if (fold) { e->SetDerivScale(in->DropoutScale()); in->SetDropoutDerivFolded(true); }
      const bool drop_pass = in->HasDropout() && !fold;
      e->SetEmitDown(want_in && !drop_pass && !in->HasSeparateDerivPass());
      // the kernel that writes in's derivative LAST can also sum its channels: that is the bias gradient of the edge below
      static const bool no_bg = getenv("CONVNET_B200_NO_FUSED_BIAS_GRAD") && getenv("CONVNET_B200_NO_FUSED_BIAS_GRAD")[0] == '1';
      if (!no_bg && i >= 2 && e->CanProduceBiasGrad() && !drop_pass && !in->HasSeparateDerivPass()) {
        Edge::BiasGradTarget t;
        if (edges_[i - 2]->OfferFusedBiasGrad(&t)) e->SetBiasGradRequest(t);
      }
      e->ComputeDown(out->GetDeriv(), in->GetState(), out->GetState(), in->GetDeriv(), /*overwrite=*/true);
    }
    // the optimizer step of a bucket follows its all-reduce on the side stream once its edges are done with the weights
    if (eager_update_)
      for (size_t bi = 0; bi < buckets_.size(); bi++)
        if (buckets_[bi].trigger == i - 1) {
          if (dp_ && dp_->world() > 1) HOST_CUDA_CHECK(cudaStreamWaitEvent(opt_, ev_reduced_[bi], 0));   // SGD after its all-reduce
          IssueBucketUpdate(buckets_[bi]);
          if (trace_.on) HOST_CUDA_CHECK(cudaEventRecord(trace_.s1[bi], opt_));
        }
  }
  if (!eager_update_ && !(dp_ && dp_->world() > 1)) WaitSide();   // stand-alone Bprop: the gradients are complete on return
}

// the SGD step of one bucket on the optimizer stream, after (events) that bucket's all-reduce, the bias-gradient sums
// queued on the side stream so far, and the compute stream's last read of the bucket's weights in this step.  Its own
// stream: an all-reduce waits for the side stream's bias gradients, and must not queue behind an earlier bucket's SGD step
void ConvNet::IssueBucketUpdate(const Bucket& b) {
  std::vector<CnbSgdTensor> tensors;
  for (int i = b.trigger; i <= b.last; i++)
    if (EdgeWithWeight* w = dynamic_cast<EdgeWithWeight*>(edges_[i])) w->AppendSgdTensors(tensors);
  if (tensors.empty()) return;
  HOST_CUDA_CHECK(cudaEventRecord(ev_main_, Matrix::Stream()));
  HOST_CUDA_CHECK(cudaStreamWaitEvent(opt_, ev_main_, 0));
  HOST_CUDA_CHECK(cudaEventRecord(ev_side_, side_));
  HOST_CUDA_CHECK(cudaStreamWaitEvent(opt_, ev_side_, 0));
  void* main_stream = convnet_b200_get_stream();
  convnet_b200_set_stream(opt_);
  cnb_sgd_momentum_multi(tensors.data(), (int)tensors.size());
  // what the next step's dgrad derives from these weights alone (bf16 filter banks): rebuilt here, behind the update
  static const bool no_prestage = getenv("CONVNET_B200_NO_PRESTAGE") && getenv("CONVNET_B200_NO_PRESTAGE")[0] == '1';
  if (!no_prestage)
    for (int i = b.trigger; i <= b.last; i++)
      if (EdgeWithWeight* w = dynamic_cast<EdgeWithWeight*>(edges_[i])) w->PrestageDown();
  convnet_b200_set_stream(main_stream);
  opt_pending_ = true;
}
void ConvNet::WaitSide() {
  if (lane_.used) { side_pending_ = true; lane_.used = false; }
  if (comm_pending_) {                                       // every all-reduce of the step (the SGD steps on side_ wait for theirs too)
    HOST_CUDA_CHECK(cudaEventRecord(ev_comm_, comm_));
    HOST_CUDA_CHECK(cudaStreamWaitEvent(Matrix::Stream(), ev_comm_, 0));
    comm_pending_ = false;
    convnet_b200_reserve_sms(0);
  }
  if (opt_pending_) {
    HOST_CUDA_CHECK(cudaEventRecord(ev_opt_, opt_));
    HOST_CUDA_CHECK(cudaStreamWaitEvent(Matrix::Stream(), ev_opt_, 0));
    opt_pending_ = false;
  }
  if (!side_pending_) return;
  HOST_CUDA_CHECK(cudaEventRecord(ev_side_, side_));
  HOST_CUDA_CHECK(cudaStreamWaitEvent(Matrix::Stream(), ev_side_, 0));
  side_pending_ = false;
}

void ConvNet::UpdateWeights() {                              // convnet.cc:440-450
  WaitSide();                                                // replaces Accumulate + Broadcast (MPI through host memory)
  if (updated_in_bprop_) { updated_in_bprop_ = false; return; }        // TrainOneBatch: every bucket was updated on the side stream
  // one multi-tensor SGD launch for every weight and bias matrix of the net (the reference loops edges: optimizer.cc:174-200)
  std::vector<CnbSgdTensor> tensors;
  for (Edge* e : edges_)
    if (EdgeWithWeight* w = dynamic_cast<EdgeWithWeight*>(e)) w->AppendSgdTensors(tensors);
  cnb_sgd_momentum_multi(tensors.data(), (int)tensors.size());
}

void ConvNet::TrainOneBatch(float* loss_out) {               // convnet.cc:475-485 (GetBatch is the caller's H2D copy)
  if (trace_.on) HOST_CUDA_CHECK(cudaEventRecord(trace_.t0, Matrix::Stream()));
  Fprop(true);
  ComputeDeriv();
  if (trace_.on) HOST_CUDA_CHECK(cudaEventRecord(trace_.fwd, Matrix::Stream()));
  if (loss_out) {                                            // GetLoss: one scalar D2H per step, like the reference
    cnb_sum(OutputLayer().GetLossPerImage(), loss_sum_.GetDevData(), batch_size_);
  }
  static const bool no_eager = getenv("CONVNET_B200_NO_EAGER_UPDATE") && getenv("CONVNET_B200_NO_EAGER_UPDATE")[0] == '1';
  eager_update_ = !no_eager;
  Bprop();
  if (trace_.on) HOST_CUDA_CHECK(cudaEventRecord(trace_.bwd, Matrix::Stream()));
  updated_in_bprop_ = eager_update_;
  eager_update_ = false;
  UpdateWeights();
  if (trace_.on) HOST_CUDA_CHECK(cudaEventRecord(trace_.end, Matrix::Stream()));
  if (loss_out) *loss_out = loss_sum_.ReadValue(0);
  step_++;
}

std::vector<float> ConvNet::TraceStep() {
  auto make = [](cudaEvent_t* e) { if (!*e) HOST_CUDA_CHECK(cudaEventCreate(e)); };
  make(&trace_.t0); make(&trace_.fwd); make(&trace_.bwd); make(&trace_.end);
  for (std::vector<cudaEvent_t>* v : {&trace_.c0, &trace_.c1, &trace_.s1})
    while (v->size() < buckets_.size()) { cudaEvent_t e = nullptr; make(&e); v->push_back(e); }
  HOST_CUDA_CHECK(cudaStreamSynchronize(Matrix::Stream()));
  trace_.on = true;
  TrainOneBatch(nullptr);
  trace_.on = false;
  HOST_CUDA_CHECK(cudaStreamSynchronize(Matrix::Stream()));
  HOST_CUDA_CHECK(cudaStreamSynchronize(side_));
  HOST_CUDA_CHECK(cudaStreamSynchronize(opt_));
  HOST_CUDA_CHECK(cudaStreamSynchronize(comm_));
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
  dropout_salt_ = ((unsigned long long)model_.seed * 0xA24BAED4963EE407ULL) ^
                  ((unsigned long long)((dp ? dp->rank() : 0) + 1) * 0xD1B54A32D192ED03ULL);
  SetBucketFloats(bucket_floats);
}
void ConvNet::SetBucketFloats(size_t bucket_floats) {
  buckets_ = PlanBuckets(edge_offset_, edge_size_, bucket_floats);
  while (ev_reduced_.size() < buckets_.size()) {
    cudaEvent_t e;
    HOST_CUDA_CHECK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    ev_reduced_.push_back(e);
  }
}
void ConvNet::BroadcastParameters() {
  if (dp_) dp_->Broadcast(parameters_.GetDevData(), parameters_.GetNumEls());
  InvalidateStaging();
}

double ConvNet::FlopsFprop() const {
  double f = 0;
  for (Edge* e : edges_) f += e->FlopsUp();
  return f;
}
double ConvNet::FlopsTrainStep() const {                     // BASELINE.md §2c: 3x fprop minus the dgrad into the input layer
  double f = 0;
  for (size_t i = 0; i < edges_.size(); i++) f += edges_[i]->FlopsUp() * (i == 0 ? 2.0 : 3.0);
  return f;
}

// =================================================================== GradChecker (src/grad_check.cc)
float GradChecker::LossAt(Matrix& w, size_t index, float value) { return (float)LossAtD(w, index, value); }

double GradChecker::LossAtD(Matrix& w, size_t index, float value) {
  w.WriteValue(index, value);
  InvalidateStaging();
  Fprop(false);
  // per-image cross-entropy on the device, summed in double on the host: the finite difference of two ~O(batch)
  // losses must not lose the 1e-3-sized signal to fp32 summation noise
  Layer& out = OutputLayer();
  cnb_softmax_ce_deriv(out.GetState().GetDevData(), out.GetLabels(), out.GetDeriv().GetDevData(), out.GetLossPerImage(),
                       batch_size_, out.GetState().GetCols());
  std::vector<float> h(batch_size_);
  HOST_CUDA_CHECK(cudaMemcpyAsync(h.data(), out.GetLossPerImage(), sizeof(float) * batch_size_, cudaMemcpyDeviceToHost, Matrix::Stream()));
  HOST_CUDA_CHECK(cudaStreamSynchronize(Matrix::Stream()));
  double s = 0;
  for (float v : h) s += v;
  return s;
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
  HOST_CUDA_CHECK(cudaMemcpy(OutputLayer().GetLabels(), hl.data(), sizeof(int) * batch_size_, cudaMemcpyHostToDevice));

  Fprop(false);
  ComputeDeriv();
  Bprop();                                                    // analytical gradients now in grad_weights of each edge

  std::vector<GradCheckResult> results;
  for (Edge* ed : edges_) {
    if (!ed->Config().grad_check) continue;
    EdgeWithWeight* e = dynamic_cast<EdgeWithWeight*>(ed);
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
