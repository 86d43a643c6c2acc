// capi.cc — plain C doors onto the host C++ (ConvNet / GradChecker / DataParallelSync) for ctypes.
//
// Every entry that can fail runs its body in Guard and reports one way: a status (0, or a count where the entry returns
// one), -1 when the library refused (an invalid_argument, a logic_error, a file it cannot read or write), -2 when a CUDA
// or NCCL call failed (DeviceError), and NULL for the entries that create an object.  The reason is in cnb_last_error()
// and on stderr as "convnet_b200 host: <reason>"; cnb_last_status() tells a NULL's -1 from its -2.  After a -2 in the
// middle of a step the net's state is undefined: the only safe call left on it is cnb_net_destroy.  The entries that only
// read fields cannot fail and return their value.
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <stdexcept>
#include <string>

#include "convnet.h"
#include "data.h"

using namespace cnbhost;

#define API extern "C" __attribute__((visibility("default")))

struct NetHandle {
  ConvNet* net = nullptr;
  GradChecker* checker = nullptr;
  DataParallelSync* dp = nullptr;
  std::vector<TrainEvent> events;                          // of the last cnb_net_train
};

static std::string g_last_error;
static int g_last_status = 0;
// the reason and the status (-1 or -2) of the last failure
API const char* cnb_last_error() { return g_last_error.c_str(); }
API int cnb_last_status() { return g_last_status; }
static int Fail(const std::exception& e, int status) {
  g_last_error = e.what();
  g_last_status = status;
  fprintf(stderr, "convnet_b200 host: %s\n", e.what());
  return status;
}
// runs f: 0, or the status of what it threw (-2 a DeviceError, -1 any other exception)
template <class F>
static int Guard(F f) {
  try {
    f();
    return 0;
  } catch (const DeviceError& e) {
    return Fail(e, -2);
  } catch (const std::exception& e) {
    return Fail(e, -1);
  }
}

API void cnb_net_destroy(void* p) {
  NetHandle* h = (NetHandle*)p;
  delete h->net; delete h->dp; delete h;
}
// a handle on the ConvNet (GradChecker when grad_checker) of a built-in name or model file, with its seed replaced unless
// `seed` is NULL, and its device memory allocated when `allocate` (else its parameters only planned).  NULL: an unknown
// name, a model that cannot be read or run, or memory that cannot be set up (the checkpoints of PRETRAINED edges, the
// device)
static void* Open(const char* model, int batch, const unsigned* seed, bool grad_checker, bool allocate) {
  NetHandle* h = new NetHandle;
  if (Guard([&] {
        ModelConfig m = BuildModel(model);
        if (seed) m.seed = *seed;
        if (grad_checker) h->net = h->checker = new GradChecker(m, batch);
        else h->net = new ConvNet(m, batch);
        if (allocate) h->net->AllocateMemory();
        else h->net->PlanParameters();
      })) {
    cnb_net_destroy(h);
    return nullptr;
  }
  return h;
}
// a host-only handle: the net built and its parameters planned, nothing allocated on the device.  The cnb_net_* calls that
// read no device memory describe the model through it: edges, layers, the parameter layout, the fusion plan, FLOPs, the
// trained tensors' optimizers, and the model-level settings below (cnb_net_model_text ... cnb_net_train_dry_run)
API void* cnb_model_open(const char* model, int batch) { return Open(model, batch, nullptr, false, false); }
// a net to run
API void* cnb_net_create(const char* model, int batch_size, unsigned seed, int grad_checker) {
  return Open(model, batch_size, &seed, grad_checker != 0, true);
}
API long long cnb_net_num_params(void* p) { return (long long)((NetHandle*)p)->net->NumParameters(); }
API int cnb_net_num_edges(void* p) { return (int)((NetHandle*)p)->net->Edges().size(); }
API const char* cnb_net_edge_name(void* p, int i) { return ((NetHandle*)p)->net->Edges()[i]->GetName().c_str(); }
API double cnb_net_edge_flops(void* p, int i) { return ((NetHandle*)p)->net->Edges()[i]->FlopsUp(); }
// where edge i's parameters begin in the flat buffers (a tied edge: its owner's), and how many floats it owns (0 if tied)
API long long cnb_net_edge_offset(void* p, int i) { return (long long)((NetHandle*)p)->net->ParamOffset(i); }
API long long cnb_net_edge_size(void* p, int i) { return (long long)((NetHandle*)p)->net->Edges()[i]->GetParameterMemoryRequirement(); }
// where the slice placed at edge position i begins (ConvNet::EdgeOffsets: a tie group's slice sits at its lowest edge)
API long long cnb_net_edge_slice(void* p, int i) { return (long long)((NetHandle*)p)->net->EdgeOffsets()[i]; }
// the epilogue fusion ConvNet::PlanFusion decided for edge i: *up_act / *down_act the CNB_ACT_* code ComputeUp applies and
// the one whose derivative ComputeDown applies; returns the Edge::FusionPlan flags (bit 0 dropout_up, 1 scale_down,
// 2 sums_bias_below, 3 offers_bias_grad)
API int cnb_net_edge_fusion(void* p, int i, int* up_act, int* down_act) {
  const Edge::FusionPlan& f = ((NetHandle*)p)->net->Edges()[i]->Plan();
  *up_act = f.up_act; *down_act = f.down_act;
  return f.dropout_up | f.scale_down << 1 | f.sums_bias_below << 2 | f.offers_bias_grad << 3;
}
// the passes left to layer i after fusion: bit 0 a separate activation pass, bit 1 a separate derivative pass
API int cnb_net_layer_passes(void* p, int i) {
  const Layer& l = *((NetHandle*)p)->net->Layers()[i];
  return l.HasSeparateActivationPass() | l.HasSeparateDerivPass() << 1;
}
// the edge whose parameters edge i runs with ("" when untied)
API const char* cnb_net_edge_tied_to(void* p, int i) { return ((NetHandle*)p)->net->Edges()[i]->Config().tied_to.c_str(); }
// the frozen edges are [0, n) (ConvNet::NumFrozenEdges); their parameters the prefix [0, *trained_offset) of the buffers
API int cnb_net_frozen_edges(void* p, long long* trained_offset) {
  *trained_offset = (long long)((NetHandle*)p)->net->TrainedOffset();
  return ((NetHandle*)p)->net->NumFrozenEdges();
}
API double cnb_net_flops_fprop(void* p) { return ((NetHandle*)p)->net->FlopsFprop(); }
API double cnb_net_flops_train(void* p) { return ((NetHandle*)p)->net->FlopsTrainStep(); }
API float* cnb_net_input(void* p) { return ((NetHandle*)p)->net->InputLayer().GetState().GetDevData(); }
API long long cnb_net_input_floats(void* p) { return (long long)((NetHandle*)p)->net->InputLayer().GetState().GetNumEls(); }
API int* cnb_net_labels(void* p) { return ((NetHandle*)p)->net->OutputLayer().GetLabels(); }
API float* cnb_net_output(void* p) { return ((NetHandle*)p)->net->OutputLayer().GetState().GetDevData(); }
API int cnb_net_num_classes(void* p) { return ((NetHandle*)p)->net->OutputLayer().GetState().GetCols(); }
// the caller may write through this pointer: staged bf16 copies of the weights are dropped
API float* cnb_net_params(void* p) { ((NetHandle*)p)->net->InvalidateStaging(); return ((NetHandle*)p)->net->Parameters().GetDevData(); }
API float* cnb_net_grads(void* p) { return ((NetHandle*)p)->net->GradParameters().GetDevData(); }
// the momentum history (laid out like the parameters); a write through it is the caller's
API float* cnb_net_history(void* p) { return ((NetHandle*)p)->net->History().GetDevData(); }
API float* cnb_net_layer_state(void* p, int i) { return ((NetHandle*)p)->net->Layers()[i]->GetState().GetDevData(); }
// the derivative of layer i's state after bprop (laid out like its state); NULL for the input layer
API float* cnb_net_layer_deriv(void* p, int i) { return ((NetHandle*)p)->net->Layers()[i]->GetDeriv().GetDevData(); }
API long long cnb_net_layer_floats(void* p, int i) { return (long long)((NetHandle*)p)->net->Layers()[i]->GetState().GetNumEls(); }
API int cnb_net_num_layers(void* p) { return (int)((NetHandle*)p)->net->Layers().size(); }
API float* cnb_net_device_loss(void* p) { return ((NetHandle*)p)->net->DeviceLoss(); }
// the seed of the dropout mask the next training-mode Fprop draws for layer i (0: the layer has no dropout)
API unsigned long long cnb_net_dropout_seed(void* p, int i) { return ((NetHandle*)p)->net->NextDropoutSeed((size_t)i); }

API int cnb_net_fprop(void* p, int train) { return Guard([&] { ((NetHandle*)p)->net->Fprop(train != 0); }); }
API int cnb_net_bprop(void* p) {
  return Guard([&] { ((NetHandle*)p)->net->ComputeDeriv(); ((NetHandle*)p)->net->Bprop(); });
}
API int cnb_net_update(void* p) { return Guard([&] { ((NetHandle*)p)->net->UpdateWeights(); }); }
API void cnb_net_reduce_learning_rate(void* p, float factor) { ((NetHandle*)p)->net->ReduceLearningRate(factor); }

// ---- optimizer settings (edge.h OptimizerConfig: proto Optimizer, SGD fields) of one trained tensor, named as its
// checkpoint records: "<edge>:weight", "<edge>:bias", "<layer>:gamma", "<layer>:beta" (ConvNet::Tensors)
static TrainedTensor* Tensor(void* p, const char* name) {
  for (TrainedTensor& t : ((NetHandle*)p)->net->Tensors())
    if (t.name == name) return &t;
  return nullptr;
}
// replaces the settings of one optimizer (its step count and momentum history stay).  Refused: no such tensor, or a
// config this tensor cannot train with (OptimizerConfigError; BnOptimizerConfigError for gamma / beta)
API int cnb_net_set_optimizer(void* p, const char* tensor, const OptimizerConfig* c) {
  return Guard([&] {
    TrainedTensor* t = Tensor(p, tensor);
    if (!t) throw std::invalid_argument(std::string("no trained tensor '") + tensor + "'");
    if (const char* err = t->ConfigError(*c)) throw std::invalid_argument(std::string(t->name) + ": " + err);
    ((NetHandle*)p)->net->SetOptimizer(*t, *c);
  });
}
// the adaptive optimizer state (cnb_net_num_params floats, carved like the parameters); NULL while no optimizer of the
// net is ADAGRAD_SGD or RMSPROP_SGD
API float* cnb_net_adaptive_state(void* p) { return ((NetHandle*)p)->net->AdaptiveState(); }
// the step count of one optimizer, the (epsilon, momentum) its next update uses and, unless `config` is NULL, its
// settings.  Returns the tensor's floats (0: the bias of a has_no_bias edge), -1 no such tensor
API long long cnb_net_get_optimizer_state(void* p, const char* tensor, long long* step, float* epsilon, float* momentum,
                                          OptimizerConfig* config) {
  const TrainedTensor* t = Tensor(p, tensor);
  if (!t) return -1;
  *step = t->step;
  OptimizerSchedule(t->opt, *step, epsilon, momentum);
  if (config) *config = t->opt;
  return t->n;
}
// pure host logic: (epsilon, momentum) of the update after `step` earlier ones.  Refused: a config OptimizerConfigError
// objects to
API int cnb_optimizer_schedule(const OptimizerConfig* c, long long step, float* epsilon, float* momentum) {
  return Guard([&] {
    if (const char* err = OptimizerConfigError(*c)) throw std::invalid_argument(err);
    OptimizerSchedule(*c, step, epsilon, momentum);
  });
}

// ---- batch normalisation (convnet.h Layer).  layer: index into the chain (0 = input).  which: 0 gamma, 1 beta.
static Layer* BnLayer(void* p, int layer) {
  auto& l = ((NetHandle*)p)->net->Layers();
  return layer >= 0 && layer < (int)l.size() && l[layer]->BatchNormalize() ? l[layer].get() : nullptr;
}
API const char* cnb_net_layer_name(void* p, int i) { return ((NetHandle*)p)->net->Layers()[i]->GetName().c_str(); }
API int cnb_net_layer_channels(void* p, int i) { return ((NetHandle*)p)->net->Layers()[i]->GetNumChannels(); }
// the running-average factor and the variance epsilon of layer i's batch normalisation (the model's, used or not)
API void cnb_net_layer_bn(void* p, int i, float* bn_f, float* bn_epsilon) {
  const LayerConfig& l = ((NetHandle*)p)->net->Model().layer[i];
  *bn_f = l.bn_f; *bn_epsilon = l.bn_epsilon;
}
// offset of the layer's [gamma | beta] (2 x channels floats) in the flat parameter / gradient buffers; -1: not batch-normalised
API long long cnb_net_bn_offset(void* p, int layer) { return BnLayer(p, layer) ? ((NetHandle*)p)->net->BnOffsets()[layer] : -1; }
// device vector of `channels` floats: which 0 running mean, 1 running sigma, 2 batch mean, 3 batch sigma (of the last
// training-mode forward pass); NULL: not batch-normalised
API float* cnb_net_bn_stat(void* p, int layer, int which) {
  Layer* l = BnLayer(p, layer);
  return l && which >= 0 && which < 4 ? l->BnStat(which) : nullptr;
}
// pure host logic: 0 if `c` can train gamma / beta, refused if not
API int cnb_bn_optimizer_check(const OptimizerConfig* c) {
  return Guard([&] {
    if (const char* err = BnOptimizerConfigError(*c)) throw std::invalid_argument(err);
  });
}

// the output layer's float targets ([batch x state columns], column-major, written by the caller); NULL / 0 for an output
// layer trained on labels (cnb_net_labels)
API float* cnb_net_targets(void* p) { return ((NetHandle*)p)->net->OutputLayer().GetTargets().GetDevData(); }
API long long cnb_net_targets_floats(void* p) { return (long long)((NetHandle*)p)->net->OutputLayer().GetTargets().GetNumEls(); }
// *out: loss_function_weight * the batch's loss (ConvNet::GetLoss) / the summed performance metric (GetPerformanceMetric)
API int cnb_net_loss(void* p, float* out) { return Guard([&] { *out = ((NetHandle*)p)->net->GetLoss(); }); }
API int cnb_net_metric(void* p, float* out) { return Guard([&] { *out = ((NetHandle*)p)->net->GetPerformanceMetric(); }); }
// the model's output layer.  *activation: the Activation enum of convnet.h; *loss / *metric: proto LossFunction numbers;
// *labels: 1 trained on integer labels, 0 on float targets
API void cnb_net_output_layer(void* p, int* activation, int* loss, int* metric, float* weight, int* labels) {
  const LayerConfig& l = ((NetHandle*)p)->net->Model().layer.back();
  *activation = l.activation; *loss = l.loss_function; *metric = l.performance_metric; *weight = l.loss_function_weight;
  *labels = TakesLabels(l.activation) ? 1 : 0;
}
// one training step; *loss (may be NULL) receives the batch's loss as cnb_net_loss gives it (one scalar D2H)
API int cnb_net_train_step(void* p, float* loss) { return Guard([&] { ((NetHandle*)p)->net->TrainOneBatch(loss); }); }
// one traced training step (ConvNet::TraceStep); returns the number of floats the full record has, writes min(cap, that)
API int cnb_net_trace_step(void* p, float* out, int cap) {
  std::vector<float> t;
  const int rc = Guard([&] { t = ((NetHandle*)p)->net->TraceStep(); });
  for (int i = 0; i < cap && i < (int)t.size(); i++) out[i] = t[i];
  return rc ? rc : (int)t.size();
}

// data parallel: rank 0 calls cnb_dp_unique_id, the launcher broadcasts the 128 bytes, every rank calls cnb_net_dp_init
API int cnb_dp_unique_id(char* out128) { return Guard([&] { DataParallelSync::GetUniqueId(out128); }); }
API int cnb_net_dp_init(void* p, int rank, int world, const char* id128, long long bucket_floats) {
  NetHandle* h = (NetHandle*)p;
  return Guard([&] {
    h->dp = new DataParallelSync();
    h->dp->Init(rank, world, id128);
    h->net->SetDataParallel(h->dp, (size_t)bucket_floats);
    h->net->BroadcastParameters();
  });
}

// grad check: fills up to `cap` results; returns the number of checked edges.  Refused on a net not created as a checker
API int cnb_net_grad_check(void* p, unsigned seed, int cap, char* names /*cap x 64*/, float* eps, float* diff_w, float* diff_b) {
  NetHandle* h = (NetHandle*)p;
  std::vector<GradCheckResult> r;
  const int rc = Guard([&] {
    if (!h->checker) throw std::invalid_argument("grad_check: the net was not created as a grad checker");
    r = h->checker->Run(seed);
  });
  if (rc) return rc;
  int n = 0;
  for (const GradCheckResult& g : r) {
    if (n >= cap) break;
    strncpy(names + 64 * n, g.edge.c_str(), 63); names[64 * n + 63] = 0;
    eps[n] = g.epsilon; diff_w[n] = g.mean_scaled_diff_w; diff_b[n] = g.mean_scaled_diff_b;
    n++;
  }
  return n;
}

// the gradient-bucket plan (pure host logic; testable without a GPU). Returns the number of buckets (<= cap).
API int cnb_plan_buckets(int n_edges, const long long* offsets, const long long* sizes, long long bucket_floats, int cap,
                         long long* lo, long long* hi, int* trigger) {
  std::vector<size_t> off(offsets, offsets + n_edges), sz(sizes, sizes + n_edges);
  std::vector<Bucket> b = PlanBuckets(off, sz, (size_t)bucket_floats);
  int n = 0;
  for (const Bucket& k : b) { if (n >= cap) break; lo[n] = (long long)k.lo; hi[n] = (long long)k.hi; trigger[n] = k.trigger; n++; }
  return n;
}
// the model as a config::Model text proto (ModelText).  Returns its length in bytes and writes up to cap - 1 of them
// and a terminating NUL into buf
API long long cnb_net_model_text(void* p, char* buf, long long cap) {
  const std::string t = ModelText(((NetHandle*)p)->net->Model());
  if (cap > 0) {
    const size_t n = std::min((size_t)(cap - 1), t.size());
    memcpy(buf, t.data(), n);
    buf[n] = 0;
  }
  return (long long)t.size();
}

// the initial weights of edge `edge` under RNG seed `seed` (EdgeWithWeight::InitialWeights; the net seeds edge i with its
// seed + 17 i), or a PRETRAINED edge's weights from its checkpoint.  Returns their number (writes up to `cap`), 0 for an
// edge out of range or without parameters of its own; refused: an unreadable checkpoint
API long long cnb_net_initial_weights(void* p, int edge, unsigned seed, float* out, long long cap) {
  ConvNet* net = ((NetHandle*)p)->net;
  EdgeWithWeight* e = edge >= 0 && edge < (int)net->Edges().size() ? dynamic_cast<EdgeWithWeight*>(net->Edges()[edge].get()) : nullptr;
  if (!e || e->Tied()) return 0;
  std::vector<float> w;
  if (const int rc = Guard([&] {
        w = e->Config().initialization == PRETRAINED ? PretrainedWeights(e->Config(), e->WeightCount()) : e->InitialWeights(seed);
      }))
    return rc;
  const long long n = (long long)w.size();
  if (cap > 0) memcpy(out, w.data(), sizeof(float) * (size_t)std::min(n, cap));
  return n;
}

// ---- checkpoints and Polyak averaging (checkpoint.cc)
API int cnb_net_save(void* p, const char* path) { return Guard([&] { ((NetHandle*)p)->net->Save(path); }); }
API int cnb_net_load(void* p, const char* path) { return Guard([&] { ((NetHandle*)p)->net->Load(path); }); }
API long long cnb_net_iteration(void* p) { return (long long)((NetHandle*)p)->net->Iteration(); }
API int cnb_net_polyak_insert(void* p) { return Guard([&] { ((NetHandle*)p)->net->InsertPolyak(); }); }
API int cnb_net_load_polyak_weights(void* p) { return Guard([&] { ((NetHandle*)p)->net->LoadPolyakWeights(); }); }
API int cnb_net_load_current_weights(void* p) { return Guard([&] { ((NetHandle*)p)->net->LoadCurrentWeights(); }); }
API int cnb_net_polyak_count(void* p) { return ((NetHandle*)p)->net->PolyakCount(); }
// the model's Polyak settings.  1 Polyak on, 0 off
API int cnb_net_polyak(void* p, int* after, int* queue_size, int* validate_after, int* save_after) {
  const ModelConfig& m = ((NetHandle*)p)->net->Model();
  *after = m.polyak_after; *queue_size = m.polyak_queue_size; *validate_after = m.validate_after; *save_after = m.save_after;
  return PolyakOn(m) ? 1 : 0;
}
// 1 if the reference's loop inserts into the Polyak queue after TrainOneBatch call `iteration` (PolyakDue), else 0
API int cnb_net_polyak_due(void* p, long long iteration) { return PolyakDue(((NetHandle*)p)->net->Model(), iteration) ? 1 : 0; }

// ---- the device side of the input pipeline (data.h): a GPU-resident chunk + per-minibatch crop / mirror into the net's input
API void* cnb_data_create(int chunk_size, int channels, int image_size_y, int image_size_x, int gpu_image_size_y,
                          int gpu_image_size_x, int translate, int flip, unsigned long long seed) {
  DataIterator* d = nullptr;
  Guard([&] {
    d = new DataIterator(chunk_size, channels, image_size_y, image_size_x, gpu_image_size_y, gpu_image_size_x,
                         translate != 0, flip != 0, seed);
  });
  return d;
}
API void cnb_data_destroy(void* d) { delete (DataIterator*)d; }
API int cnb_data_upload(void* d, const float* host, int first, int count) {
  return Guard([&] { ((DataIterator*)d)->Upload(host, first, count); });
}
// DataHandler::GetBatch for the input layer of `net`: sample the jitter, then cut images [start, start + batch) into it
API int cnb_data_get_batch(void* d, void* net, int start, int multiplicity_id) {
  return Guard([&] {
    DataIterator* it = (DataIterator*)d;
    Matrix& dest = ((NetHandle*)net)->net->InputLayer().GetState();
    it->SampleNoise(dest.GetRows(), multiplicity_id);
    it->AddNoise(start, dest);
  });
}
// the jitter of the last minibatch (host copies): out = {width offsets, height offsets, mirror bits}, 3 x batch floats
API int cnb_data_last_noise(void* d, float* out, int cap) {
  const NoiseStage& noise = ((DataIterator*)d)->Noise();
  const int n = noise.LastBatch();
  if (cap < 3 * n) return -1;
  memcpy(out, noise.Last(), sizeof(float) * 3 * n);
  return n;
}
// pure host logic (no GPU): offset of deterministic view `multiplicity_id` for a free range of (max_x, max_y) pixels
API void cnb_data_view_offset(int multiplicity_id, int max_offset_x, int max_offset_y, int* w, int* h) {
  Jitter::ViewOffset(multiplicity_id, max_offset_x, max_offset_y, w, h);
}

// ---- the data set feed (data.h): DataSchedule is the pure host state machine, DataHandler runs it on the GPU
API void* cnb_schedule_create(const DatasetOrder* c, int dataset_size, unsigned long long seed) {
  DataSchedule* s = nullptr;
  Guard([&] { s = new DataSchedule(*c, dataset_size, seed); });
  return s;
}
API void cnb_schedule_destroy(void* s) { delete (DataSchedule*)s; }
API int cnb_schedule_chunk_size(void* s) { return ((DataSchedule*)s)->ChunkSize(); }
// the next minibatch: *start, *multiplicity_id; returns 1 if a chunk was loaded for it (its data set rows into rows[chunk]),
// else 0; perm[chunk] receives the permutation in force
API int cnb_schedule_next(void* p, int* start, int* multiplicity_id, int* rows, int* perm) {
  DataSchedule* s = (DataSchedule*)p;
  const DataSchedule::Batch b = s->Next();
  *start = b.start; *multiplicity_id = b.multiplicity_id;
  memcpy(perm, s->Permutation().data(), sizeof(int) * s->ChunkSize());
  if (b.loaded) memcpy(rows, s->Rows().data(), sizeof(int) * s->ChunkSize());
  return b.loaded ? 1 : 0;
}
API int cnb_schedule_seek(void* s, int row) { return Guard([&] { ((DataSchedule*)s)->Seek(row); }); }
// images: dataset_size x channels*y*x floats, labels: dataset_size ints (or NULL), targets: dataset_size x target_dims
// floats (or NULL), all in host memory that outlives the handler
API void* cnb_handler_create(const DatasetOrder* c, int dataset_size, int channels, int image_size_y, int image_size_x,
                             int gpu_image_size_y, int gpu_image_size_x, int translate, int flip, const float* images,
                             const int* labels, const float* targets, int target_dims, unsigned long long seed) {
  DataHandler* h = nullptr;
  Guard([&] {
    h = new DataHandler(*c, dataset_size, channels, image_size_y, image_size_x, gpu_image_size_y, gpu_image_size_x,
                        translate != 0, flip != 0, images, labels, targets, target_dims, seed);
  });
  return h;
}
API void cnb_handler_destroy(void* h) { delete (DataHandler*)h; }
API int cnb_handler_get_batch(void* h, void* net) { return Guard([&] { ((DataHandler*)h)->GetBatch(*((NetHandle*)net)->net); }); }
API int cnb_handler_seek(void* h, int row) { return Guard([&] { ((DataHandler*)h)->Seek(row); }); }
// the last minibatch (host copies): *start, *multiplicity_id, the data set row of each image (rows[batch]) and its jitter
// (noise[3 x batch]: width offsets, height offsets, mirror bits); returns the batch size
API int cnb_handler_last(void* p, int* start, int* multiplicity_id, int* rows, float* noise) {
  DataHandler* h = (DataHandler*)p;
  const DataSchedule& s = h->Schedule();
  const int n = h->Noise().LastBatch();
  *start = h->LastBatch().start; *multiplicity_id = h->LastBatch().multiplicity_id;
  for (int i = 0; i < n; i++) rows[i] = s.Rows()[s.Permutation()[h->LastBatch().start + i]];
  memcpy(noise, h->Noise().Last(), sizeof(float) * 3 * n);
  return n;
}
// the model's train_dataset (which 0) or valid_dataset (1): 1 and its fields, 0 when the model has none
API int cnb_net_dataset(void* p, int which, DatasetOrder* order, int* translate, int* flip, int* gpu_image_size_y,
                        int* gpu_image_size_x) {
  const ModelConfig& m = ((NetHandle*)p)->net->Model();
  const ModelConfig::Dataset& d = which ? m.valid_dataset : m.train_dataset;
  *order = d.order; *translate = d.translate; *flip = d.flip;
  *gpu_image_size_y = d.gpu_image_size_y; *gpu_image_size_x = d.gpu_image_size_x;
  return d.present ? 1 : 0;
}

// ---- the training loop (train.cc).  Host only: a model's schedule, CheckReduceLearningRate and the loop's decisions
// the model's training schedule: ints = {max_iter, print_after, validate_after, save_after, reduce_lr_num_steps,
// reduce_lr_max, smaller_is_better}, floats = {reduce_lr_factor, reduce_lr_threshold}, and reduce_lr_layer_name and
// checkpoint_dir (NUL-terminated, owned by the handle)
API void cnb_net_schedule(void* p, int* ints, float* floats, const char** layer_name, const char** checkpoint_dir) {
  const ModelConfig& m = ((NetHandle*)p)->net->Model();
  const int v[] = {m.max_iter, m.print_after, m.validate_after, m.save_after, m.reduce_lr_num_steps, m.reduce_lr_max,
                   m.smaller_is_better ? 1 : 0};
  memcpy(ints, v, sizeof(v));
  floats[0] = m.reduce_lr_factor; floats[1] = m.reduce_lr_threshold;
  *layer_name = m.reduce_lr_layer_name.c_str();
  *checkpoint_dir = m.checkpoint_dir.c_str();
}
API int cnb_reduce_lr_due(const float* history, int len, int num_steps, float threshold, int smaller_is_better) {
  return ReduceLrDue(std::vector<float>(history, history + len), num_steps, threshold, smaller_is_better != 0) ? 1 : 0;
}
// ConvNet::Train's decisions for the model, from TrainOneBatch call `start` + 1 to max_iter: per iteration with an action,
// iters[k] and actions[k] (TrainSchedule::Action bits, plus 16: the learning rate is reduced after this validation, 32:
// this validation runs on the Polyak average), and for the save after the loop a last record (max_iter, 8 | 64).  The
// validations take the values values[0, n_values) in order.  Returns the number of records (writes up to `cap`); refused:
// a schedule the loop refuses, or more validations than values
API long long cnb_net_train_dry_run(void* p, long long start, int lr_reduce_counter, int validation_set,
                                    const float* values, int n_values, long long cap, long long* iters, int* actions) {
  long long n = 0;
  const int rc = Guard([&] {
    const ModelConfig& m = ((NetHandle*)p)->net->Model();
    TrainSchedule s(m, lr_reduce_counter);
    auto put = [&](long long it, int a) { if (n < cap) { iters[n] = it; actions[n] = a; } n++; };
    int validated = 0;
    long long inserted = 0;
    for (long long it = start + 1; it <= m.max_iter; it++) {
      int a = s.Actions(it, validation_set != 0);
      if (a & TrainSchedule::INSERT) inserted++;
      if (a & TrainSchedule::VALIDATE) {
        if (validated == n_values) throw std::invalid_argument("more validations than values");
        if (PolyakOn(m) && inserted > 0) a |= 32;
        if (s.Validated(values[validated++])) a |= 16;
      }
      if (a) put(it, a);
    }
    if (s.FinalSave()) put(m.max_iter, TrainSchedule::SAVE | 64);
  });
  return rc ? rc : n;
}

API int cnb_net_validate(void* p, void* handler, float* out) {
  return Guard([&] { *out = ((NetHandle*)p)->net->Validate(*(DataHandler*)handler); });
}
// ConvNet::Train; valid, checkpoint_dir and run_name may be NULL.  Returns the number of events (cnb_net_train_event)
API int cnb_net_train(void* p, void* train, void* valid, const char* checkpoint_dir, const char* run_name) {
  NetHandle* h = (NetHandle*)p;
  h->events.clear();
  const int rc = Guard([&] {
    h->events = h->net->Train(*(DataHandler*)train, (DataHandler*)valid, checkpoint_dir ? checkpoint_dir : "",
                              run_name ? run_name : "");
  });
  return rc ? rc : (int)h->events.size();
}
// event k of the last cnb_net_train: *kind 0 train, 1 valid.  0 ok, -1 k out of range
API int cnb_net_train_event(void* p, int k, long long* iteration, int* kind, float* value, int* lr_reduced, int* polyak) {
  const std::vector<TrainEvent>& e = ((NetHandle*)p)->events;
  if (k < 0 || k >= (int)e.size()) return -1;
  *iteration = e[k].iteration; *kind = e[k].kind; *value = e[k].value;
  *lr_reduced = e[k].lr_reduced; *polyak = e[k].polyak;
  return 0;
}
API int cnb_net_lr_reduce_counter(void* p) { return ((NetHandle*)p)->net->LrReduceCounter(); }
