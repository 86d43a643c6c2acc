// checkpoint.cc — ConvNet::Save / Load (src/convnet.cc:669-751), Polyak averaging (InsertPolyak / LoadPolyakWeights /
// LoadCurrentWeights, :686-730) and PRETRAINED edges (edge_with_weight.cc:132-135).  The reference writes HDF5; there is no
// HDF5 library here, so the container is the project's own (DESIGN.md §5 "Checkpoints"), with the reference's dataset
// names as record names.
#include "convnet.h"

#include <fcntl.h>
#include <unistd.h>

#include <cerrno>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <set>
#include <stdexcept>

namespace cnbhost {

namespace {

const char kMagic[8] = {'C', 'N', 'B', 'C', 'K', 'P', 'T', '\0'};
const uint32_t kVersion = 1;
const char* const kTypeNames[] = {"float32", "int64", "text"};
const size_t kTypeBytes[] = {4, 8, 1};

std::string Errno() { return strerror(errno); }

// little-endian scalars (the hosts this runs on are little-endian; the format fixes the byte order)
template <class T>
void Put(std::string& out, T v) { out.append(reinterpret_cast<const char*>(&v), sizeof(v)); }

class RecordWriter {
 public:
  RecordWriter(FILE* f, const std::string& path) : f_(f), path_(path) {}
  void Header(const std::string& name, uint8_t type, uint64_t count) {
    std::string h;
    Put<uint32_t>(h, (uint32_t)name.size());
    h += name;
    Put<uint8_t>(h, type);
    Put<uint64_t>(h, count);
    Write(h.data(), h.size());
  }
  void Write(const void* p, size_t bytes) {
    if (bytes && fwrite(p, 1, bytes, f_) != bytes) throw std::runtime_error("cannot write '" + path_ + "': " + Errno());
  }
  void Text(const std::string& name, const std::string& s) { Header(name, CheckpointFile::TEXT, s.size()); Write(s.data(), s.size()); }
  void Int(const std::string& name, long long v) { Header(name, CheckpointFile::INT64, 1); Write(&v, 8); }
  void Floats(const std::string& name, const float* dev, long long n) {
    Header(name, CheckpointFile::FLOAT32, (uint64_t)n);
    std::vector<float> h((size_t)n);
    if (n) CUDA_CHECK(cudaMemcpy(h.data(), dev, sizeof(float) * (size_t)n, cudaMemcpyDeviceToHost));
    Write(h.data(), sizeof(float) * h.size());
  }

 private:
  FILE* f_;
  const std::string& path_;
};

const char* AdaptiveSuffix(const OptimizerConfig& o) {
  return o.optimizer_type == ADAGRAD_SGD ? "_adagrad_history" : o.optimizer_type == RMSPROP_SGD ? "_rms_history" : nullptr;
}

}  // namespace

// ---------------------------------------------------------------- the file
CheckpointFile::CheckpointFile(const std::string& path) : path_(path) {
  auto fail = [&](const std::string& what) { throw std::invalid_argument("checkpoint '" + path + "': " + what); };
  FILE* f = fopen(path.c_str(), "rb");
  if (!f) fail("cannot open: " + Errno());
  struct Closer { FILE* f; ~Closer() { fclose(f); } } closer{f};
  if (fseeko(f, 0, SEEK_END) != 0) fail("cannot seek: " + Errno());
  const long long size = (long long)ftello(f);
  rewind(f);
  char magic[8];
  uint32_t version = 0;
  if (fread(magic, 1, 8, f) != 8 || memcmp(magic, kMagic, 8) != 0) fail("not a checkpoint file (bad magic)");
  if (fread(&version, 4, 1, f) != 1) fail("truncated in the header");
  if (version != kVersion) fail("version " + std::to_string(version) + " (this build reads version " + std::to_string(kVersion) + ")");
  long long pos = 12;
  while (pos < size) {
    const std::string after = names_.empty() ? "the header" : "record '" + names_.back() + "'";
    uint32_t len = 0;
    if (fread(&len, 4, 1, f) != 1) fail("truncated after " + after);
    if ((long long)len > size - pos - 4) fail("truncated in the name of the record after " + after);
    std::string name(len, '\0');
    uint8_t type = 0;
    uint64_t count = 0;
    if ((len && fread(&name[0], 1, len, f) != len) || fread(&type, 1, 1, f) != 1 || fread(&count, 8, 1, f) != 1)
      fail("truncated in the header of record '" + name + "'");
    if (type > TEXT) fail("record '" + name + "': unknown type " + std::to_string(type));
    pos += 4 + (long long)len + 1 + 8;
    const long long avail = size - pos;
    if (count > (uint64_t)avail / kTypeBytes[type])
      fail("record '" + name + "' is truncated: it holds " + std::to_string(count) + " " + kTypeNames[type] + " elements, the file has " +
           std::to_string(avail / (long long)kTypeBytes[type]) + " left");
    if (!records_.emplace(name, Record{type, (long long)count, pos}).second) fail("record '" + name + "' appears twice");
    names_.push_back(name);
    pos += (long long)count * (long long)kTypeBytes[type];
    if (fseeko(f, (off_t)pos, SEEK_SET) != 0) fail("cannot seek: " + Errno());
  }
}

std::string CheckpointFile::Check(const std::string& name, int type, long long count) const {
  const std::string at = "checkpoint '" + path_ + "': record '" + name + "'";
  auto it = records_.find(name);
  if (it == records_.end()) return at + " is missing";
  const Record& r = it->second;
  if (r.type != type) return at + " is " + kTypeNames[r.type] + ", expected " + kTypeNames[type];
  if (count >= 0 && r.count != count)
    return at + " holds " + std::to_string(r.count) + " " + kTypeNames[type] + " elements, the net's tensor has " +
           std::to_string(count);
  return "";
}

std::vector<char> CheckpointFile::Read(const std::string& name) const {
  const Record& r = records_.at(name);
  std::vector<char> out((size_t)(r.count * (long long)kTypeBytes[r.type]));
  const int fd = open(path_.c_str(), O_RDONLY);
  if (fd < 0) throw std::runtime_error("checkpoint '" + path_ + "': cannot open: " + Errno());
  size_t done = 0;
  while (done < out.size()) {
    const ssize_t k = pread(fd, out.data() + done, out.size() - done, (off_t)(r.offset + (long long)done));
    if (k <= 0) {
      const std::string why = k < 0 ? Errno() : "unexpected end of file";
      close(fd);
      throw std::runtime_error("checkpoint '" + path_ + "': record '" + name + "': " + why);
    }
    done += (size_t)k;
  }
  close(fd);
  return out;
}

// ---------------------------------------------------------------- what a net writes and reads
std::vector<CheckpointEntry> ConvNet::CheckpointEntries(const std::vector<OptimizerConfig>& opt) {
  std::vector<CheckpointEntry> out;
  for (size_t k = 0; k < tensors_.size(); k++) {
    const TrainedTensor& t = tensors_[k];
    // a tensor and its optimizer's records (SGDOptimizer / AdagradSGDOptimizer / RMSPropSGDOptimizer ::SaveParameters)
    if (t.n > 0) {
      out.push_back({t.name, CheckpointEntry::PARAMS, t.offset, t.n, k, nullptr});
      out.push_back({t.name + "_gradient_history", CheckpointEntry::HISTORY, t.offset, t.n, k, nullptr});
      out.push_back({t.name + "_step", CheckpointEntry::STEP, 0, 1, k, nullptr});
      if (const char* s = AdaptiveSuffix(opt[k])) out.push_back({t.name + s, CheckpointEntry::STATE, t.offset, t.n, k, nullptr});
    }
    if (t.kind == TrainedTensor::BETA) {               // the layer's running statistics follow its gamma and beta
      Layer* l = layers_[t.edge + 1].get();
      out.push_back({l->GetName() + ":running_mean", CheckpointEntry::RUNNING, 0, t.n, k, l->BnStat(0)});
      out.push_back({l->GetName() + ":running_sigma", CheckpointEntry::RUNNING, 0, t.n, k, l->BnStat(1)});
    }
  }
  return out;
}

float* ConvNet::EntryData(const CheckpointEntry& e) {
  switch (e.buffer) {
    case CheckpointEntry::PARAMS: return parameters_.GetDevData() + e.offset;
    case CheckpointEntry::HISTORY: return history_.GetDevData() + e.offset;
    case CheckpointEntry::STATE: return AdaptiveState() + e.offset;
    case CheckpointEntry::RUNNING: return e.running;
    default: return nullptr;
  }
}

ModelConfig ConvNet::CurrentModel() const {
  ModelConfig m = model_;
  for (const TrainedTensor& t : tensors_) ModelOptimizer(m, t) = t.opt;
  return m;
}

void ConvNet::WaitAllStreams() {
  CUDA_CHECK(cudaStreamSynchronize(Matrix::Stream()));
  for (cudaStream_t s : {side_, comm_, opt_}) if (s) CUDA_CHECK(cudaStreamSynchronize(s));
}

// after a bulk write of the parameters: the dgrad banks are rebuilt now, on the main stream, rather than inside the next
// step's dgrad (the optimizer stream's next prestage waits for the main stream)
void ConvNet::PrestageAll() {
  if (!prestage_) return;
  for (auto& e : edges_)
    if (EdgeWithWeight* w = dynamic_cast<EdgeWithWeight*>(e.get())) w->PrestageDown();
}

void ConvNet::Save(const std::string& path) {
  WaitAllStreams();                                  // the last bucket's update may still be running on opt_
  const ModelConfig m = CurrentModel();
  const std::string tmp = path + "temp";
  FILE* f = fopen(tmp.c_str(), "wb");
  if (!f) throw std::runtime_error("cannot create '" + tmp + "': " + Errno());
  try {
    RecordWriter w(f, tmp);
    w.Write(kMagic, 8);
    w.Write(&kVersion, 4);
    w.Text("__model__", ModelText(m));
    w.Int("__current_iter__", (long long)step_);
    w.Int("__seed__", (long long)model_.seed);
    if (lr_reduce_counter_) w.Int("__lr_reduce_counter__", lr_reduce_counter_);   // (a net the loop never reduced: no record)
    std::vector<OptimizerConfig> opt;
    for (const TrainedTensor& t : tensors_) opt.push_back(t.opt);
    for (const CheckpointEntry& e : CheckpointEntries(opt)) {
      if (e.buffer == CheckpointEntry::STEP)
        w.Int(e.name, tensors_[e.tensor].step);
      else
        w.Floats(e.name, EntryData(e), e.n);
    }
    if (fflush(f) != 0 || fsync(fileno(f)) != 0) throw std::runtime_error("cannot write '" + tmp + "': " + Errno());
  } catch (...) {
    fclose(f);
    remove(tmp.c_str());
    throw;
  }
  if (fclose(f) != 0) { remove(tmp.c_str()); throw std::runtime_error("cannot write '" + tmp + "': " + Errno()); }
  if (rename(tmp.c_str(), path.c_str()) != 0)
    throw std::runtime_error("cannot rename '" + tmp + "' to '" + path + "': " + Errno());
}

void ConvNet::Load(const std::string& path) {
  // 1. read and check everything before anything changes
  const CheckpointFile f(path);
  auto fail = [&](const std::string& record, const std::string& what) {
    throw std::invalid_argument("checkpoint '" + path + "': record '" + record + "' " + what);
  };
  for (const char* name : {"__model__", "__current_iter__", "__seed__"}) {
    const std::string why = f.Check(name, name[2] == 'm' ? CheckpointFile::TEXT : CheckpointFile::INT64, name[2] == 'm' ? -1 : 1);
    if (!why.empty()) throw std::invalid_argument(why);
  }
  const std::vector<char> text = f.Read("__model__");
  ModelConfig saved;
  try {
    saved = ReadModelText(std::string(text.begin(), text.end()), path + " (record __model__)", false);
  } catch (const std::invalid_argument& e) {
    fail("__model__", std::string("cannot be read: ") + e.what());
  }
  // the optimizer blocks in force when the file was written, matched to this net's edges and layers by name
  ModelConfig opt = CurrentModel();
  std::string unmatched;
  for (size_t i = 0; i < edges_.size(); i++) {
    if (owner_[i] != (int)i) continue;                 // no parameters, or a tied edge's (its owner's records hold them)
    bool found = false;
    for (const EdgeConfig& e : saved.edge)
      if (e.source + ":" + e.dest == edges_[i]->GetName() && e.edge_type == model_.edge[i].edge_type && e.tied_to.empty()) {
        opt.edge[i].weight_optimizer = e.weight_optimizer;
        if (!e.has_no_bias) opt.edge[i].bias_optimizer = e.bias_optimizer;
        found = true;
      }
    if (!found && unmatched.empty()) unmatched = "has no edge '" + edges_[i]->GetName() + "' of this net's type";
  }
  for (size_t i = 0; i < layers_.size(); i++) {
    if (!layers_[i]->BatchNormalize()) continue;
    bool found = false;
    for (const LayerConfig& l : saved.layer)
      if (l.name == layers_[i]->GetName() && l.batch_normalize) {
        opt.layer[i].gamma_optimizer = l.gamma_optimizer;
        opt.layer[i].beta_optimizer = l.beta_optimizer;
        found = true;
      }
    if (!found && unmatched.empty()) unmatched = "has no batch-normalised layer '" + layers_[i]->GetName() + "'";
  }
  std::vector<OptimizerConfig> configs;
  for (const TrainedTensor& t : tensors_) configs.push_back(ModelOptimizer(opt, t));
  const std::vector<CheckpointEntry> entries = CheckpointEntries(configs);
  // optional: the reductions of the learning rate ConvNet::Train applied.  Unlike the reference's Load (src/convnet.cc:
  // 745-748) they are not applied again: __model__ already holds the epsilons they left
  long long lr_reduce_counter = 0;
  if (f.Has("__lr_reduce_counter__")) {
    const std::string why = f.Check("__lr_reduce_counter__", CheckpointFile::INT64, 1);
    if (!why.empty()) throw std::invalid_argument(why);
    memcpy(&lr_reduce_counter, f.Read("__lr_reduce_counter__").data(), 8);
  }
  std::set<std::string> known = {"__model__", "__current_iter__", "__seed__", "__lr_reduce_counter__"};
  for (const CheckpointEntry& e : entries) {
    const bool step = e.buffer == CheckpointEntry::STEP;
    const std::string why = f.Check(e.name, step ? CheckpointFile::INT64 : CheckpointFile::FLOAT32, e.n);
    if (!why.empty()) throw std::invalid_argument(why);
    known.insert(e.name);
  }
  for (const std::string& name : f.Names())
    if (!known.count(name)) fail(name, "has no place in this net");
  if (!unmatched.empty()) fail("__model__", unmatched);
  std::vector<std::vector<char>> data;
  for (const CheckpointEntry& e : entries) data.push_back(f.Read(e.name));
  long long iter = 0, seed = 0;
  memcpy(&iter, f.Read("__current_iter__").data(), 8);
  memcpy(&seed, f.Read("__seed__").data(), 8);

  // 2. nothing runs on any stream any more
  WaitAllStreams();
  // 3. the optimizer settings (these allocate the adaptive state if the file's optimizers need it)
  for (size_t k = 0; k < tensors_.size(); k++) SetOptimizer(tensors_[k], configs[k]);
  // 4. every tensor, step count, the iteration and the seed
  for (size_t k = 0; k < entries.size(); k++) {
    const CheckpointEntry& e = entries[k];
    if (e.buffer == CheckpointEntry::STEP) {
      memcpy(&tensors_[e.tensor].step, data[k].data(), 8);
    } else if (e.n) {
      CUDA_CHECK(cudaMemcpyAsync(EntryData(e), data[k].data(), sizeof(float) * (size_t)e.n, cudaMemcpyHostToDevice,
                                 Matrix::Stream()));
    }
  }
  step_ = (unsigned long long)iter;
  lr_reduce_counter_ = (int)lr_reduce_counter;
  model_.seed = (unsigned)seed;
  if (salted_) SaltDropout();                        // the file's seed, this net's rank
  CUDA_CHECK(cudaStreamSynchronize(Matrix::Stream()));        // (the host buffers go away)
  // 5. the staged copies of the old weights: dropped, and the dgrad banks rebuilt
  InvalidateStaging();
  PrestageAll();
}

void ConvNet::LoadPretrained(size_t i) {
  const EdgeConfig& c = model_.edge[i];
  const std::string& edge = edges_[i]->GetName();
  const std::string from = c.pretrained_edge_name.empty() ? edge : c.pretrained_edge_name;
  const CheckpointFile f(c.pretrained_model);
  for (TrainedTensor& t : tensors_) {
    if (t.owner != (int)i || !t.OnEdge() || t.n == 0) continue;
    const std::string prefix = from + t.name.substr(edge.size());            // <from>:weight, <from>:bias
    const char* adaptive = AdaptiveSuffix(t.opt);
    std::vector<std::pair<std::string, float*>> tensors = {{prefix, parameters_.GetDevData() + t.offset},
                                                          {prefix + "_gradient_history", history_.GetDevData() + t.offset}};
    // the adaptive state where the file has it for this edge's kind of optimizer; otherwise the fresh start stays
    if (adaptive && f.Has(prefix + adaptive)) tensors.push_back({prefix + adaptive, AdaptiveState() + t.offset});
    for (const auto& [name, dev] : tensors) {
      const std::string why = f.Check(name, CheckpointFile::FLOAT32, t.n);
      if (!why.empty()) throw std::invalid_argument("edge '" + edge + "' (PRETRAINED): " + why);
    }
    const std::string why = f.Check(prefix + "_step", CheckpointFile::INT64, 1);
    if (!why.empty()) throw std::invalid_argument("edge '" + edge + "' (PRETRAINED): " + why);
    for (const auto& [name, dev] : tensors) {
      const std::vector<char> h = f.Read(name);
      CUDA_CHECK(cudaMemcpy(dev, h.data(), h.size(), cudaMemcpyHostToDevice));
    }
    memcpy(&t.step, f.Read(prefix + "_step").data(), 8);
  }
}

std::vector<float> PretrainedWeights(const EdgeConfig& c, long long n) {
  const CheckpointFile f(c.pretrained_model);
  const std::string name = (c.pretrained_edge_name.empty() ? c.source + ":" + c.dest : c.pretrained_edge_name) + ":weight";
  const std::string why = f.Check(name, CheckpointFile::FLOAT32, n);
  if (!why.empty()) throw std::invalid_argument(why);
  const std::vector<char> h = f.Read(name);
  std::vector<float> out((size_t)n);
  memcpy(out.data(), h.data(), h.size());
  return out;
}

// ---------------------------------------------------------------- Polyak averaging
bool PolyakDue(const ModelConfig& m, long long it) {
  if (!PolyakOn(m) || m.validate_after == 0 || m.save_after == 0) return false;   // (the reader refuses the zeros)
  const long long after = m.polyak_after, span = after * m.polyak_queue_size;
  const long long start_val = m.validate_after - span, start_save = m.save_after - span;
  return it % after == 0 && ((it % m.validate_after) >= start_val || (it % m.save_after) >= start_save);
}

void ConvNet::InsertPolyak() {
  if (!PolyakOn(model_)) throw std::invalid_argument("the model has no Polyak averaging (polyak_after, polyak_queue_size)");
  const size_t n = num_params_, slots = (size_t)model_.polyak_queue_size + 1;
  if (!polyak_) {
    if (cudaMalloc((void**)&polyak_, sizeof(float) * n * slots) != cudaSuccess) {
      cudaGetLastError();
      polyak_ = nullptr;
      throw std::runtime_error("cannot allocate the Polyak queue: " + std::to_string(slots) + " x " + std::to_string(n) +
                               " floats (" + std::to_string(sizeof(float) * n * slots >> 20) + " MB)");
    }
  }
  // after the optimizer stream's pending updates, without a host wait; the next step's updates wait for the main stream
  CUDA_CHECK(cudaEventRecord(ev_opt_, opt_));
  CUDA_CHECK(cudaStreamWaitEvent(Matrix::Stream(), ev_opt_, 0));
  CUDA_CHECK(cudaMemcpyAsync(polyak_ + (size_t)polyak_index_ * n, parameters_.GetDevData(), sizeof(float) * n,
                             cudaMemcpyDeviceToDevice, Matrix::Stream()));
  if (++polyak_index_ == model_.polyak_queue_size) { polyak_index_ = 0; polyak_full_ = true; }
}

void ConvNet::LoadPolyakWeights() {
  if (!PolyakOn(model_)) throw std::invalid_argument("the model has no Polyak averaging (polyak_after, polyak_queue_size)");
  if (PolyakCount() == 0) throw std::invalid_argument("LoadPolyakWeights: nothing has been inserted into the Polyak queue");
  const size_t n = num_params_;
  CUDA_CHECK(cudaEventRecord(ev_opt_, opt_));
  CUDA_CHECK(cudaStreamWaitEvent(Matrix::Stream(), ev_opt_, 0));
  float* backup = polyak_ + (size_t)model_.polyak_queue_size * n;
  CUDA_CHECK(cudaMemcpyAsync(backup, parameters_.GetDevData(), sizeof(float) * n, cudaMemcpyDeviceToDevice, Matrix::Stream()));
  // the kernel's write drops the staged copies of the old weights (bf16 twins and dgrad banks) itself.  Only the trained
  // range: the frozen parameters are equal in every slot, and their average could still round (DESIGN.md §5)
  const size_t lo = TrainedOffset();
  if (lo < n) cnb_polyak_average(parameters_.GetDevData() + lo, polyak_ + lo, (long long)(n - lo), (long long)n, PolyakCount());
  polyak_backup_ = true;
  PrestageAll();
}

void ConvNet::LoadCurrentWeights() {
  if (!polyak_backup_) throw std::invalid_argument("LoadCurrentWeights without an earlier LoadPolyakWeights");
  const size_t n = num_params_;
  CUDA_CHECK(cudaMemcpyAsync(parameters_.GetDevData(), polyak_ + (size_t)model_.polyak_queue_size * n, sizeof(float) * n,
                             cudaMemcpyDeviceToDevice, Matrix::Stream()));
  InvalidateStaging();
  PrestageAll();
}

}  // namespace cnbhost
