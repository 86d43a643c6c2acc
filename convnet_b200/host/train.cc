// train.cc — the reference's training driver (src/convnet.cc:866-1006 Train, :571-589 Validate, :788-818
// CheckReduceLearningRate, :659-667 Save, :765-785 WriteLog / WriteValLog, :830-838 TimestampModel) over DataHandlers.
// The schedule is TrainSchedule, host logic only; the loop runs it on the net.  Per step the loop adds the output layer's
// metric and its cnb_sum into a device slot and nothing else: the host copies the slots back, and waits for the device,
// only at a print, a validation or a checkpoint.
#include "convnet.h"

#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <ctime>
#include <filesystem>
#include <fstream>
#include <stdexcept>

namespace cnbhost {

bool ReduceLrDue(const std::vector<float>& history, int num_steps, float threshold, bool smaller_is_better) {
  const int len = (int)history.size();
  if (len < num_steps) return false;
  int i = len - num_steps;
  float mean1 = 0, mean2 = 0;
  for (int j = 0; j < num_steps / 2; j++) mean1 = (mean1 * j) / (j + 1) + history[i++] / (j + 1);
  for (int j = 0; j < num_steps - num_steps / 2; j++) mean2 = (mean2 * j) / (j + 1) + history[i++] / (j + 1);
  const float diff = smaller_is_better ? mean1 - mean2 : mean2 - mean1;
  return diff < threshold;
}

TrainSchedule::TrainSchedule(const ModelConfig& m, int lr_reduce_counter) : m_(m), lr_reduce_counter_(lr_reduce_counter) {
  for (const auto& [field, period] : {std::make_pair("print_after", m.print_after), std::make_pair("save_after", m.save_after)})
    if (period == 0)
      throw std::invalid_argument(std::string("field '") + field + "': 0 (the loop acts where the iteration modulo " + field +
                                  " is 0; -1 acts after every step)");
  const std::string& out = m.layer.back().name;
  if (!m.reduce_lr_layer_name.empty() && m.reduce_lr_layer_name != out)
    throw std::invalid_argument("field 'reduce_lr_layer_name': '" + m.reduce_lr_layer_name + "' is not the output layer ('" +
                                out + "')");
}

int TrainSchedule::Actions(long long it, bool validation_set) const {
  int a = 0;
  if (it % m_.print_after == 0) a |= PRINT;                                          // :937
  if (PolyakDue(m_, it)) a |= INSERT;                                                // :965-969
  if (validation_set && m_.validate_after > 0 && it % m_.validate_after == 0) a |= VALIDATE;   // :971-972
  if (it % m_.save_after == 0) a |= SAVE;                                            // :998
  return a;
}

bool TrainSchedule::Validated(float value) {
  history_.push_back(value);
  if (!(m_.reduce_lr_factor < 1.f)) return false;
  // :988-989: the && short-circuits, so dont_reduce_lr counts down only where the first two terms hold
  if (ReduceLrDue(history_, m_.reduce_lr_num_steps, m_.reduce_lr_threshold, m_.smaller_is_better) &&
      lr_reduce_counter_ < m_.reduce_lr_max && dont_reduce_lr_-- < 0) {
    dont_reduce_lr_ = m_.reduce_lr_num_steps;
    ++lr_reduce_counter_;
    return true;
  }
  return false;
}

namespace {

void CheckBatch(const DataHandler& d, int batch_size, const char* what) {
  if (d.Schedule().BatchSize() != batch_size)
    throw std::invalid_argument(std::string(what) + ": the net's batch size is " + std::to_string(batch_size) +
                                " and the handler's " + std::to_string(d.Schedule().BatchSize()));
}

void AppendLine(const std::string& path, const std::string& line) {
  std::ofstream f(path, std::ofstream::out | std::ofstream::app);
  f << line << '\n';
  if (!f) throw std::runtime_error("cannot write '" + path + "'");
}

std::string Format(const char* fmt, long long it, double a, double b = 0) {
  char buf[128];
  snprintf(buf, sizeof(buf), fmt, it, a, b);
  return buf;
}

std::string Timestamp() {                                     // src/util.cc GetTimeStamp
  const time_t now = time(nullptr);
  struct tm t;
  localtime_r(&now, &t);
  char buf[32];
  strftime(buf, sizeof(buf), "%Y%m%d%H%M%S", &t);
  return buf;
}

}  // namespace

float ConvNet::Validate(DataHandler& data) {
  CheckBatch(data, batch_size_, "Validate");
  const int batches = data.Schedule().DatasetSize() / batch_size_;
  Matrix slots;
  slots.AllocateGPUMemory(1, std::max(batches, 1));
  data.Seek(0);
  for (int k = 0; k < batches; k++) {
    data.GetBatch(*this);
    Fprop(false);
    SumPerformanceMetric(slots.GetDevData() + k);
  }
  std::vector<float> e((size_t)batches);
  if (batches) slots.CopyToHost(e.data(), e.size());
  float total = 0;
  for (int k = 0; k < batches; k++) total = (total * k) / (k + 1) + e[k] / (batch_size_ * (k + 1));
  return total;
}

void ConvNet::SaveWithPolyak(const std::string& path) {
  printf("Saving model to %s\n", path.c_str());
  fflush(stdout);
  Save(path);
  if (!PolyakOn(model_)) return;
  if (PolyakCount() == 0) {                                   // the reference divides by zero here
    printf("Saving model to %spolyak: the Polyak queue is empty, so it holds the current weights\n", path.c_str());
    fflush(stdout);
    Save(path + "polyak");
    return;
  }
  LoadPolyakWeights();
  Save(path + "polyak");
  LoadCurrentWeights();
}

std::vector<TrainEvent> ConvNet::Train(DataHandler& train, DataHandler* valid, const std::string& checkpoint_dir,
                                       const std::string& run_name) {
  if (dp_) throw std::invalid_argument("Train: the net trains data parallel, and the loop runs on one GPU only");
  TrainSchedule schedule(model_, lr_reduce_counter_);
  CheckBatch(train, batch_size_, "Train");
  if (valid) CheckBatch(*valid, batch_size_, "Train (validation set)");
  const ModelConfig& m = model_;
  const std::string dir = !checkpoint_dir.empty() ? checkpoint_dir : !m.checkpoint_dir.empty() ? m.checkpoint_dir : ".";
  const std::string base = dir + "/" + (run_name.empty() ? m.name + "_" + Timestamp() : run_name);
  std::error_code ec;
  std::filesystem::create_directories(dir, ec);
  if (ec) throw std::runtime_error("cannot create '" + dir + "': " + ec.message());
  {                                                           // TimestampModel: the model the run starts from
    std::ofstream f(base + ".pbtxt", std::ofstream::out | std::ofstream::trunc);
    f << ModelText(CurrentModel());
    if (!f) throw std::runtime_error("cannot write '" + base + ".pbtxt'");
  }
  printf("Checkpointing at %s\n", base.c_str());
  fflush(stdout);

  const long long start = (long long)step_, end = m.max_iter;
  // one slot per step since the last print: at most |print_after| of them
  Matrix slots;
  slots.AllocateGPUMemory(1, (int)std::max(1LL, std::min(std::llabs((long long)m.print_after), end - start)));
  std::vector<float> host;
  std::vector<TrainEvent> events;
  int k = 0;
  auto t0 = std::chrono::steady_clock::now();
  for (long long i = start; i < end; i++) {
    train.GetBatch(*this);
    TrainOneBatch(nullptr);
    SumPerformanceMetric(slots.GetDevData() + k++);
    const long long it = i + 1;
    const int a = schedule.Actions(it, valid != nullptr);
    if (a & TrainSchedule::PRINT) {
      host.resize((size_t)k);
      slots.CopyToHost(host.data(), host.size());
      float sum = 0;                                          // AddVectors, then / (print_after * batch_size): :947
      for (float v : host) sum += v;
      sum /= (float)(m.print_after * batch_size_);
      k = 0;
      const auto t1 = std::chrono::steady_clock::now();
      const double secs = std::chrono::duration<double>(t1 - t0).count();
      t0 = t1;
      printf("Step %lld Time %.5g s Train Acc : %.6g\n", it, secs, sum);
      fflush(stdout);
      AppendLine(base + "_train.log", Format("%lld %.6g %.9g", it, secs, sum));
      events.push_back({it, TrainEvent::TRAIN, sum});
    }
    if (a & TrainSchedule::INSERT) InsertPolyak();
    if (a & TrainSchedule::VALIDATE) {
      // with Polyak on: on the average, and training continues from it (the reference's :976 is commented out)
      const bool average = PolyakOn(m) && PolyakCount() > 0;
      if (average) LoadPolyakWeights();
      const float v = Validate(*valid);
      const bool reduce = schedule.Validated(v);
      if (reduce) {
        ReduceLearningRate(m.reduce_lr_factor);
        lr_reduce_counter_ = schedule.LrReduceCounter();
      }
      printf("Step %lld Val Acc : %.6g%s", it, v,
             PolyakOn(m) ? (average ? " (Polyak average)" : " (current weights: the Polyak queue is empty)") : "");
      if (reduce) printf(" Learning rate reduced %d time(s).", lr_reduce_counter_);
      printf("\n");
      fflush(stdout);
      AppendLine(base + "_valid.log", Format("%lld %.9g", it, v));
      events.push_back({it, TrainEvent::VALID, v, reduce, average});
    }
    if (a & TrainSchedule::SAVE) SaveWithPolyak(base + ".ckpt");
  }
  if (schedule.FinalSave()) SaveWithPolyak(base + ".ckpt");
  return events;
}

}  // namespace cnbhost
