// data.cc — see data.h.
#include "data.h"

#include <cstring>
#include <stdexcept>
#include <string>

#include "convnet.h"

namespace cnbhost {

uint64_t SplitMix64(uint64_t& state) {
  uint64_t z = (state += 0x9E3779B97F4A7C15ULL);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL; z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
  return z ^ (z >> 31);
}

// the status of a crop launch: 0 ok, -1 shapes or pointers it cannot crop with, -3 the launch failed
static void CheckCrop(const char* call, int rc) {
  if (rc == -3) throw DeviceError(std::string(call) + ": the launch failed");
  if (rc != 0) throw std::invalid_argument(std::string(call) + " cannot crop with these shapes or pointers");
}

// ---------------------------------------------------------------- Jitter
Jitter::Jitter(int image_size_y, int image_size_x, int gpu_image_size_y, int gpu_image_size_x, bool translate, bool flip,
               uint64_t seed)
    : max_offset_y_(image_size_y - gpu_image_size_y), max_offset_x_(image_size_x - gpu_image_size_x), translate_(translate),
      flip_(flip), rng_(seed * 0x9E3779B97F4A7C15ULL + 0xD1B54A32D192ED03ULL) {}

float Jitter::Uniform() { return (float)(SplitMix64(rng_) >> 40) * (1.0f / 16777216.0f); }

void Jitter::ViewOffset(int multiplicity_id, int max_offset_x, int max_offset_y, int* w, int* h) {
  // position of view k = multiplicity_id % 5 along (x, y), in halves of the free range: 1 = centred, 0 / 2 = the two ends
  static const int kView[5][2] = {{1, 1}, {0, 0}, {2, 0}, {2, 2}, {0, 2}};
  auto place = [](int half_steps, int max_offset) { return half_steps == 1 ? max_offset / 2 : (half_steps == 2 ? max_offset : 0); };
  const int view = multiplicity_id % 5;
  *w = place(kView[view][0], max_offset_x);
  *h = place(kView[view][1], max_offset_y);
}

void Jitter::Sample(int batch_size, int multiplicity_id, float* out) {
  float *wo = out, *ho = out + batch_size, *fl = out + 2 * (size_t)batch_size;
  if (translate_) {                                          // random jitter: uniform * (max + 1), rounded down
    for (int i = 0; i < batch_size; i++) {
      const int oy = (int)(Uniform() * (max_offset_y_ + 1)), ox = (int)(Uniform() * (max_offset_x_ + 1));
      ho[i] = (float)(oy > max_offset_y_ ? max_offset_y_ : oy);        // (the product can round up to max + 1 in fp32)
      wo[i] = (float)(ox > max_offset_x_ ? max_offset_x_ : ox);
    }
  } else {                                                   // deterministic views: the centre, then the four corners
    int w, h;
    ViewOffset(multiplicity_id, max_offset_x_, max_offset_y_, &w, &h);
    for (int i = 0; i < batch_size; i++) { wo[i] = (float)w; ho[i] = (float)h; }
  }
  for (int i = 0; i < batch_size; i++) fl[i] = flip_ ? Uniform() : (float)(multiplicity_id / 5);
}

// ---------------------------------------------------------------- NoiseStage
NoiseStage::~NoiseStage() {
  if (!pinned_) return;                                      // nothing staged yet: nothing was created
  cudaStreamSynchronize(Matrix::Stream());                   // copies may still read the ring, crops the device block
  for (int k = 0; k < kRing; k++) cudaEventDestroy(done_[k]);
  cudaFree(device_); cudaFreeHost(pinned_);
}

const float* NoiseStage::Stage(Jitter& jitter, int batch_size, int multiplicity_id) {
  const cudaStream_t s = Matrix::Stream();
  if (batch_size > cap_) {
    if (pinned_) {
      CUDA_CHECK(cudaStreamSynchronize(s));
      CUDA_CHECK(cudaFree(device_)); CUDA_CHECK(cudaFreeHost(pinned_));
    } else {
      for (int k = 0; k < kRing; k++) CUDA_CHECK(cudaEventCreateWithFlags(&done_[k], cudaEventDisableTiming));
    }
    CUDA_CHECK(cudaMalloc((void**)&device_, sizeof(float) * 3 * (size_t)batch_size));
    CUDA_CHECK(cudaMallocHost((void**)&pinned_, sizeof(float) * 3 * (size_t)batch_size * kRing));
    cap_ = batch_size;
  }
  float* block = pinned_ + (size_t)slot_ * 3 * cap_;
  CUDA_CHECK(cudaEventSynchronize(done_[slot_]));           // kRing batches ago: long done
  jitter.Sample(batch_size, multiplicity_id, block);
  CUDA_CHECK(cudaMemcpyAsync(device_, block, sizeof(float) * 3 * batch_size, cudaMemcpyHostToDevice, s));
  CUDA_CHECK(cudaEventRecord(done_[slot_], s));
  slot_ = (slot_ + 1) % kRing;
  last_ = block;
  last_batch_ = batch_size;
  return device_;
}

// ---------------------------------------------------------------- DataIterator
DataIterator::DataIterator(int chunk_size, int channels, int image_size_y, int image_size_x, int gpu_image_size_y,
                           int gpu_image_size_x, bool translate, bool flip, uint64_t seed)
    : chunk_size_(chunk_size), channels_(channels), image_size_y_(image_size_y), image_size_x_(image_size_x),
      gpu_image_size_y_(gpu_image_size_y), gpu_image_size_x_(gpu_image_size_x),
      jitter_(image_size_y, image_size_x, gpu_image_size_y, gpu_image_size_x, translate, flip, seed) {
  if (chunk_size <= 0 || channels <= 0) throw std::invalid_argument("DataIterator: chunk_size and channels must be positive");
  if (gpu_image_size_y > image_size_y || gpu_image_size_x > image_size_x)
    throw std::invalid_argument("DataIterator: the crop (gpu_image_size " + std::to_string(gpu_image_size_y) + " x " +
                                std::to_string(gpu_image_size_x) + ") must fit the image (image_size " +
                                std::to_string(image_size_y) + " x " + std::to_string(image_size_x) + ")");
  data_.AllocateGPUMemory(NumDims(), chunk_size);          // one image per column (src/datahandler.cc:60-75)
}

void DataIterator::Upload(const float* host, int first, int count) {
  if (first < 0 || count < 0 || first + count > chunk_size_)
    throw std::invalid_argument("DataIterator::Upload: images [" + std::to_string(first) + ", " + std::to_string(first + count) +
                                ") are outside the chunk of " + std::to_string(chunk_size_));
  CUDA_CHECK(cudaMemcpyAsync(data_.GetDevData() + (size_t)first * NumDims(), host, sizeof(float) * (size_t)count * NumDims(),
                             cudaMemcpyHostToDevice, Matrix::Stream()));
}

void DataIterator::AddNoise(int start, Matrix& dest) {
  const int batch_size = dest.GetRows();
  if (start < 0 || start + batch_size > chunk_size_ || noise_.LastBatch() != batch_size)
    throw std::invalid_argument("DataIterator::AddNoise: slice out of range, or SampleNoise was not called for this batch size");
  if (dest.GetCols() != channels_ * gpu_image_size_y_ * gpu_image_size_x_)
    throw std::invalid_argument("DataIterator::AddNoise: dest is not batch x channels * crop");
  // (the reference copies with CopyTranspose when there is neither crop nor mirror; the same kernel covers that case)
  const int rc = cnb_extract_patches(data_.GetDevData() + (size_t)start * NumDims(), dest.GetDevData(), nullptr, d_noise_,
                                     d_noise_ + batch_size, d_noise_ + 2 * batch_size, batch_size, channels_, image_size_x_,
                                     image_size_y_, gpu_image_size_x_, gpu_image_size_y_, nullptr, nullptr, nullptr, nullptr, 0);
  CheckCrop("DataIterator::AddNoise: cnb_extract_patches", rc);
}

// ---------------------------------------------------------------- DataSchedule
DataSchedule::DataSchedule(const DatasetOrder& c, int dataset_size, uint64_t seed)
    : c_(c), dataset_size_(dataset_size), chunk_size_(c.chunk_size),
      cpu_rng_(seed * 0x9E3779B97F4A7C15ULL + 0x632BE59BD9B4E019ULL), gpu_rng_(seed * 0x9E3779B97F4A7C15ULL + 0x8CB92BA72F3D8DD7ULL) {
  auto refuse = [](const std::string& why) { throw std::invalid_argument("DataHandler: " + why); };
  if (dataset_size <= 0) refuse("the data set is empty");
  if (c.batch_size <= 0) refuse("batch_size must be positive");
  if (c.multiplicity <= 0) refuse("multiplicity must be positive");
  if (c.max_reuse_count < 0) refuse("max_reuse_count must not be negative");
  if (c.random_access_chunk_size <= 0) refuse("random_access_chunk_size must be positive");
  if (chunk_size_ <= 0 || chunk_size_ > dataset_size) {              // :45-48
    chunk_size_ = dataset_size;
    fits_on_gpu_ = true;
  }
  if (c.batch_size > chunk_size_)
    refuse("batch_size " + std::to_string(c.batch_size) + " is larger than the chunk (" + std::to_string(chunk_size_) +
           " images): every minibatch would reload it");
  if (c.randomize_cpu && chunk_size_ % c.random_access_chunk_size != 0)
    refuse("random_access_chunk_size " + std::to_string(c.random_access_chunk_size) + " does not divide the chunk (" +
           std::to_string(chunk_size_) + " images); the reference's LoadChunk would write past the chunk's end");
  perm_.resize(chunk_size_);                                        // SetupShuffler, :111-118 (identity when not shuffled)
  for (int i = 0; i < chunk_size_; i++) perm_[i] = i;
  if (c.randomize_cpu) {                                            // :54-60
    random_indices_.resize(dataset_size);
    for (int i = 0; i < dataset_size; i++) random_indices_[i] = i;
    Shuffle(random_indices_, cpu_rng_);
  }
  Seek(0);
}

void DataSchedule::Shuffle(std::vector<int>& v, uint64_t& rng) {
  for (size_t i = v.size(); i > 1; i--) std::swap(v[i - 1], v[SplitMix64(rng) % i]);
}

void DataSchedule::Seek(int row) {
  if (row < 0 || row >= dataset_size_) throw std::invalid_argument("DataHandler::Seek: row " + std::to_string(row) + " is outside the data set");
  preloading_ = false; preload_.clear();                            // Sync(): the preload finishes and is not used
  start_ = row;
  reuse_counter_ = 0;
  multiplicity_counter_ = 0;
  restart_ = true;
  row_ = row;                                                       // the data iterators' Seek(row)
}

std::vector<int> DataSchedule::DiskAccess() {
  std::vector<int> rows;
  rows.reserve(chunk_size_);
  if (c_.randomize_cpu) {
    const size_t num_rand = (size_t)(chunk_size_ / c_.random_access_chunk_size);
    if (random_indices_ind_ + num_rand > (size_t)dataset_size_) {
      Shuffle(random_indices_, cpu_rng_);
      random_indices_ind_ = 0;
    }
    for (size_t i = 0; i < num_rand; i++) {                         // LoadChunk(it, mat, random_rows), :290-307
      const int row = random_indices_[random_indices_ind_++];
      for (int k = 0; k < c_.random_access_chunk_size; k++) rows.push_back((row + k) % dataset_size_);
    }
  } else {
    for (int i = 0; i < chunk_size_; i++) {                         // LoadChunk(it, mat): GetNext, wrapping at the end
      rows.push_back(row_);
      if (++row_ == dataset_size_) row_ = 0;
    }
  }
  return rows;
}

DataSchedule::Batch DataSchedule::Next() {
  Batch b;
  int end = start_ + c_.batch_size;
  if (end > chunk_size_ || restart_) {
    if (reuse_counter_ < c_.max_reuse_count && !restart_) {
      reuse_counter_++;
    } else if (nothing_on_gpu_ || !fits_on_gpu_) {
      if (restart_ && c_.pipeline_loads) { preload_ = DiskAccess(); preloading_ = true; }    // StartPreload
      nothing_on_gpu_ = false;
      reuse_counter_ = 0;
      if (c_.pipeline_loads) { rows_ = preload_; preloading_ = false; }                   // PipelinedDiskAccess
      else rows_ = DiskAccess();
      b.loaded = true;
      if (c_.pipeline_loads) { preload_ = DiskAccess(); preloading_ = true; }
    }
    restart_ = false;
    if (c_.randomize_gpu) { Shuffle(perm_, gpu_rng_); b.reshuffled = true; }             // ShuffleIndices
    start_ = 0;
    end = c_.batch_size;
  }
  b.start = start_;
  b.multiplicity_id = multiplicity_counter_;
  if (++multiplicity_counter_ == c_.multiplicity) {
    multiplicity_counter_ = 0;
    start_ = end;
  }
  if (!preloading_) preload_.clear();
  return b;
}

// ---------------------------------------------------------------- DataHandler
DataHandler::DataHandler(const DatasetOrder& c, int dataset_size, int channels, int image_size_y, int image_size_x,
                         int gpu_image_size_y, int gpu_image_size_x, bool translate, bool flip, const float* images,
                         const int* labels, const float* targets, int target_dims, uint64_t seed)
    : schedule_(c, dataset_size, seed), channels_(channels), isy_(image_size_y), isx_(image_size_x), gy_(gpu_image_size_y),
      gx_(gpu_image_size_x), target_dims_(targets ? target_dims : 0), batch_(c.batch_size), images_(images), labels_(labels),
      targets_(targets), jitter_(image_size_y, image_size_x, gpu_image_size_y, gpu_image_size_x, translate, flip, seed) {
  if (channels <= 0 || gy_ <= 0 || gx_ <= 0 || gy_ > isy_ || gx_ > isx_)
    throw std::invalid_argument("DataHandler: the crop must fit the image");
  if (!images || (targets && target_dims <= 0)) throw std::invalid_argument("DataHandler: no images, or targets without a width");
  const size_t chunk = (size_t)schedule_.ChunkSize(), dims = (size_t)channels * isy_ * isx_;
  const int nbuf = schedule_.Pipelined() && !schedule_.FitsOnGpu() ? 2 : 1;
  for (int b = 0; b < nbuf; b++) {
    CUDA_CHECK(cudaMalloc((void**)&d_images_[b], sizeof(float) * chunk * dims));
    if (labels_) CUDA_CHECK(cudaMalloc((void**)&d_labels_[b], sizeof(int) * chunk));
    if (targets_) CUDA_CHECK(cudaMalloc((void**)&d_targets_[b], sizeof(float) * chunk * target_dims_));
  }
  CUDA_CHECK(cudaMalloc((void**)&d_perm_, sizeof(int) * chunk));
  CUDA_CHECK(cudaMallocHost((void**)&pinned_perm_, sizeof(int) * chunk * kRing));
  for (int k = 0; k < kRing; k++) CUDA_CHECK(cudaEventCreateWithFlags(&perm_done_[k], cudaEventDisableTiming));
  for (int b = 0; b < 2; b++) {
    CUDA_CHECK(cudaEventCreateWithFlags(&loaded_[b], cudaEventDisableTiming));
    CUDA_CHECK(cudaEventCreateWithFlags(&consumed_[b], cudaEventDisableTiming));
  }
  if (nbuf == 2) CUDA_CHECK(cudaStreamCreateWithFlags(&copy_stream_, cudaStreamNonBlocking));
  UploadPermutation();                                              // the identity, until a pass reshuffles it
}

DataHandler::~DataHandler() {
  cudaStreamSynchronize(Matrix::Stream());                          // crops and uploads may still read these buffers
  if (copy_stream_) { cudaStreamSynchronize(copy_stream_); cudaStreamDestroy(copy_stream_); }
  for (int b = 0; b < 2; b++) {
    cudaFree(d_images_[b]); cudaFree(d_labels_[b]); cudaFree(d_targets_[b]);
    cudaEventDestroy(loaded_[b]); cudaEventDestroy(consumed_[b]);
  }
  for (int k = 0; k < kRing; k++) cudaEventDestroy(perm_done_[k]);
  cudaFree(d_perm_);
  cudaFreeHost(pinned_perm_);
}

// the data set rows `rows` into chunk buffer `buf`, one copy per run of consecutive rows
void DataHandler::CopyRows(const std::vector<int>& rows, int buf, cudaStream_t s) {
  const size_t dims = (size_t)channels_ * isy_ * isx_;
  for (size_t i = 0; i < rows.size();) {
    size_t run = 1;
    while (i + run < rows.size() && rows[i + run] == rows[i] + (int)run) run++;
    const size_t r = (size_t)rows[i];
    CUDA_CHECK(cudaMemcpyAsync(d_images_[buf] + i * dims, images_ + r * dims, sizeof(float) * run * dims,
                               cudaMemcpyHostToDevice, s));
    if (labels_) CUDA_CHECK(cudaMemcpyAsync(d_labels_[buf] + i, labels_ + r, sizeof(int) * run, cudaMemcpyHostToDevice, s));
    if (targets_)
      CUDA_CHECK(cudaMemcpyAsync(d_targets_[buf] + i * target_dims_, targets_ + r * target_dims_,
                                 sizeof(float) * run * target_dims_, cudaMemcpyHostToDevice, s));
    i += run;
  }
}

void DataHandler::UploadPermutation() {
  const int slot = perm_slot_;
  perm_slot_ = (perm_slot_ + 1) % kRing;
  const std::vector<int>& perm = schedule_.Permutation();
  int* block = pinned_perm_ + (size_t)slot * perm.size();
  CUDA_CHECK(cudaEventSynchronize(perm_done_[slot]));               // the block's last copy has left it
  memcpy(block, perm.data(), sizeof(int) * perm.size());
  CUDA_CHECK(cudaMemcpyAsync(d_perm_, block, sizeof(int) * perm.size(), cudaMemcpyHostToDevice, Matrix::Stream()));
  CUDA_CHECK(cudaEventRecord(perm_done_[slot], Matrix::Stream()));
}

void DataHandler::Seek(int row) {
  schedule_.Seek(row);
  staged_ = false;                                                  // a copy still in flight is overwritten in stream order
}

void DataHandler::GetBatch(Matrix& input, int* labels_out, float* targets_out) {
  if (input.GetRows() != batch_ || input.GetCols() != channels_ * gy_ * gx_)
    throw std::invalid_argument("DataHandler::GetBatch: the input layer is not batch_size x channels * crop");
  if ((labels_out && !labels_) || (targets_out && !targets_))
    throw std::invalid_argument(std::string("DataHandler::GetBatch: the net trains on ") + (labels_out ? "labels" : "targets") +
                                " and the data set has none");
  const cudaStream_t s = Matrix::Stream();
  last_ = schedule_.Next();
  if (last_.loaded) {
    if (!copy_stream_) {
      CopyRows(schedule_.Rows(), cur_, s);
    } else {                                                        // WaitForPreload: swap in the staged chunk
      const int next = 1 - cur_;
      if (!staged_) {                                               // a preload begun within this GetBatch (a restart)
        CUDA_CHECK(cudaStreamWaitEvent(copy_stream_, consumed_[next], 0));
        CopyRows(schedule_.Rows(), next, copy_stream_);
        CUDA_CHECK(cudaEventRecord(loaded_[next], copy_stream_));
      }
      CUDA_CHECK(cudaStreamWaitEvent(s, loaded_[next], 0));
      CUDA_CHECK(cudaEventRecord(consumed_[cur_], s));              // behind the last crop that read the old chunk
      cur_ = next;
      staged_ = false;
      if (!schedule_.PreloadRows().empty()) {                       // StartPreload: the next chunk into the free buffer
        CUDA_CHECK(cudaStreamWaitEvent(copy_stream_, consumed_[1 - cur_], 0));
        CopyRows(schedule_.PreloadRows(), 1 - cur_, copy_stream_);
        CUDA_CHECK(cudaEventRecord(loaded_[1 - cur_], copy_stream_));
        staged_ = true;
      }
    }
  }
  if (last_.reshuffled) UploadPermutation();
  const float* noise = noise_.Stage(jitter_, batch_, last_.multiplicity_id);
  const int rc = cnb_extract_patches_indexed(d_images_[cur_], input.GetDevData(), d_perm_ + last_.start, noise,
                                             noise + batch_, noise + 2 * batch_, batch_, channels_, isx_, isy_, gx_, gy_,
                                             labels_out ? d_labels_[cur_] : nullptr, labels_out,
                                             targets_out ? d_targets_[cur_] : nullptr, targets_out, target_dims_);
  CheckCrop("DataHandler::GetBatch: cnb_extract_patches_indexed", rc);
}

void DataHandler::GetBatch(ConvNet& net) {
  Layer& out = net.OutputLayer();
  Matrix& targets = out.GetTargets();
  if (targets.GetNumEls() > 0) {
    if (targets.GetCols() != target_dims_)
      throw std::invalid_argument("DataHandler::GetBatch: the output layer takes " + std::to_string(targets.GetCols()) +
                                  " targets per image and the data set has " + std::to_string(target_dims_));
    GetBatch(net.InputLayer().GetState(), nullptr, targets.GetDevData());
  } else {
    GetBatch(net.InputLayer().GetState(), out.GetLabels(), nullptr);
  }
}

}  // namespace cnbhost
