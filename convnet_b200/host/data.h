// data.h — the device side of the reference's input pipeline (SURVEY.md §8 f4): a chunk of the data set resident on the GPU,
// one image per column, and per minibatch a crop + mirror + transpose into the input layer (src/datahandler.cc:146-200
// DataHandler::GetBatch, :520-531 DataIterator::AddNoise, :533-568 DataIterator::SampleNoise).  Reading the data set from
// disk (HDF5 / image lists) stays with the caller: it hands over float pixels in the reference's (colour, row, column)
// order, to DataIterator::Upload or in host memory to DataHandler.
// The two feeds share the per-minibatch work: Jitter draws the offsets and mirror bits, NoiseStage carries them to the
// device, and one crop launch cuts the batch (DataIterator: cnb_extract_patches on a contiguous slice of its chunk;
// DataHandler: cnb_extract_patches_indexed through a permutation, gathering the labels or targets in the same launch).
// What each owns apart from that is its chunk and how it fills it.
#pragma once
#include <cstdint>
#include <vector>

#include "matrix.h"

namespace cnbhost {

class ConvNet;

// splitmix64: the generator behind the jitter and the shuffles of DataSchedule
uint64_t SplitMix64(uint64_t& state);

// :533-568 — the jitter of one minibatch: random offsets when `translate`, else the centre / corner crop number
// multiplicity_id % 5; random mirror bits when `flip`, else multiplicity_id / 5.  Per image the height offset is drawn
// before the width offset, and the mirror bits after all offsets.
class Jitter {
 public:
  Jitter(int image_size_y, int image_size_x, int gpu_image_size_y, int gpu_image_size_x, bool translate, bool flip,
         uint64_t seed);
  // out[0, 3 * batch_size): width offsets | height offsets | mirror bits (mirrored when > 0.5)
  void Sample(int batch_size, int multiplicity_id, float* out);
  // the deterministic (translate == false) views of :547-556: centre, top-left, top-right, bottom-right, bottom-left
  static void ViewOffset(int multiplicity_id, int max_offset_x, int max_offset_y, int* w, int* h);

 private:
  int max_offset_y_, max_offset_x_;
  bool translate_, flip_;
  uint64_t rng_;
  float Uniform();                                // [0, 1)
};

// The jitter on its way to the crop: kRing pinned blocks that Jitter fills in place, each reused only after the event
// recorded behind its last copy, so no batch waits for the stream, and one device block of 3 x batch floats that the copy
// lands in and the crop reads.  A batch larger than any before grows both, once the stream has drained.
class NoiseStage {
 public:
  NoiseStage() = default;                         // creates nothing on the device: the first Stage does
  ~NoiseStage();
  // draws a batch's jitter and copies it on Matrix::Stream(); returns the device block
  const float* Stage(Jitter& jitter, int batch_size, int multiplicity_id);
  const float* Last() const { return last_; }     // host copy of the last batch's jitter, 3 x LastBatch() floats
  int LastBatch() const { return last_batch_; }   // 0 before the first

 private:
  static constexpr int kRing = 4;
  float* pinned_ = nullptr;                       // kRing blocks of 3 x cap_ floats
  float* device_ = nullptr;                       // 3 x cap_
  const float* last_ = nullptr;
  int cap_ = 0, last_batch_ = 0, slot_ = 0;
  cudaEvent_t done_[kRing] = {};
};

class DataIterator {
 public:
  // images of image_size_y x image_size_x x channels, `chunk_size` of them on the GPU; the net sees gpu_image_size_* crops
  DataIterator(int chunk_size, int channels, int image_size_y, int image_size_x, int gpu_image_size_y, int gpu_image_size_x,
               bool translate, bool flip, uint64_t seed);
  int ChunkSize() const { return chunk_size_; }
  int NumDims() const { return channels_ * image_size_y_ * image_size_x_; }
  // host pixels of images [first, first + count) of the chunk, image-major, each image (colour, row, column); async
  void Upload(const float* host, int first, int count);
  // the jitter of the next minibatch of batch_size images (Jitter::Sample), staged for AddNoise
  void SampleNoise(int batch_size, int multiplicity_id) { d_noise_ = noise_.Stage(jitter_, batch_size, multiplicity_id); }
  // :520-531 + GetBatch's slice: images [start, start + batch) of the chunk -> dest (batch x C*gy*gx, image fastest)
  void AddNoise(int start, Matrix& dest);
  const NoiseStage& Noise() const { return noise_; }

 private:
  int chunk_size_, channels_, image_size_y_, image_size_x_, gpu_image_size_y_, gpu_image_size_x_;
  Matrix data_;
  Jitter jitter_;
  NoiseStage noise_;
  const float* d_noise_ = nullptr;
};

// The fields of the reference's DatasetConfig (proto/convnet_config.proto:371-382) that decide the batch order, with the
// proto's defaults.  max_dataset_size and the data streams' file fields are the caller's business.
struct DatasetOrder {
  int batch_size = 1, chunk_size = 0, max_reuse_count = 0;
  int pipeline_loads = 0, randomize_cpu = 0, randomize_gpu = 0;
  int random_access_chunk_size = 1, multiplicity = 1;
};

// The reference's DataHandler state machine (src/datahandler.cc:124-315) without the data: which data set rows each chunk
// holds, which slice of the chunk each minibatch takes, its multiplicity_id, and the permutation it is read through.
// Rule for rule: GetBatch's start_ / restart_ / reuse_counter_ / multiplicity_counter_, DiskAccess's random_indices_ when
// randomize_cpu (blocks of random_access_chunk_size rows from random starts, wrapping at the end of the data set, the
// index reshuffled when too few are left) and consecutive rows with wrap-around otherwise (LoadChunk), the preload that
// pipeline_loads runs one chunk ahead (and that Seek discards), and a reshuffle of the GPU permutation on every pass.
// Shuffles are seeded Fisher-Yates (j = SplitMix64 % (i + 1) for i = n-1 .. 1), on one generator for the CPU side and one
// for the GPU side, so that pipelining does not change the order.  Configurations the reference cannot run correctly are
// refused with std::invalid_argument: a batch larger than the chunk, and a random_access_chunk_size that does not divide
// the chunk (the reference's LoadChunk writes past its chunk).
class DataSchedule {
 public:
  DataSchedule(const DatasetOrder& c, int dataset_size, uint64_t seed);
  struct Batch {
    bool loaded = false;           // a new chunk became resident before this batch: `rows` holds its data set rows
    bool reshuffled = false;       // the permutation was redrawn before this batch
    int start = 0, multiplicity_id = 0;
  };
  Batch Next();                    // DataHandler::GetBatch, :146-200
  void Seek(int row);              // DataHandler::Seek, :124-133
  int ChunkSize() const { return chunk_size_; }
  int DatasetSize() const { return dataset_size_; }
  int BatchSize() const { return c_.batch_size; }
  bool FitsOnGpu() const { return fits_on_gpu_; }
  bool Pipelined() const { return c_.pipeline_loads != 0; }
  const std::vector<int>& Rows() const { return rows_; }            // the resident chunk's data set rows
  const std::vector<int>& Permutation() const { return perm_; }     // batch image n is chunk column perm[start + n]
  // with pipeline_loads: the rows of the chunk being preloaded (empty when none is); a new preload begins after each load
  const std::vector<int>& PreloadRows() const { return preload_; }

 private:
  DatasetOrder c_;
  int dataset_size_, chunk_size_;
  bool fits_on_gpu_ = false, nothing_on_gpu_ = true, restart_ = true, preloading_ = false;
  int start_ = 0, reuse_counter_ = 0, multiplicity_counter_ = 0, row_ = 0;
  size_t random_indices_ind_ = 0;
  uint64_t cpu_rng_, gpu_rng_;
  std::vector<int> random_indices_, perm_, rows_, preload_;
  void Shuffle(std::vector<int>& v, uint64_t& rng);
  std::vector<int> DiskAccess();   // :232-264: the rows of the next chunk
};

// The reference's DataHandler over a data set the caller holds in host memory (pinned or not): images image-major, each
// (colour, row, column); optional labels (one int per image) and targets (target_dims floats per image).  The resident
// chunk lives on the GPU with its labels and targets; each minibatch is one cnb_extract_patches_indexed launch that crops
// through the schedule's permutation into the input layer and gathers the labels or targets the output layer takes.
// Streams: chunk copies without pipeline_loads, the jitter and permutation uploads, and the crop run on the library
// stream.  With pipeline_loads (and a data set larger than a chunk) the next chunk is copied into a second buffer on a
// copy stream of its own; that copy waits for an event recorded after the last crop that read the buffer, and the crop
// after the swap waits for the copy's event.  Jitter (NoiseStage) and permutations reach the device through rings of
// pinned blocks, each reused only after the event recorded behind its last copy: no stream is synchronised per batch.
class DataHandler {
 public:
  DataHandler(const DatasetOrder& c, int dataset_size, int channels, int image_size_y, int image_size_x,
              int gpu_image_size_y, int gpu_image_size_x, bool translate, bool flip, const float* images, const int* labels,
              const float* targets, int target_dims, uint64_t seed);
  ~DataHandler();
  // the next minibatch into `input` (batch x C*gy*gx, image fastest) and `labels_out` / `targets_out` (batch x
  // target_dims, column-major) when not null
  void GetBatch(Matrix& input, int* labels_out, float* targets_out);
  void GetBatch(ConvNet& net);     // into the net's input layer and its labels or targets, whichever its output takes
  void Seek(int row);
  const DataSchedule& Schedule() const { return schedule_; }
  const DataSchedule::Batch& LastBatch() const { return last_; }
  const NoiseStage& Noise() const { return noise_; }

 private:
  static constexpr int kRing = 4;
  DataSchedule schedule_;
  int channels_, isy_, isx_, gy_, gx_, target_dims_, batch_;
  const float* images_;
  const int* labels_;
  const float* targets_;
  Jitter jitter_;
  NoiseStage noise_;
  int cur_ = 0;                                    // which of the chunk buffers is resident
  float* d_images_[2] = {nullptr, nullptr};
  int* d_labels_[2] = {nullptr, nullptr};
  float* d_targets_[2] = {nullptr, nullptr};
  int* d_perm_ = nullptr;
  int* pinned_perm_ = nullptr;                     // kRing blocks of chunk ints
  cudaEvent_t perm_done_[kRing], loaded_[2], consumed_[2];
  int perm_slot_ = 0;
  bool staged_ = false;                            // the schedule's preload has been issued into buffer 1 - cur_
  cudaStream_t copy_stream_ = nullptr;            // with two chunk buffers only
  DataSchedule::Batch last_;
  void CopyRows(const std::vector<int>& rows, int buf, cudaStream_t s);
  void UploadPermutation();
};

}  // namespace cnbhost
