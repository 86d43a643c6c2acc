// matrix.cc — see matrix.h.  Thin dispatch to the C ABI, like src/matrix.cc:785-1011.
#include "matrix.h"

#include "../../include/convnet_b200_conv.h"

#include <stdexcept>
#include <string>
#include <vector>

namespace cnbhost {

cudaStream_t Matrix::Stream() { return (cudaStream_t)convnet_b200_get_stream(); }

Matrix::Matrix() : owns_(false) {
  mat_.data_host = nullptr; mat_.data_device = nullptr;
  mat_.on_device = 1; mat_.on_host = 0; mat_.size[0] = mat_.size[1] = 0;
  mat_.is_trans = 0; mat_.owns_data = 0; mat_.tex_obj = 0;
  shape_.shape[0] = shape_.shape[1] = shape_.shape[2] = shape_.shape[3] = 0;
}
Matrix::Matrix(int rows, int cols) : Matrix() { AllocateGPUMemory(rows, cols); }
Matrix::~Matrix() {
  if (owns_ && mat_.data_device) cudaFree(mat_.data_device);
}

void Matrix::AllocateGPUMemory(int rows, int cols) {
  if (owns_ && mat_.data_device) { CUDA_CHECK(cudaFree(mat_.data_device)); mat_.data_device = nullptr; }
  const size_t n = (size_t)rows * cols;
  if (n > 0) {
    CUDA_CHECK(cudaMalloc((void**)&mat_.data_device, n * sizeof(float)));
    CUDA_CHECK(cudaMemsetAsync(mat_.data_device, 0, n * sizeof(float), Stream()));        // the reference calloc's + uploads
  }
  owns_ = true; mat_.owns_data = 1;
  mat_.size[0] = rows; mat_.size[1] = cols;
  SetShape4D(rows, cols, 1, 1);
}

void Matrix::GetSlice(Matrix& slice, int start, int end) {
  if (slice.owns_ && slice.mat_.data_device) cudaFree(slice.mat_.data_device);
  slice.owns_ = false; slice.mat_.owns_data = 0;
  slice.mat_.data_device = mat_.data_device + (size_t)start * mat_.size[0];
  slice.mat_.size[0] = mat_.size[0]; slice.mat_.size[1] = end - start;
  slice.SetShape4D(mat_.size[0], end - start, 1, 1);
}

void Matrix::Reshape(int rows, int cols) {
  const size_t n = GetNumEls();
  if (rows < 0) rows = (int)(n / cols);
  if (cols < 0) cols = (int)(n / rows);
  if ((size_t)rows * cols != n)
    throw std::logic_error("Matrix::Reshape: " + std::to_string(rows) + " x " + std::to_string(cols) + " for " +
                           std::to_string(n) + " elements");
  mat_.size[0] = rows; mat_.size[1] = cols;
}

void Matrix::SetShape4D(int d1, int d2, int d3, int d4) {
  shape_.shape[0] = d1; shape_.shape[1] = d2; shape_.shape[2] = d3; shape_.shape[3] = d4;
}

void Matrix::Set(float v) {
  if (v == 0.f) { CUDA_CHECK(cudaMemsetAsync(mat_.data_device, 0, GetNumEls() * sizeof(float), Stream())); return; }
  // rare path (non-zero constants): host staging
  const std::vector<float> tmp(GetNumEls(), v);
  CUDA_CHECK(cudaMemcpyAsync(mat_.data_device, tmp.data(), GetNumEls() * sizeof(float), cudaMemcpyHostToDevice, Stream()));
  CUDA_CHECK(cudaStreamSynchronize(Stream()));
}
void Matrix::CopyFromHost(const float* src, size_t n) {
  CUDA_CHECK(cudaMemcpyAsync(mat_.data_device, src, n * sizeof(float), cudaMemcpyHostToDevice, Stream()));
}
void Matrix::CopyToHost(float* dst, size_t n) {
  CUDA_CHECK(cudaMemcpyAsync(dst, mat_.data_device, n * sizeof(float), cudaMemcpyDeviceToHost, Stream()));
  CUDA_CHECK(cudaStreamSynchronize(Stream()));
}
float Matrix::ReadValue(size_t index) {
  float v;
  CUDA_CHECK(cudaMemcpyAsync(&v, mat_.data_device + index, sizeof(float), cudaMemcpyDeviceToHost, Stream()));
  CUDA_CHECK(cudaStreamSynchronize(Stream()));
  return v;
}
void Matrix::WriteValue(size_t index, float v) {
  CUDA_CHECK(cudaMemcpyAsync(mat_.data_device + index, &v, sizeof(float), cudaMemcpyHostToDevice, Stream()));
  CUDA_CHECK(cudaStreamSynchronize(Stream()));
}

void Matrix::AddRowVec(Matrix& v) { cnb_add_channel_bias(mat_.data_device, v.GetDevData(), GetRows(), GetCols()); }
void Matrix::SumRows(Matrix& target, float scale_targets, float scale) {
  cnb_channel_bias_grad(mat_.data_device, target.GetDevData(), GetRows(), GetCols(), scale_targets, scale);
}
void Matrix::ApplyReLU() { cnb_relu(mat_.data_device, (long long)GetNumEls()); }
void Matrix::ApplyDerivOfReLU(Matrix& state) { cnb_relu_deriv(mat_.data_device, state.GetDevData(), (long long)GetNumEls()); }
void Matrix::ApplySoftmax() { cnb_softmax(mat_.data_device, GetRows(), GetCols()); }

// ---- the hot path (USE_GEMM branch of src/matrix.cc:785-1011) ---------------------------------------
void Matrix::ConvUp(Matrix& input, Matrix& w, Matrix& output, ConvDesc conv_desc, float scale_targets) {
  convUpGemm(input.GetMat(), w.GetMat(), output.GetMat(), &input.GetShape4D(), &w.GetShape4D(), &output.GetShape4D(),
             conv_desc, scale_targets);
}
void Matrix::ConvDown(Matrix& deriv_output, Matrix& w, Matrix& deriv_input, ConvDesc conv_desc, float scale_targets) {
  convDownGemm(deriv_output.GetMat(), w.GetMat(), deriv_input.GetMat(), &deriv_output.GetShape4D(), &w.GetShape4D(),
               &deriv_input.GetShape4D(), conv_desc, scale_targets);
}
void Matrix::ConvRGBToYUV(Matrix& input, Matrix& output) { RGBToYUV(input.GetMat(), output.GetMat()); }

void Matrix::ConvOutp(Matrix& input, Matrix& deriv_output, Matrix& dw, ConvDesc conv_desc, int, int,
                      float scale_targets, float scale_outputs) {
  convOutpGemm(input.GetMat(), deriv_output.GetMat(), dw.GetMat(), &input.GetShape4D(), &deriv_output.GetShape4D(),
               &dw.GetShape4D(), conv_desc, scale_targets, scale_outputs);
}
void Matrix::LocalUp(Matrix& input, Matrix& w, Matrix& output, ConvDesc conv_desc, float scale_targets) {   // :859-870
  localUpGemm(input.GetMat(), w.GetMat(), output.GetMat(), &input.GetShape4D(), &w.GetShape4D(), &output.GetShape4D(),
              conv_desc, scale_targets);
}
void Matrix::LocalDown(Matrix& deriv_output, Matrix& w, Matrix& deriv_input, ConvDesc conv_desc, float scale_targets) {
  localDownGemm(deriv_output.GetMat(), w.GetMat(), deriv_input.GetMat(), &deriv_output.GetShape4D(), &w.GetShape4D(),
                &deriv_input.GetShape4D(), conv_desc, scale_targets);
}
void Matrix::LocalOutp(Matrix& input, Matrix& deriv_output, Matrix& dw, ConvDesc conv_desc, float scale_targets,
                       float scale_outputs) {                                                                  // :883-893
  localOutpGemm(input.GetMat(), deriv_output.GetMat(), dw.GetMat(), &input.GetShape4D(), &deriv_output.GetShape4D(),
                &dw.GetShape4D(), conv_desc, scale_targets, scale_outputs);
}
void Matrix::Conv3DUp(Matrix& input, Matrix& w, Matrix& output, ConvDesc conv_desc, float scale_targets) {
  convUp3DGemm(input.GetMat(), w.GetMat(), output.GetMat(), &input.GetShape4D(), &w.GetShape4D(),
               &output.GetShape4D(), conv_desc, scale_targets);
}
void Matrix::Conv3DDown(Matrix& deriv_output, Matrix& w, Matrix& deriv_input, ConvDesc conv_desc, float scale_targets) {
  convDown3DGemm(deriv_output.GetMat(), w.GetMat(), deriv_input.GetMat(), &deriv_output.GetShape4D(),
                 &w.GetShape4D(), &deriv_input.GetShape4D(), conv_desc, scale_targets);
}
void Matrix::Conv3DOutp(Matrix& input, Matrix& deriv_output, Matrix& dw, ConvDesc conv_desc, float scale_targets,
                        float scale_outputs) {
  convOutp3DGemm(input.GetMat(), deriv_output.GetMat(), dw.GetMat(), &input.GetShape4D(),
                 &deriv_output.GetShape4D(), &dw.GetShape4D(), conv_desc, scale_targets, scale_outputs);
}
void Matrix::ConvMaxPool(Matrix& input, Matrix& output, ConvDesc conv_desc) {
  MaxPoolGemm(input.GetMat(), output.GetMat(), &input.GetShape4D(), &output.GetShape4D(), conv_desc, 0, 1);
}
void Matrix::ConvMaxPoolUndo(Matrix& input, Matrix& deriv_output, Matrix& output, Matrix& deriv_input,
                             ConvDesc conv_desc, float scale_targets) {
  MaxPoolUndoGemm(input.GetMat(), deriv_output.GetMat(), output.GetMat(), deriv_input.GetMat(), &input.GetShape4D(),
                  &deriv_output.GetShape4D(), conv_desc, scale_targets);
}
void Matrix::ConvAvgPool(Matrix& input, Matrix& output, ConvDesc conv_desc) {
  AvgPoolGemm(input.GetMat(), output.GetMat(), &input.GetShape4D(), &output.GetShape4D(), conv_desc, 0, 1);
}
void Matrix::ConvAvgPoolUndo(Matrix& input, Matrix& deriv_output, ConvDesc conv_desc, float scale_targets) {
  AvgPoolUndoGemm(input.GetMat(), deriv_output.GetMat(), &input.GetShape4D(), &deriv_output.GetShape4D(), conv_desc,
                  scale_targets);
}
void Matrix::ConvResponseNormCrossMap(Matrix& input, Matrix& output, int numFilters, int sizeF, float addScale,
                                      float powScale, bool blocked) {
  ResponseNormCrossMapGemm(input.GetMat(), output.GetMat(), numFilters, sizeF, addScale, powScale, blocked);
}
void Matrix::ConvResponseNormCrossMap3D(Matrix& input, Matrix& output, int numFilters, int sizeF, float addScale,
                                        float powScale, bool blocked, int image_size_t) {
  ResponseNormCrossMap3DGemm(input.GetMat(), output.GetMat(), numFilters, sizeF, addScale, powScale, blocked,
                             image_size_t);
}
void Matrix::ConvResponseNormCrossMapUndo(Matrix& outGrads, Matrix& inputs, Matrix& /*acts*/, Matrix& targets,
                                          int numFilters, int sizeF, float addScale, float powScale, bool blocked) {
  ResponseNormCrossMapUndoGemm(outGrads.GetMat(), inputs.GetMat(), targets.GetMat(), numFilters, sizeF, addScale,
                               powScale, blocked);
}
void Matrix::ConvResponseNormCrossMapUndo3D(Matrix& outGrads, Matrix& inputs, Matrix& /*acts*/, Matrix& targets,
                                            int numFilters, int sizeF, float addScale, float powScale, bool blocked,
                                            int image_size_t) {
  ResponseNormCrossMap3DUndoGemm(outGrads.GetMat(), inputs.GetMat(), targets.GetMat(), numFilters, sizeF, addScale,
                                 powScale, blocked, image_size_t);
}

void Matrix::SetupCUDADevice(int board) { CUDA_CHECK(cudaSetDevice(board)); }

}  // namespace cnbhost
