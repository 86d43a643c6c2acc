// matrix.h — host-side `Matrix` facade over the C ABI (GPU only).
//
// Mirror of the reference's src/matrix.h for the hot path: same class name, same
// static conv / pool / response-norm methods with the same argument meaning
// (src/matrix.cc:785-1011), so the Edge classes in edge.cc read like the reference's
// src/*_edge.cc.  A Matrix is a column-major rows x cols fp32 device matrix
// (rows = images) plus the logical Shape4D; slices are views into a parent
// allocation exactly like the reference's get_slice (owns_data = 0).
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <string>

#include "../../include/convnet_b200_conv_gemm.h"
#include "../../include/convnet_b200_ext.h"
#include "check.h"

namespace cnbhost {

class Matrix {
 public:
  Matrix();
  Matrix(int rows, int cols);
  ~Matrix();
  Matrix(const Matrix&) = delete;
  Matrix& operator=(const Matrix&) = delete;

  void AllocateGPUMemory(int rows, int cols);                 // src/matrix.cc:144
  void AllocateGPUMemory(int rows, int cols, const std::string& name) { AllocateGPUMemory(rows, cols); }
  void GetSlice(Matrix& slice, int start, int end);           // columns [start, end) as a view (src/matrix.cc:225)
  void Reshape(int rows, int cols);                           // one of them may be -1 (src/matrix.cc:198)
  void SetShape4D(int d1, int d2, int d3, int d4);
  void SetShape4D_like(Matrix& m) { shape_ = m.shape_; }
  Shape4D& GetShape4D() { return shape_; }
  cudamat* GetMat() { return &mat_; }
  int GetRows() const { return mat_.size[0]; }
  int GetCols() const { return mat_.size[1]; }
  size_t GetNumEls() const { return (size_t)mat_.size[0] * mat_.size[1]; }
  float* GetDevData() { return mat_.data_device; }

  void Set(float v);
  void CopyFromHost(const float* src, size_t n);              // async on the library stream
  void CopyToHost(float* dst, size_t n);                      // synchronous
  float ReadValue(size_t index);                              // grad_check.cc:20-35 (1-float D2H)
  void WriteValue(size_t index, float v);

  // elementwise steps the edges / layers use (libcudamat calls in the reference)
  void AddRowVec(Matrix& v);                                  // this[r, c] += v[c]        (cudamat.cu:1064)
  void SumRows(Matrix& target, float scale_targets, float scale);   // target[c] = st*target[c] + scale*sum_r this[r, c]
  void ApplyReLU();                                           // LowerBound(0)
  void ApplyDerivOfReLU(Matrix& state);                       // this *= (state > 0)
  void ApplySoftmax();

  // ---- the hot path: identical signatures to src/matrix.h ----
  static void ConvUp(Matrix& input, Matrix& w, Matrix& output, ConvDesc conv_desc, float scale_targets);
  static void ConvDown(Matrix& deriv_output, Matrix& w, Matrix& deriv_input, ConvDesc conv_desc, float scale_targets);
  static void ConvOutp(Matrix& input, Matrix& deriv_output, Matrix& dw, ConvDesc conv_desc, int partial_sum_y,
                       int partial_sum_x, float scale_targets, float scale_outputs);
  static void LocalUp(Matrix& input, Matrix& w, Matrix& output, ConvDesc conv_desc, float scale_targets);
  static void LocalDown(Matrix& deriv_output, Matrix& w, Matrix& deriv_input, ConvDesc conv_desc, float scale_targets);
  static void LocalOutp(Matrix& input, Matrix& deriv_output, Matrix& dw, ConvDesc conv_desc, float scale_targets,
                        float scale_outputs);
  static void Conv3DUp(Matrix& input, Matrix& w, Matrix& output, ConvDesc conv_desc, float scale_targets);
  static void Conv3DDown(Matrix& deriv_output, Matrix& w, Matrix& deriv_input, ConvDesc conv_desc, float scale_targets);
  static void Conv3DOutp(Matrix& input, Matrix& deriv_output, Matrix& dw, ConvDesc conv_desc, float scale_targets,
                         float scale_outputs);
  static void ConvMaxPool(Matrix& input, Matrix& output, ConvDesc conv_desc);
  static void ConvMaxPoolUndo(Matrix& input, Matrix& deriv_output, Matrix& output, Matrix& deriv_input,
                              ConvDesc conv_desc, float scale_targets);
  static void ConvAvgPool(Matrix& input, Matrix& output, ConvDesc conv_desc);
  static void ConvAvgPoolUndo(Matrix& input, Matrix& deriv_output, ConvDesc conv_desc, float scale_targets);
  static void ConvResponseNormCrossMap(Matrix& input, Matrix& output, int numFilters, int sizeF, float addScale,
                                       float powScale, bool blocked);
  static void ConvResponseNormCrossMap3D(Matrix& input, Matrix& output, int numFilters, int sizeF, float addScale,
                                         float powScale, bool blocked, int image_size_t);
  static void ConvResponseNormCrossMapUndo(Matrix& outGrads, Matrix& inputs, Matrix& acts, Matrix& targets,
                                           int numFilters, int sizeF, float addScale, float powScale, bool blocked);
  static void ConvResponseNormCrossMapUndo3D(Matrix& outGrads, Matrix& inputs, Matrix& acts, Matrix& targets,
                                             int numFilters, int sizeF, float addScale, float powScale, bool blocked,
                                             int image_size_t);

  // RGB -> YUV of a batch: input (images, 3 * pixels) holds the R, G and B planes, output gets Y, U and V (src/matrix.cc:1013)
  static void ConvRGBToYUV(Matrix& input, Matrix& output);

  static void SetupCUDADevice(int board);                     // src/matrix.cc:528
  static cudaStream_t Stream();

 private:
  cudamat mat_;
  Shape4D shape_;
  bool owns_;
};

}  // namespace cnbhost
