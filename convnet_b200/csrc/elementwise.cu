// elementwise.cu — the memory-bound steps the Edge layer runs either side of the conv ops
// (bias add, bias gradient, ReLU, SGD).  See include/convnet_b200_ext.h for the reference
// call sites they correspond to.  All are single-pass, float4-vectorised where aligned.
#include <algorithm>
#include <vector>

#include <cuda_bf16.h>

#include "../../include/convnet_b200_ext.h"
#include "conv_kernels.h"

namespace cnb {

// optional bf16 twin of a float4 result (convnet_b200_emit_bf16_next): 8 more bytes per thread, no extra pass
__device__ __forceinline__ void emit4(__nv_bfloat16* out16, long long i4, const float4& v) {
  if (!out16) return;
  const __nv_bfloat162 lo = __floats2bfloat162_rn(v.x, v.y), hi = __floats2bfloat162_rn(v.z, v.w);
  uint2 o; o.x = *reinterpret_cast<const uint32_t*>(&lo); o.y = *reinterpret_cast<const uint32_t*>(&hi);
  reinterpret_cast<uint2*>(out16)[i4] = o;
}

static int blocks_for(long long work, int threads) {
  return (int)std::max<long long>(1, std::min<long long>(ceil_div<long long>(work, threads), (long long)num_sms() * 16));
}
__device__ __forceinline__ float4 ldg4(const float* p, long long i4) { return __ldg(reinterpret_cast<const float4*>(p) + i4); }

// Streaming passes over the n floats of x, in place: x[i] = op(x[i], op.at(i)), and the bf16 twin of the result when
// out16 is given.  One launch takes n4 float4 groups (op.at4(i4) gives the operands of group i4, read once) and then the
// scalar tail [4*n4, n).  The steps are the ones the fused epilogues apply (act_apply, act_deriv, dropout_keep), so a pass
// and the epilogue it stands in for compute the same bits.
//   ActOp       act_apply with a constant act: ReLU, logistic
//   ActDerivOp  act_deriv at the state s: ReLU', logistic'
//   MultOp      times m
//   DropOp      times the keep value of element i, which it also stores to mask when there is one
//   BiasOp      + bias[i / rows], then a constant act; rows % 4 == 0 on the vector body, so a group reads one bias value
template <int ACT>
struct ActOp {
  __device__ float at(long long) const { return 0.f; }
  __device__ float4 at4(long long) const { return make_float4(0.f, 0.f, 0.f, 0.f); }
  __device__ float operator()(float v, float) const { return act_apply(v, ACT); }
};
struct Operand {                                       // the operand is a second tensor, read alongside x
  const float* p;
  __device__ float at(long long i) const { return p[i]; }
  __device__ float4 at4(long long i4) const { return ldg4(p, i4); }
};
template <int ACT>
struct ActDerivOp : Operand {
  __device__ float operator()(float d, float s) const { return act_deriv(d, s, ACT); }
};
struct MultOp : Operand {
  __device__ float operator()(float v, float m) const { return v * m; }
};
struct DropOp {
  float* mask; float dropprob, scale; unsigned long long seed;
  __device__ float at(long long i) const {
    const float m = dropout_keep(seed + (unsigned long long)i, dropprob, scale);
    if (mask) mask[i] = m;
    return m;
  }
  __device__ float4 at4(long long i4) const {
    const unsigned long long e = seed + 4ULL * (unsigned long long)i4;
    const float4 m = make_float4(dropout_keep(e, dropprob, scale), dropout_keep(e + 1, dropprob, scale),
                                 dropout_keep(e + 2, dropprob, scale), dropout_keep(e + 3, dropprob, scale));
    if (mask) reinterpret_cast<float4*>(mask)[i4] = m;
    return m;
  }
  __device__ float operator()(float v, float m) const { return v * m; }
};
template <int ACT>
struct BiasOp {
  const float* bias; long long rows;
  __device__ float at(long long i) const { return __ldg(bias + i / rows); }
  __device__ float4 at4(long long i4) const { const float b = __ldg(bias + 4 * i4 / rows); return make_float4(b, b, b, b); }
  __device__ float operator()(float v, float b) const { return act_apply(v + b, ACT); }
};

// The vector body reads the operands before x, the tail x first.  That is what keeps BiasOp, whose operand read waits on a
// 64-bit division, at the speed and registers of the kernels it replaced: no float4 of x live across the division (20
// registers, not 26), and a scalar load of x in flight during it.
template <class Op>
__global__ void stream_kernel(float* x, long long n, long long n4, const Op op, __nv_bfloat16* out16) {
  const long long tid = blockIdx.x * (long long)blockDim.x + threadIdx.x, nt = (long long)gridDim.x * blockDim.x;
  for (long long i = tid; i < n4; i += nt) {
    const float4 s = op.at4(i);
    float4 v = reinterpret_cast<float4*>(x)[i];
    v.x = op(v.x, s.x); v.y = op(v.y, s.y); v.z = op(v.z, s.z); v.w = op(v.w, s.w);
    reinterpret_cast<float4*>(x)[i] = v;
    emit4(out16, i, v);
  }
  for (long long i = 4 * n4 + tid; i < n; i += nt) {
    const float xv = x[i], v = op(xv, op.at(i));
    x[i] = v;
    if (out16) out16[i] = __float2bfloat16_rn(v);
  }
}
// vec: x and the op's operands are 16-byte aligned (and, for BiasOp, rows % 4 == 0)
template <class Op>
static void stream_launch(float* x, long long n, bool vec, const Op& op, __nv_bfloat16* out16) {
  const long long n4 = vec ? n / 4 : 0;
  stream_kernel<<<blocks_for(std::max(n4, n - 4 * n4), 256), 256, 0, state().stream>>>(x, n, n4, op, out16);
}

// One pass writing the n floats of x, on the pending emit request (consumed even when there is nothing to write): the
// writer protocol around launch(out16), where out16 is the twin the kernel fills (nullptr unless can_emit).
template <class Launch>
static void write_pass(const char* what, float* x, long long n, bool can_emit, const Launch& launch) {
  const bool want = take_fuse().emit_bf16 != 0;
  if (n <= 0) return;
  Emit emit(x, n, want, can_emit);
  launch(emit.buf);
  count_launch(); CNB_LAUNCH_CHECK(what);
  emit.done = can_emit;
  emit.finish();
}
template <class Op>
static void stream_pass(const char* what, float* x, long long n, bool vec, bool can_emit, const Op& op) {
  write_pass(what, x, n, can_emit, [&](__nv_bfloat16* out16) { stream_launch(x, n, vec, op, out16); });
}

// Column reductions of a column-major [rows x cols] matrix (a column = one channel of a 2-D layer, DESIGN.md §3): one
// block per (column, row slice), a fixed summation order, no atomics.  Op accumulates Op::K quantities per element; slice
// s of column c leaves quantity k in part[(k * slices + s) * cols + c], and colsum_final_kernel<Fin> adds the slices up
// in slice order.  VEC (rows % 4 == 0, 16-byte aligned operands): float4 loads, slice boundaries on multiples of 4.
//   SumOp      the column sum: the bias gradient (scalar, the order it has always had) and the batch-norm mean
//   SqDevOp    sum of (x - mu[c])^2: the batch-norm variance, taken about the mean
//   BnGradOp   sum of d and of d * (x - mu[c]) / sigma[c]: the batch-norm backward pass
struct SumOp {
  static constexpr int K = 1;
  const float* a;
  struct Col { const float* p; };
  __device__ Col column(int c, long long rows) const { return {a + (long long)c * rows}; }
  __device__ void add(const Col& k, long long r, float* s) const { s[0] += __ldg(k.p + r); }
  __device__ void add4(const Col& k, long long r, float* s) const {
    const float4 v = ldg4(k.p, r);
    s[0] += (v.x + v.y) + (v.z + v.w);
  }
};
struct SqDevOp {
  static constexpr int K = 1;
  const float* a; const float* mu;
  struct Col { const float* p; float m; };
  __device__ Col column(int c, long long rows) const { return {a + (long long)c * rows, __ldg(mu + c)}; }
  __device__ void add(const Col& k, long long r, float* s) const { const float d = __ldg(k.p + r) - k.m; s[0] = __fmaf_rn(d, d, s[0]); }
  __device__ void add4(const Col& k, long long r, float* s) const {
    const float4 v = ldg4(k.p, r);
    const float a = v.x - k.m, b = v.y - k.m, c = v.z - k.m, d = v.w - k.m;
    s[0] += __fmaf_rn(a, a, b * b) + __fmaf_rn(c, c, d * d);
  }
};
struct BnGradOp {
  static constexpr int K = 2;
  const float* d; const float* x; const float* mu; const float* sigma;
  struct Col { const float* pd; const float* px; float m, inv; };
  __device__ Col column(int c, long long rows) const {
    return {d + (long long)c * rows, x + (long long)c * rows, __ldg(mu + c), 1.f / __ldg(sigma + c)};
  }
  __device__ void add(const Col& k, long long r, float* s) const {
    const float g = __ldg(k.pd + r), xh = (__ldg(k.px + r) - k.m) * k.inv;
    s[0] += g; s[1] = __fmaf_rn(g, xh, s[1]);
  }
  __device__ void add4(const Col& k, long long r, float* s) const {
    const float4 g = ldg4(k.pd, r), v = ldg4(k.px, r);
    s[0] += (g.x + g.y) + (g.z + g.w);
    s[1] += __fmaf_rn(g.x, (v.x - k.m) * k.inv, g.y * ((v.y - k.m) * k.inv)) +
            __fmaf_rn(g.z, (v.z - k.m) * k.inv, g.w * ((v.w - k.m) * k.inv));
  }
};

template <class Op, bool VEC>
__global__ void __launch_bounds__(256) colsum_partial_kernel(const Op op, float* __restrict__ part, long long rows, int cols,
                                                             int slices) {
  constexpr int K = Op::K;
  const int col = blockIdx.x, slice = blockIdx.y;
  const typename Op::Col k = op.column(col, rows);
  float s[K];
#pragma unroll
  for (int q = 0; q < K; q++) s[q] = 0.f;
  if (VEC) {
    const long long rv = rows / 4, per = ceil_div<long long>(rv, slices);
    const long long r0 = slice * per, r1 = min(rv, r0 + per);
    for (long long r = r0 + threadIdx.x; r < r1; r += blockDim.x) op.add4(k, r, s);
  } else {
    const long long per = ceil_div<long long>(rows, slices);
    const long long r0 = slice * per, r1 = min(rows, r0 + per);
    for (long long r = r0 + threadIdx.x; r < r1; r += blockDim.x) op.add(k, r, s);
  }
  __shared__ float sh[K][32];
#pragma unroll
  for (int q = 0; q < K; q++) {
    for (int o = 16; o > 0; o >>= 1) s[q] += __shfl_xor_sync(0xffffffffu, s[q], o);
    if ((threadIdx.x & 31) == 0) sh[q][threadIdx.x >> 5] = s[q];
  }
  __syncthreads();
  if (threadIdx.x < 32) {
#pragma unroll
    for (int q = 0; q < K; q++) {
      float t = threadIdx.x < (blockDim.x >> 5) ? sh[q][threadIdx.x] : 0.f;
      for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
      if (threadIdx.x == 0) part[((long long)q * slices + slice) * cols + col] = t;
    }
  }
}
// The per-column finish: the slices of each of the Fin::K quantities of column c, each added from 0 in slice order, and
// fin(c, sums) writes what the column's caller wants from them.
//   BiasGradFin  grad_bias = st * grad_bias + so * sum (the old value unread when st == 0)
//   MeanFin      the batch-norm mean
//   SigmaFin     sigma = sqrt(mean((x - mu)^2) + eps); the running averages (layer.cc:468-471) when run_mu is given
//   BnGradFin    grad_beta = mean(d), grad_gamma = mean(d * xhat) (the reference's 1/n scaling, layer.cc:493-496)
struct BiasGradFin {
  static constexpr int K = 1;
  float* out; float st, so;
  __device__ void operator()(int c, const float* s) const { out[c] = (st == 0.f) ? so * s[0] : st * out[c] + so * s[0]; }
};
struct MeanFin {
  static constexpr int K = 1;
  float* mu; float inv_n;
  __device__ void operator()(int c, const float* s) const { mu[c] = s[0] * inv_n; }
};
struct SigmaFin {
  static constexpr int K = 1;
  const float* mu; float* sigma; float* run_mu; float* run_sigma; float inv_n, eps, f;
  __device__ void operator()(int c, const float* s) const {
    const float sg = sqrtf(s[0] * inv_n + eps);
    sigma[c] = sg;
    if (run_mu) {
      run_mu[c] = __fmaf_rn(1.f - f, mu[c], f * run_mu[c]);
      run_sigma[c] = __fmaf_rn(1.f - f, sg, f * run_sigma[c]);
    }
  }
};
struct BnGradFin {
  static constexpr int K = 2;
  float* grad_gamma; float* grad_beta; float inv_n;
  __device__ void operator()(int c, const float* s) const { grad_beta[c] = s[0] * inv_n; grad_gamma[c] = s[1] * inv_n; }
};
template <class Fin>
__global__ void colsum_final_kernel(const float* __restrict__ part, int cols, int slices, const Fin fin) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= cols) return;
  float s[Fin::K];
#pragma unroll
  for (int q = 0; q < Fin::K; q++) s[q] = 0.f;
  for (int j = 0; j < slices; j++)
#pragma unroll
    for (int q = 0; q < Fin::K; q++) s[q] += part[((long long)q * slices + j) * cols + c];
  fin(c, s);
}
// the partial kernel into part (Op::K * slices * cols floats), then its finish
template <class Op, class Fin>
static void colsum(const char* what, const Op& op, const Fin& fin, float* part, long long rows, int cols, int slices, bool vec) {
  static_assert(Op::K == Fin::K, "a finish takes the quantities its partial kernel sums");
  const dim3 grid(cols, slices);
  if (vec) colsum_partial_kernel<Op, true><<<grid, 256, 0, state().stream>>>(op, part, rows, cols, slices);
  else colsum_partial_kernel<Op, false><<<grid, 256, 0, state().stream>>>(op, part, rows, cols, slices);
  colsum_final_kernel<<<ceil_div(cols, 128), 128, 0, state().stream>>>(part, cols, slices, fin);
  count_launch(2); CNB_LAUNCH_CHECK(what);
}

// Polyak average of k queue slots, laid out like stream_kernel (slot_stride % 4 == 0 on the vector body).  K > 0: k known
// at compile time, so the k loads of a float4 group are all issued before the first add; K == 0: any k
template <int K>
__global__ void __launch_bounds__(256) polyak_kernel(float* out, const float* __restrict__ queue, long long n, long long n4,
                                                     long long stride, int k, __nv_bfloat16* out16) {
  const int kk = K > 0 ? K : k;
  const float kf = (float)kk;
  const long long tid = blockIdx.x * (long long)blockDim.x + threadIdx.x, nt = (long long)gridDim.x * blockDim.x;
  for (long long i = tid; i < n4; i += nt) {
    float4 s[K > 0 ? K : 1];
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
    if (K > 0) {
#pragma unroll
      for (int j = 0; j < (K > 0 ? K : 1); j++) s[j] = __ldcs(reinterpret_cast<const float4*>(queue + j * stride) + i);
#pragma unroll
      for (int j = 0; j < (K > 0 ? K : 1); j++) { a.x += s[j].x; a.y += s[j].y; a.z += s[j].z; a.w += s[j].w; }
    } else {
#pragma unroll 4
      for (int j = 0; j < kk; j++) {
        const float4 v = __ldcs(reinterpret_cast<const float4*>(queue + j * stride) + i);
        a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w;
      }
    }
    a.x = __fdiv_rn(a.x, kf); a.y = __fdiv_rn(a.y, kf); a.z = __fdiv_rn(a.z, kf); a.w = __fdiv_rn(a.w, kf);
    reinterpret_cast<float4*>(out)[i] = a;
    emit4(out16, i, a);
  }
  for (long long i = 4 * n4 + tid; i < n; i += nt) {
    float a = 0.f;
    for (int j = 0; j < kk; j++) a += queue[j * stride + i];
    a = __fdiv_rn(a, kf);
    out[i] = a;
    if (out16) out16[i] = __float2bfloat16_rn(a);
  }
}

// ---- output layers (src/loss_functions.cc).  y, t, deriv: column-major [rows = images x cols], images fastest.  One
// thread per image walks its columns in order, so each per-image value is a fixed-order float sum; ConvNet adds the images
// up with sum_kernel.  Per column, with w = loss_function_weight (deriv may be NULL: the value alone, the performance
// metric of a loss):
//   SQUARED_ERROR                          deriv (y - t) * w          value 0.5 * sum (y - t)^2        (:39-53)
//   LINEAR_ERROR                           deriv w                    value sum (y - t)                (:55-68)
//   CROSS_ENTROPY_MULTINOMIAL (labels)     deriv (y - [c == l]) * w   value -log max(y[l], 1e-30)      (:70-83)
//   CROSS_ENTROPY_BINARY (t < 0: ignored)  deriv (y - t) * w, 0       value sum -t log(y + 1e-10) - (1 - t) log(1 - y + 1e-10)
//   CROSS_ENTROPY_MULTINOMIAL_DISTRIBUTED  deriv (y - t) * w          value sum -t log(y + 1e-10)      (:97-109)
// Every operation is rounded to nearest (logf: <= 1 ulp); sums accumulate left to right over the columns.
constexpr float kTiny = 1e-10f;
__global__ void loss_kernel(int loss, const float* __restrict__ y, const float* __restrict__ t, const int* __restrict__ labels,
                            float* deriv, float* value, int rows, int cols, float w) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= rows) return;
  const int lab = loss == CNB_LOSS_CROSS_ENTROPY_MULTINOMIAL ? labels[n] : -1;
  float s = 0.f;
  for (int c = 0; c < cols; c++) {
    const long long i = n + (long long)rows * c;
    const float yv = __ldg(y + i);
    const float tv = loss == CNB_LOSS_CROSS_ENTROPY_MULTINOMIAL ? (c == lab ? 1.f : 0.f) : __ldg(t + i);
    const float d = __fsub_rn(yv, tv);
    float g = d;
    switch (loss) {
      case CNB_LOSS_SQUARED_ERROR: s = __fmaf_rn(d, d, s); break;
      case CNB_LOSS_LINEAR_ERROR: s = __fadd_rn(s, d); g = 1.f; break;
      case CNB_LOSS_CROSS_ENTROPY_BINARY:
        if (tv < 0.f) { g = 0.f; break; }
        s = __fsub_rn(__fsub_rn(s, __fmul_rn(tv, logf(__fadd_rn(yv, kTiny)))),
                      __fmul_rn(__fsub_rn(1.f, tv), logf(__fadd_rn(__fsub_rn(1.f, yv), kTiny))));
        break;
      case CNB_LOSS_CROSS_ENTROPY_MULTINOMIAL_DISTRIBUTED: s = __fsub_rn(s, __fmul_rn(tv, logf(__fadd_rn(yv, kTiny)))); break;
      default: break;                                   // CROSS_ENTROPY_MULTINOMIAL: the value is the label's alone
    }
    if (deriv) deriv[i] = __fmul_rn(g, w);
  }
  if (loss == CNB_LOSS_SQUARED_ERROR) s = __fmul_rn(0.5f, s);
  if (loss == CNB_LOSS_CROSS_ENTROPY_MULTINOMIAL) s = -logf(fmaxf(__ldg(y + n + (long long)rows * lab), 1e-30f));
  value[n] = s;
}
// CLASSIFICATION_MULTINOMIAL: one warp per image decides the argmax as kSoftMaxCorrectRowMajor (cudamat_kernels.cu:1139,
// launched with 32 threads) does: lane j keeps the first strict maximum of columns j, j + 32, ... (from -FLT_MAX), then the
// lanes are compared in lane order, again strictly.  value = 1 when that column is the label.
__global__ void __launch_bounds__(256) classification_multinomial_kernel(const float* __restrict__ y, const int* __restrict__ labels,
                                                                         float* value, int rows, int cols) {
  const int lane = threadIdx.x & 31, n = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (n >= rows) return;
  float m = -3.402823466e38f;
  int arg = 0;
  for (int c = lane; c < cols; c += 32) {
    const float v = __ldg(y + n + (long long)rows * c);
    if (v > m) { m = v; arg = c; }
  }
  float bm = -3.402823466e38f;
  int barg = 0;
  for (int j = 0; j < 32; j++) {
    const float mj = __shfl_sync(0xffffffffu, m, j);
    const int aj = __shfl_sync(0xffffffffu, arg, j);
    if (mj > bm) { bm = mj; barg = aj; }
  }
  if (lane == 0) value[n] = barg == labels[n] ? 1.f : 0.f;
}
// CLASSIFICATION_BINARY (kLogisticCorrectNormalized, cudamat_kernels.cu:827): the share of the features with t >= 0 whose
// (t >= 0.5) == (y >= 0.5); 0 for an image without such features
__global__ void classification_binary_kernel(const float* __restrict__ y, const float* __restrict__ t, float* value, int rows,
                                             int cols) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= rows) return;
  float correct = 0.f, total = 0.f;
  for (int c = 0; c < cols; c++) {
    const long long i = n + (long long)rows * c;
    const float p = __ldg(y + i), tv = __ldg(t + i);
    if (tv < 0.f) continue;
    correct += ((tv >= 0.5f && p >= 0.5f) || (tv < 0.5f && p < 0.5f)) ? 1.f : 0.f;
    total += 1.f;
  }
  value[n] = total > 0.f ? correct / total : 0.f;
}

// Multi-tensor SGD (SGDOptimizer::Optimize, src/optimizer.cc:174-200): ONE launch updates every tensor of a batch (an
// all-reduce bucket, or the whole net).  The block -> tensor map is a prefix table that travels in the kernel parameters
// (no device-side descriptor to keep coherent).  Tensors whose staged bf16 copy exists (conv weights in bf16 mode) get it
// refreshed from the same registers.
//   Plain tensors: a block owns kSgdChunk consecutive elements.
//   Row-norm tensors (weight_norm_limit / weight_norm_constraint): the tensor is [rows x K] with the rows fastest, row r =
//   the elements r + rows*k (one output unit's incoming weights, DESIGN.md §3).  A block owns a tile of up to 128 rows x
//   (8192 / tile rows) columns, and while it stores the updated weights it also sums their squares per row; the tile's
//   per-row sums go to part[slab * rows + r] (slab = the tile's column range) in a fixed order — no atomics, so the
//   result is bit-reproducible.  norm_rescale_kernel then finishes the norms and rescales the rows that need it.
// Each tensor has a rule (Adagrad / RMSProp: AdagradSGDOptimizer / RMSPropSGDOptimizer::Optimize, optimizer.cc:202-279),
// uniform over its blocks; the adaptive rules also read and write a per-element state s.  The batch is larger than the
// classic 4 KB parameter limit: sm_70+ with CUDA 12.1+ takes up to 32 KB of kernel parameters.
constexpr int kSgdMaxTensors = 48, kSgdChunk = 4096, kNormTile = 8192, kNormRescaleRows = 32;
enum { kNormNone = 0, kNormLimit = 1, kNormConstraint = 2 };
enum { kRuleSgd = 0, kRuleAdagrad = 1, kRuleRmsProp = 2, kRuleAdagradState = 3 };   // the last: s only, w and h untouched
struct SgdItem {
  float* w; float* h; const float* g; __nv_bfloat16* w16; float* part;   // part: row-norm partial sums (norm tensors)
  float* s;                                                              // adaptive rules: the state
  long long n; float lr, mom, l2, clip, norm;
  float rp, scale;                                                       // Adagrad: delta, sqrt(step + 1); RMSProp: factor
  int rows, mode, vec, rule;
};
struct SgdBatch { int count; int first_block[kSgdMaxTensors + 1]; SgdItem t[kSgdMaxTensors]; };
static_assert(sizeof(SgdBatch) <= 32764, "kernel parameter limit");

__device__ __forceinline__ int batch_item(const SgdBatch& b) {
  int ti = 0;
  while (ti + 1 < b.count && (int)blockIdx.x >= b.first_block[ti + 1]) ti++;      // <= 48 uniform steps
  return ti;
}
// x / s, and 0 where x is 0: the reference's 0 / 0 (Adagrad with delta 0, RMSProp with factor 0 and a zero gradient) is NaN
__device__ __forceinline__ float safe_div(float x, float s) { return x == 0.f ? 0.f : __fdiv_rn(x, s); }
// One element, in this order.  Every operation is rounded to nearest and written with an intrinsic, so nothing is
// contracted and every tensor and block mapping computes the same bits; fma() is the one fused operation.
//   Adagrad:  e = s - delta;  s = delta + sqrt(e*e + g*g);  g = safe_div(g, s) * scale   (state only: stop here)
//   all:      d = fma(l2, w, g);  d = clamp(d, -clip, clip) if clip > 0
//   RMSProp:  s = sqrt((f*s)*s + ((1-f)*d)*d);  d = safe_div(d, s)
//   all:      h = fma(mom, h, lr*d);  w = w - h
// The SGD rule is exactly the update this kernel has always computed.
template <int R>
__device__ __forceinline__ void opt1(float& w, float& h, float& s, float g, const SgdItem& t) {
  if (R == kRuleAdagrad || R == kRuleAdagradState) {
    const float e = __fsub_rn(s, t.rp);
    s = __fadd_rn(t.rp, __fsqrt_rn(__fadd_rn(__fmul_rn(e, e), __fmul_rn(g, g))));
    if (R == kRuleAdagradState) return;
    g = __fmul_rn(safe_div(g, s), t.scale);
  }
  float d = __fmaf_rn(t.l2, w, g);
  if (t.clip > 0.f) d = d > t.clip ? t.clip : (d < -t.clip ? -t.clip : d);     // UpperBoundMod (keeps NaN)
  if (R == kRuleRmsProp) {
    s = __fsqrt_rn(__fadd_rn(__fmul_rn(__fmul_rn(t.rp, s), s), __fmul_rn(__fmul_rn(__fsub_rn(1.f, t.rp), d), d)));
    d = safe_div(d, s);
  }
  h = __fmaf_rn(t.mom, h, __fmul_rn(t.lr, d));
  w = __fsub_rn(w, h);
}
// element i of a tensor: load what rule R reads, update, store what it writes (and the bf16 twin of w)
template <int R>
__device__ __forceinline__ float opt_at(const SgdItem& t, long long i) {
  constexpr bool S = R != kRuleSgd, W = R != kRuleAdagradState;
  float w = W ? t.w[i] : 0.f, h = W ? t.h[i] : 0.f, s = S ? t.s[i] : 0.f;
  opt1<R>(w, h, s, t.g[i], t);
  if (S) t.s[i] = s;
  if (W) { t.h[i] = h; t.w[i] = w; if (t.w16) t.w16[i] = __float2bfloat16_rn(w); }
  return w;
}
// four elements from i (16-byte aligned operands)
template <int R>
__device__ __forceinline__ float4 opt_at4(const SgdItem& t, long long i) {
  constexpr bool S = R != kRuleSgd, W = R != kRuleAdagradState;
  const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
  float4 w = W ? *reinterpret_cast<const float4*>(t.w + i) : z, h = W ? *reinterpret_cast<const float4*>(t.h + i) : z;
  float4 s = S ? *reinterpret_cast<const float4*>(t.s + i) : z;
  const float4 g = __ldg(reinterpret_cast<const float4*>(t.g + i));
  opt1<R>(w.x, h.x, s.x, g.x, t); opt1<R>(w.y, h.y, s.y, g.y, t); opt1<R>(w.z, h.z, s.z, g.z, t); opt1<R>(w.w, h.w, s.w, g.w, t);
  if (S) *reinterpret_cast<float4*>(t.s + i) = s;
  if (W) {
    *reinterpret_cast<float4*>(t.h + i) = h;
    *reinterpret_cast<float4*>(t.w + i) = w;
    emit4(t.w16, i >> 2, w);
  }
  return w;
}
__host__ __device__ inline int norm_tile_rows(int rows) {                      // power of two <= 128
  int r = 1;
  while (r < rows && r < 128) r <<= 1;
  return r;
}
__host__ __device__ inline long long norm_slabs(const SgdItem& t) {
  return ceil_div<long long>(t.n / t.rows, kNormTile / norm_tile_rows(t.rows));
}

template <int R>
__device__ void sgd_chunk(const SgdItem& t, int block) {
  const long long e0 = (long long)block * kSgdChunk;
  const long long e1 = min(t.n, e0 + kSgdChunk);
  if (t.vec) {                                                                     // all pointers 16-byte aligned
    for (long long i = e0 + 4 * threadIdx.x; i < e1; i += 4 * 256) {
      if (i + 4 <= e1) opt_at4<R>(t, i);
      else for (long long j = i; j < e1; j++) opt_at<R>(t, j);
    }
  } else {
    for (long long i = e0 + threadIdx.x; i < e1; i += 256) opt_at<R>(t, i);
  }
}

// a row-norm tile.  vec (rows % 4 == 0, tile of 128 rows, aligned): lane = 4 consecutive rows (512 contiguous bytes per
// column and warp), warp = every 8th column of the tile's 64.  Otherwise: thread = one row and every (256 / tile rows)-th
// column.  Either way each thread holds the sums of its rows over its columns; red[] combines them in lane order.
template <int RULE>
__device__ void sgd_norm_tile(const SgdItem& t, int block, float* red) {
  const int R = norm_tile_rows(t.rows), C = kNormTile / R;
  const long long K = t.n / t.rows;
  const int strips = (int)ceil_div<long long>(t.rows, R);
  const int strip = block % strips;
  const long long slab = block / strips;
  const int r0 = strip * R;
  const long long c0 = slab * C, c1 = min(K, c0 + C);
  const int lanes = t.vec ? 8 : 256 / R;
  if (t.vec) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, r = r0 + 4 * lane;
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    if (r < t.rows) {
      for (long long k = c0 + warp; k < c1; k += 8) {
        const float4 w = opt_at4<RULE>(t, r + (long long)t.rows * k);
        s.x = __fmaf_rn(w.x, w.x, s.x); s.y = __fmaf_rn(w.y, w.y, s.y);
        s.z = __fmaf_rn(w.z, w.z, s.z); s.w = __fmaf_rn(w.w, w.w, s.w);
      }
    }
    reinterpret_cast<float4*>(red)[warp * 32 + lane] = s;                        // red[warp * 128 + row in tile]
  } else {
    const int rr = threadIdx.x % R, lane = threadIdx.x / R, r = r0 + rr;
    float s = 0.f;
    if (r < t.rows) {
      for (long long k = c0 + lane; k < c1; k += lanes) {
        const float wi = opt_at<RULE>(t, r + (long long)t.rows * k);
        s = __fmaf_rn(wi, wi, s);
      }
    }
    red[lane * R + rr] = s;
  }
  __syncthreads();
  if ((int)threadIdx.x < R && r0 + (int)threadIdx.x < t.rows) {
    float s = 0.f;
    for (int l = 0; l < lanes; l++) s += red[l * R + threadIdx.x];
    t.part[slab * t.rows + r0 + threadIdx.x] = s;
  }
}

__global__ void __launch_bounds__(256) sgd_multi_kernel(const __grid_constant__ SgdBatch b) {
  __shared__ __align__(16) float red[1024];
  const int ti = batch_item(b);
  const SgdItem& t = b.t[ti];
  const int block = (int)blockIdx.x - b.first_block[ti];
  if (t.mode == kNormNone) {
    switch (t.rule) {
      case kRuleSgd: sgd_chunk<kRuleSgd>(t, block); break;
      case kRuleAdagrad: sgd_chunk<kRuleAdagrad>(t, block); break;
      case kRuleRmsProp: sgd_chunk<kRuleRmsProp>(t, block); break;
      default: sgd_chunk<kRuleAdagradState>(t, block); break;
    }
  } else {
    switch (t.rule) {                                       // (a state-only tensor never has a norm rule: no update)
      case kRuleSgd: sgd_norm_tile<kRuleSgd>(t, block, red); break;
      case kRuleAdagrad: sgd_norm_tile<kRuleAdagrad>(t, block, red); break;
      default: sgd_norm_tile<kRuleRmsProp>(t, block, red); break;
    }
  }
}

// Second pass, norm tensors only: a block owns kNormRescaleRows rows.  It adds up each row's partial sums in slab order
// (warp w takes every 8th slab, then the 8 warp sums in warp order), takes the reference's scale (kNormLimitRowwise,
// cudamat_kernels.cu:1549-1569: c/|w| under a constraint, L/|w| where |w| > L under a limit) and rewrites the weights and
// their bf16 twin only in rows whose scale is not 1.  A limit no row exceeds costs the read of the partial sums.
// Deviation: under a constraint a row of norm 0 stays 0 (the reference writes 0 * inf = NaN there).
__global__ void __launch_bounds__(256) norm_rescale_kernel(const __grid_constant__ SgdBatch b) {
  __shared__ float red[8][kNormRescaleRows];
  __shared__ float scale[kNormRescaleRows];
  const int ti = batch_item(b);
  const SgdItem& t = b.t[ti];
  const int r0 = ((int)blockIdx.x - b.first_block[ti]) * kNormRescaleRows;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, r = r0 + lane;
  const long long slabs = norm_slabs(t), K = t.n / t.rows;
  float s = 0.f;
  if (r < t.rows)
    for (long long j = warp; j < slabs; j += 8) s += t.part[j * t.rows + r];
  red[warp][lane] = s;
  __syncthreads();
  if (warp == 0) {
    float ss = 0.f;
    for (int k = 0; k < 8; k++) ss += red[k][lane];
    const float nrm = sqrtf(ss);
    float sc = 1.f;
    if (r < t.rows && nrm > 0.f && (t.mode == kNormConstraint || nrm > t.norm)) sc = t.norm / nrm;
    scale[lane] = sc;
  }
  if (!__syncthreads_or(warp == 0 && scale[lane] != 1.f)) return;
  const float sc = scale[lane];
  if (r >= t.rows || sc == 1.f) return;
  for (long long k = warp; k < K; k += 8) {
    const long long i = r + (long long)t.rows * k;
    const float v = t.w[i] * sc;
    t.w[i] = v;
    if (t.w16) t.w16[i] = __float2bfloat16_rn(v);
  }
}

// ---- batch normalisation (Layer::ApplyBatchNormalization / ApplyDerivativeofBatchNormalization, src/layer.cc:452-510)
// The per-channel statistics are column reductions (colsum); the two elementwise passes run bn_channel_kernel<Op>.  Its
// block works inside one channel (blockIdx.y): op.channel reads that channel's constants once, and the block walks the
// channel's n values with a grid stride over blockIdx.x, t = op(k, t, x) on the target t, with the bf16 twin of t when
// out16 is given.  vec: n % 4 == 0 and x, t 16-byte aligned (a float4 never straddles two channels).
//   BnApplyOp  t = gamma * (x - mu) / sigma + beta, then a constant act (the old t is not read)
//   BnBackOp   in place: d = gamma / sigma * (d - mean(d) - xhat * mean(d * xhat)), xhat = (x - mu) / sigma; mean(d) and
//              mean(d * xhat) are grad_beta and grad_gamma (BnGradFin).  train == 0: d = gamma / sigma * d (the running
//              statistics are constants of the test-mode transform)
template <int ACT>
struct BnApplyOp {
  const float* gamma; const float* beta; const float* mu; const float* sigma;
  struct Ch { float m, a, b; };
  __device__ Ch channel(int c) const { return {__ldg(mu + c), __ldg(gamma + c) / __ldg(sigma + c), __ldg(beta + c)}; }
  __device__ float operator()(const Ch& k, float, float v) const { return act_apply(__fmaf_rn(v - k.m, k.a, k.b), ACT); }
};
struct BnBackOp {
  const float* gamma; const float* mu; const float* sigma; const float* grad_gamma; const float* grad_beta; int train;
  struct Ch { float m, inv, a, md, mdx; };
  __device__ Ch channel(int c) const {
    const float m = __ldg(mu + c), inv = 1.f / __ldg(sigma + c), a = __ldg(gamma + c) * inv;
    return {m, inv, a, train ? __ldg(grad_beta + c) : 0.f, train ? __ldg(grad_gamma + c) : 0.f};
  }
  __device__ float operator()(const Ch& k, float d, float v) const { return k.a * __fmaf_rn(-(v - k.m) * k.inv, k.mdx, d - k.md); }
};
template <class Op>
__global__ void __launch_bounds__(256) bn_channel_kernel(const float* __restrict__ x, float* __restrict__ t, long long n, int vec,
                                                         const Op op, __nv_bfloat16* out16) {
  const int c = blockIdx.y;
  const typename Op::Ch k = op.channel(c);
  const long long stride = (long long)gridDim.x * blockDim.x, base = (long long)c * n;
  if (vec) {
    const long long n4 = n / 4, b4 = base / 4;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += stride) {
      float4 d = reinterpret_cast<const float4*>(t)[b4 + i];
      const float4 v = ldg4(x, b4 + i);
      d.x = op(k, d.x, v.x); d.y = op(k, d.y, v.y); d.z = op(k, d.z, v.z); d.w = op(k, d.w, v.w);
      reinterpret_cast<float4*>(t)[b4 + i] = d;
      emit4(out16, b4 + i, d);
    }
  } else {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += stride) {
      const float v = op(k, t[base + i], __ldg(x + base + i));
      t[base + i] = v;
      if (out16) out16[base + i] = __float2bfloat16_rn(v);
    }
  }
}

int bn_slices(long long n, int channels) {
  const long long want = ceil_div<long long>(8LL * num_sms(), channels), most = std::max<long long>(1, n / 2048);
  return (int)std::max<long long>(1, std::min<long long>(std::min(want, most), 1024));
}
bool bn_vec(long long n, const void* a, const void* b) { return n % 4 == 0 && aligned16(a) && aligned16(b); }
dim3 bn_grid(long long n, int channels, bool vec) {
  const long long per = ceil_div<long long>(vec ? n / 4 : n, 256), fill = ceil_div<long long>(16LL * num_sms(), channels);
  return dim3((unsigned)std::max<long long>(1, std::min(per, fill)), (unsigned)channels);
}

// softmax over classes of a column-major [rows x cols] matrix: one block per 32 images; lane = image (coalesced
// along rows), the block's warps split the classes; max and sum combined through shared memory.
__global__ void __launch_bounds__(256) softmax_kernel(float* x, int rows, int cols) {
  __shared__ float red[8][33];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int n = blockIdx.x * 32 + lane;
  const bool ok = n < rows;
  float m = -INFINITY;
  if (ok) for (int c = w; c < cols; c += 8) m = fmaxf(m, x[n + (long long)rows * c]);
  red[w][lane] = m;
  __syncthreads();
  for (int k = 0; k < 8; k++) m = fmaxf(m, red[k][lane]);
  __syncthreads();
  float s = 0.f;
  if (ok) for (int c = w; c < cols; c += 8) { const float e = expf(x[n + (long long)rows * c] - m); x[n + (long long)rows * c] = e; s += e; }
  red[w][lane] = s;
  __syncthreads();
  s = 0.f;
  for (int k = 0; k < 8; k++) s += red[k][lane];
  const float inv = 1.f / s;
  if (ok) for (int c = w; c < cols; c += 8) x[n + (long long)rows * c] *= inv;
}
__global__ void softmax_ce_deriv_kernel(const float* __restrict__ p, const int* __restrict__ labels, float* deriv,
                                        float* loss, int rows, int cols) {
  // blockIdx.y walks the classes: one thread per (image, class slice) instead of one per image (1 block for batch 128)
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= rows) return;
  const int lab = labels[n];
  for (int c = blockIdx.y; c < cols; c += gridDim.y)
    deriv[n + (long long)rows * c] = p[n + (long long)rows * c] - (c == lab ? 1.f : 0.f);
  if (loss && blockIdx.y == 0) loss[n] = -logf(fmaxf(p[n + (long long)rows * lab], 1e-30f));
}
__global__ void sum_kernel(const float* __restrict__ a, float* out, int n) {   // single block
  float s = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) s += a[i];
  __shared__ float sh[32];
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    s = threadIdx.x < (blockDim.x >> 5) ? sh[threadIdx.x] : 0.f;
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (threadIdx.x == 0) *out = s;
  }
}

void colsum_finish(const float* part, float* grad_bias, int cols, int slices, float st, float so) {
  colsum_final_kernel<<<ceil_div(cols, 128), 128, 0, state().stream>>>(part, cols, slices, BiasGradFin{grad_bias, st, so});
  count_launch();
  CNB_LAUNCH_CHECK("colsum_finish");
}

// dropout without a mask tensor, writing the bf16 twin when given: the fallback of convnet_b200_fuse_next_dropout for calls
// whose kernel cannot apply it in the epilogue (the caller owns the staging bookkeeping of x)
void dropout_apply(float* x, long long n, float dropprob, float scale, unsigned long long seed, __nv_bfloat16* out16) {
  if (n <= 0) return;
  stream_launch(x, n, aligned16(x), DropOp{nullptr, dropprob, scale, seed}, out16);
  count_launch(); CNB_LAUNCH_CHECK("dropout_apply");
}

// crop + mirror + transpose of a minibatch out of an image-major chunk (cnb_extract_patches).  A 32 x 32 tile of
// (image, patch column) for one (patch row, colour) goes through shared memory: the reads run along a source row (128
// contiguous bytes per image, reversed when mirrored), the writes along the images (the fastest axis of the layer state).
// The reference's kernel maps threads to patch columns and so stores with a stride of N floats (cudamat_kernels.cu:1655).
// Batch image n reads chunk column index[n], or column n when index is null.
__device__ __forceinline__ void extract_patch_tile(const float* __restrict__ images, float* __restrict__ patches,
                                                   const float* __restrict__ width_offset,
                                                   const float* __restrict__ height_offset, const float* __restrict__ flip,
                                                   const int* __restrict__ index, int N, int W, int H, int pw, int ph, int C) {
  __shared__ float tile[32][33];
  const int row = (int)(blockIdx.z % (unsigned)ph), color = (int)(blockIdx.z / (unsigned)ph);
  const int n0 = blockIdx.y * 32, c0 = blockIdx.x * 32;
  for (int k = threadIdx.y; k < 32; k += 8) {
    const int n = n0 + k, dc = c0 + (int)threadIdx.x;
    if (n < N && dc < pw) {
      int sr = (int)height_offset[n] + row, sc = (int)width_offset[n] + dc;
      if (flip[n] > 0.5f) sc = W - sc - 1;
      sr = min(max(sr, 0), H - 1); sc = min(max(sc, 0), W - 1);
      const size_t col = index ? (size_t)__ldg(index + n) : (size_t)n;
      tile[k][threadIdx.x] = __ldg(images + sc + (size_t)W * (sr + (size_t)H * (color + (size_t)C * col)));
    }
  }
  __syncthreads();
  for (int k = threadIdx.y; k < 32; k += 8) {
    const int dc = c0 + k, n = n0 + (int)threadIdx.x;
    if (n < N && dc < pw) patches[n + (size_t)N * (dc + (size_t)pw * (row + (size_t)ph * color))] = tile[threadIdx.x][k];
  }
}
// The tile kernel above, plus, when an indexed launch asks for a gather, one tail slice of blocks (blockIdx.z == ph * C)
// that gathers the same 32 images' labels and targets.  Only the tail's blockIdx.x == 0 column works, so each image's
// label and target row is written once.  Without kIndexed the index and the tail test are compiled out, and the tile's
// arguments come first, so the plain crop compiles to the code of a kernel that takes only those: testing the index at
// run time made it 3.5 % slower (98 -> 101 us for 128 images cropped 256 -> 224, one H100 80GB HBM3 at 700 W).
template <bool kIndexed>
__global__ void __launch_bounds__(256) extract_patches_indexed_kernel(
    const float* __restrict__ images, float* __restrict__ patches, const float* __restrict__ width_offset,
    const float* __restrict__ height_offset, const float* __restrict__ flip, int N, int W, int H, int pw, int ph, int C,
    const int* __restrict__ index, const int* __restrict__ labels_src, int* __restrict__ labels_dst,
    const float* __restrict__ targets_src, float* __restrict__ targets_dst, int target_dims) {
  if (!kIndexed || blockIdx.z < (unsigned)(ph * C)) {
    extract_patch_tile(images, patches, width_offset, height_offset, flip, kIndexed ? index : nullptr, N, W, H, pw, ph, C);
    return;
  }
  if (blockIdx.x != 0) return;
  const int n0 = blockIdx.y * 32, t = threadIdx.x + 32 * threadIdx.y;
  const int rows = min(32, N - n0);
  if (labels_dst && t < rows) labels_dst[n0 + t] = __ldg(labels_src + __ldg(index + n0 + t));
  if (targets_dst)                                           // thread t: image t % 32, features t / 32, t / 32 + 8, ...
    for (int j = t >> 5; j < target_dims; j += 8) {
      const int n = n0 + (t & 31);
      if ((t & 31) < rows) targets_dst[n + (size_t)N * j] = __ldg(targets_src + (size_t)target_dims * __ldg(index + n) + j);
    }
}
}  // namespace cnb

using namespace cnb;

extern "C" {

int cnb_extract_patches(const float* images, float* patches, const int* index, const float* width_offset,
                        const float* height_offset, const float* flip, int N, int C, int W, int H, int pw, int ph,
                        const int* labels_src, int* labels_dst, const float* targets_src, float* targets_dst,
                        int target_dims) {
  if (N <= 0 || pw <= 0 || ph <= 0 || C <= 0) return 0;
  const int gather = labels_dst || targets_dst ? 1 : 0;
  if (!labels_src != !labels_dst || !targets_src != !targets_dst || (gather && !index)) return -1;
  if ((long long)ph * C + gather > 65535 || ceil_div(N, 32) > 65535) return -1;
  bf16_note_write(patches, (long long)N * pw * ph * C);
  if (targets_dst) bf16_note_write(targets_dst, (long long)N * target_dims);
  const dim3 grid((unsigned)ceil_div(pw, 32), (unsigned)ceil_div(N, 32), (unsigned)(ph * C + gather));
  const auto kernel = index ? extract_patches_indexed_kernel<true> : extract_patches_indexed_kernel<false>;
  kernel<<<grid, dim3(32, 8), 0, state().stream>>>(images, patches, width_offset, height_offset, flip, N, W, H, pw, ph, C,
                                                   index, labels_src, labels_dst, targets_src, targets_dst, target_dims);
  count_launch();
  return cudaGetLastError() == cudaSuccess ? 0 : -3;
}
int cnb_extract_patches_indexed(const float* images, float* patches, const int* index, const float* width_offset,
                                const float* height_offset, const float* flip, int N, int C, int W, int H, int pw,
                                int ph, const int* labels_src, int* labels_dst, const float* targets_src,
                                float* targets_dst, int target_dims) {
  if (N < 0 || C <= 0 || W <= 0 || H <= 0 || pw <= 0 || ph <= 0 || pw > W || ph > H || target_dims < 0) return -1;
  if (!images || !patches || !index || !width_offset || !height_offset || !flip) return -1;
  if (!labels_src != !labels_dst || !targets_src != !targets_dst || (targets_dst && target_dims == 0)) return -1;
  if (N == 0) return 0;
  if ((long long)ph * C + 1 > 65535 || ceil_div(N, 32) > 65535) return -1;
  return cnb_extract_patches(images, patches, index, width_offset, height_offset, flip, N, C, W, H, pw, ph, labels_src,
                             labels_dst, targets_src, targets_dst, target_dims);
}
void cnb_add_channel_bias(float* acts, const float* bias, long long rows, int cols) {
  stream_pass("add_channel_bias", acts, rows > 0 && cols > 0 ? rows * cols : 0, rows % 4 == 0 && aligned16(acts), false,
              BiasOp<kActNone>{bias, rows});
}
void cnb_add_channel_bias_relu(float* acts, const float* bias, long long rows, int cols) {
  stream_pass("add_channel_bias", acts, rows > 0 && cols > 0 ? rows * cols : 0, rows % 4 == 0 && aligned16(acts), false,
              BiasOp<kActRelu>{bias, rows});
}
// A device buffer that grows on demand.  The partial sums of the bias gradient and those of the SGD row norms each have
// their OWN, not the shared workspace: a host may run those passes on side streams beside conv kernels that are using the
// workspace, and beside each other (host/convnet.cc does).
struct GrowingScratch {
  float* buf = nullptr; size_t cap = 0; int dev = -1;
  float* get(size_t floats) {
    const int cur = current_device();
    if (buf && (cap < floats || dev != cur)) {
      CNB_CUDA_CHECK(cudaDeviceSynchronize());
      if (dev != cur) CNB_CUDA_CHECK(cudaSetDevice(dev));
      CNB_CUDA_CHECK(cudaFree(buf));
      if (dev != cur) CNB_CUDA_CHECK(cudaSetDevice(cur));
      buf = nullptr; cap = 0;
    }
    if (!buf) {
      const size_t want = std::max<size_t>(floats, (size_t)1 << 18);
      CNB_CUDA_CHECK(cudaMalloc((void**)&buf, want * sizeof(float)));
      cap = want; dev = cur;
    }
    return buf;
  }
};
static float* colsum_scratch(size_t floats) { static GrowingScratch s; return s.get(floats); }
// one buffer for every update call: calls are ordered on one stream (the optimizer's), so each may reuse it from the start
static float* sgd_norm_scratch(size_t floats) { static GrowingScratch s; return s.get(floats); }
void cnb_channel_bias_grad(const float* derivs, float* grad_bias, long long rows, int cols, float st, float so) {
  if (cols <= 0) return;
  int slices = (int)std::max<long long>(1, std::min<long long>(64, (4LL * num_sms()) / cols));
  slices = (int)std::min<long long>(slices, std::max<long long>(1, rows / 1024));
  float* part = colsum_scratch((size_t)slices * cols);
  colsum("channel_bias_grad", SumOp{derivs}, BiasGradFin{grad_bias, st, so}, part, rows, cols, slices, false);
}
void cnb_relu(float* x, long long n) { stream_pass("relu", x, n, aligned16(x), true, ActOp<kActRelu>{}); }
// its bf16 twin, when asked for, is a conversion pass
void cnb_relu_deriv(float* dx, const float* y, long long n) {
  stream_pass("relu_deriv", dx, n, aligned16(dx) && aligned16(y), false, ActDerivOp<kActRelu>{{y}});
}
void cnb_logistic(float* x, long long n) { stream_pass("logistic", x, n, aligned16(x), true, ActOp<kActLogistic>{}); }
void cnb_logistic_deriv(float* dx, const float* y, long long n) {
  stream_pass("logistic_deriv", dx, n, aligned16(dx) && aligned16(y), true, ActDerivOp<kActLogistic>{{y}});
}
static bool is_loss(int f) { return f >= CNB_LOSS_SQUARED_ERROR && f <= CNB_LOSS_CROSS_ENTROPY_MULTINOMIAL_DISTRIBUTED; }
void cnb_loss_deriv(int loss, const float* y, const float* targets, const int* labels, float* deriv, float* loss_per_image,
                    int rows, int cols, float weight) {
  CNB_REQUIRE(is_loss(loss), "cnb_loss_deriv");
  if (rows <= 0) return;
  if (loss == CNB_LOSS_CROSS_ENTROPY_MULTINOMIAL && weight == 1.f) {     // the kernel every softmax net has always run
    cnb_softmax_ce_deriv(y, labels, deriv, loss_per_image, rows, cols);
    return;
  }
  bf16_note_write(deriv, (long long)rows * cols);
  loss_kernel<<<ceil_div(rows, 128), 128, 0, state().stream>>>(loss, y, targets, labels, deriv, loss_per_image, rows, cols, weight);
  count_launch(); CNB_LAUNCH_CHECK("loss_deriv");
}
void cnb_metric(int metric, const float* y, const float* targets, const int* labels, float* metric_per_image, int rows, int cols) {
  CNB_REQUIRE(is_loss(metric) || metric == CNB_LOSS_CLASSIFICATION_MULTINOMIAL || metric == CNB_LOSS_CLASSIFICATION_BINARY,
              "cnb_metric");
  if (rows <= 0) return;
  if (metric == CNB_LOSS_CLASSIFICATION_MULTINOMIAL)
    classification_multinomial_kernel<<<ceil_div(rows, 8), 256, 0, state().stream>>>(y, labels, metric_per_image, rows, cols);
  else if (metric == CNB_LOSS_CLASSIFICATION_BINARY)
    classification_binary_kernel<<<ceil_div(rows, 128), 128, 0, state().stream>>>(y, targets, metric_per_image, rows, cols);
  else
    loss_kernel<<<ceil_div(rows, 128), 128, 0, state().stream>>>(metric, y, targets, labels, nullptr, metric_per_image, rows, cols, 1.f);
  count_launch(); CNB_LAUNCH_CHECK("metric");
}
void cnb_dropout(float* x, float* mask, long long n, float dropprob, float scale, unsigned long long seed) {
  write_pass("dropout", x, n, true, [&](__nv_bfloat16* out16) {
    bf16_note_write(mask, n);
    stream_launch(x, n, aligned16(x) && aligned16(mask), DropOp{mask, dropprob, scale, seed}, out16);
  });
}
void cnb_mult(float* a, const float* b, long long n) {
  stream_pass("mult", a, n, aligned16(a) && aligned16(b), true, MultOp{{b}});
}
void cnb_softmax(float* x, int rows, int cols) {
  if (rows <= 0) return;
  bf16_note_write(x, (long long)rows * cols);
  softmax_kernel<<<ceil_div(rows, 32), 256, 0, state().stream>>>(x, rows, cols);
  count_launch(); CNB_LAUNCH_CHECK("softmax");
}
void cnb_softmax_ce_deriv(const float* probs, const int* labels, float* deriv, float* loss_per_image, int rows, int cols) {
  if (rows <= 0) return;
  bf16_note_write(deriv, (long long)rows * cols);
  const dim3 grid(ceil_div(rows, 128), std::max(1, std::min(cols, 4 * num_sms() / std::max(1, ceil_div(rows, 128)))));
  softmax_ce_deriv_kernel<<<grid, 128, 0, state().stream>>>(probs, labels, deriv, loss_per_image, rows, cols);
  count_launch(); CNB_LAUNCH_CHECK("softmax_ce_deriv");
}
void cnb_sum(const float* a, float* out, int n) {
  sum_kernel<<<1, 256, 0, state().stream>>>(a, out, n);
  count_launch(); CNB_LAUNCH_CHECK("sum");
}
void cnb_opt_update_multi(const CnbOptTensorEx* tensors, int count) {
  // partial sums of every norm tensor of the call, laid out one after the other (slabs x rows each)
  size_t part_floats = 0;
  for (int i = 0; i < count; i++) {
    const CnbOptTensorEx& x = tensors[i];
    const CnbOptTensor& s = x.t;
    CNB_REQUIRE(x.rule == CNB_RULE_SGD || x.rule == CNB_RULE_ADAGRAD || x.rule == CNB_RULE_RMSPROP, "cnb_opt_update_multi");
    CNB_REQUIRE(x.rule == CNB_RULE_SGD || s.n <= 0 || x.state != nullptr, "cnb_opt_update_multi");
    CNB_REQUIRE(!x.state_only || x.rule == CNB_RULE_ADAGRAD, "cnb_opt_update_multi");
    if (s.n <= 0 || s.norm_mode == CNB_NORM_NONE || x.state_only) continue;
    CNB_REQUIRE(s.norm_mode == CNB_NORM_LIMIT || s.norm_mode == CNB_NORM_CONSTRAINT, "cnb_opt_update_multi");
    CNB_REQUIRE(s.rows > 0 && s.n % s.rows == 0 && s.norm_value > 0.f, "cnb_opt_update_multi");
    SgdItem t; t.n = s.n; t.rows = s.rows;
    part_floats += (size_t)norm_slabs(t) * s.rows;
  }
  float* part = part_floats ? sgd_norm_scratch(part_floats) : nullptr;
  for (int base = 0; base < count; base += kSgdMaxTensors) {
    SgdBatch b, nb;                                                 // update pass; rescale pass (norm tensors)
    b.count = 0; nb.count = 0;
    int blocks = 0, nblocks = 0;
    for (int i = base; i < count && i < base + kSgdMaxTensors; i++) {
      const CnbOptTensorEx& x = tensors[i];
      const CnbOptTensor& s = x.t;
      if (s.n <= 0) continue;
      SgdItem& t = b.t[b.count];
      t.w = s.w; t.h = s.hist; t.g = s.grad; t.n = s.n; t.lr = s.lr; t.mom = s.momentum; t.l2 = s.l2;
      t.clip = s.clip > 0.f ? s.clip : 0.f;
      t.mode = x.state_only ? CNB_NORM_NONE : s.norm_mode;
      t.norm = s.norm_value; t.rows = t.mode ? s.rows : 1; t.part = nullptr;
      t.s = x.rule == CNB_RULE_SGD ? nullptr : x.state;
      t.rp = x.rule_param; t.scale = x.scale;
      t.rule = x.state_only ? kRuleAdagradState
                            : (x.rule == CNB_RULE_ADAGRAD ? kRuleAdagrad : (x.rule == CNB_RULE_RMSPROP ? kRuleRmsProp : kRuleSgd));
      t.vec = (aligned16(s.w) && aligned16(s.hist) && aligned16(s.grad) && (!t.s || aligned16(t.s))) ? 1 : 0;
      if (t.mode) t.vec = t.vec && t.rows % 4 == 0 && norm_tile_rows(t.rows) == 128;
      if (t.s) bf16_note_write(t.s, s.n);
      if (t.rule == kRuleAdagradState) {                            // the weights stay as they are
        t.w16 = nullptr;
      } else {
        // the weights change: a staged bf16 copy of exactly this tensor is refreshed in the same pass, any other overlap dropped
        const bool had_copy = bf16_staged(s.w, s.n) != nullptr;    // only a copy somebody keeps valid is worth refreshing
        bf16_note_write(s.w, s.n);                  // every derived copy (bf16 twin, dgrad banks) goes stale ...
        t.w16 = had_copy ? bf16_refresh_slot(s.w, s.n) : nullptr;  // ... and the bf16 twin is rewritten by this kernel
      }
      b.first_block[b.count] = blocks;
      if (t.mode) {
        const long long slabs = norm_slabs(t);
        t.part = part;
        part += slabs * t.rows;
        blocks += (int)(ceil_div<long long>(t.rows, norm_tile_rows(t.rows)) * slabs);
        nb.t[nb.count] = t;
        nb.first_block[nb.count] = nblocks;
        nblocks += (int)ceil_div<long long>(t.rows, kNormRescaleRows);
        nb.count++;
      } else {
        blocks += (int)ceil_div<long long>(s.n, kSgdChunk);
      }
      b.count++;
    }
    if (b.count == 0) continue;
    b.first_block[b.count] = blocks;
    sgd_multi_kernel<<<blocks, 256, 0, state().stream>>>(b);
    count_launch(); CNB_LAUNCH_CHECK("opt_update_multi");
    if (nb.count == 0) continue;
    nb.first_block[nb.count] = nblocks;
    norm_rescale_kernel<<<nblocks, 256, 0, state().stream>>>(nb);
    count_launch(); CNB_LAUNCH_CHECK("sgd_norm_rescale");
  }
}
void cnb_polyak_average(float* out, const float* queue, long long n, long long slot_stride, int k) {
  CNB_REQUIRE(k >= 1 && slot_stride >= n && (n <= 0 || queue + (k - 1) * slot_stride + n <= out ||
                                             out + n <= queue), "cnb_polyak_average");
  write_pass("polyak_average", out, n, true, [&](__nv_bfloat16* o16) {
    const long long n4 = aligned16(out) && aligned16(queue) && slot_stride % 4 == 0 ? n / 4 : 0;
    const int grid = blocks_for(std::max(n4, n - 4 * n4), 256);
    switch (k) {
#define CNB_POLYAK_K(K) case K: polyak_kernel<K><<<grid, 256, 0, state().stream>>>(out, queue, n, n4, slot_stride, k, o16); break;
      CNB_POLYAK_K(1) CNB_POLYAK_K(2) CNB_POLYAK_K(3) CNB_POLYAK_K(4) CNB_POLYAK_K(5) CNB_POLYAK_K(6) CNB_POLYAK_K(7)
      CNB_POLYAK_K(8)
#undef CNB_POLYAK_K
      default: polyak_kernel<0><<<grid, 256, 0, state().stream>>>(out, queue, n, n4, slot_stride, k, o16);
    }
  });
}
void cnb_sgd_update_multi(const CnbOptTensor* tensors, int count) {
  std::vector<CnbOptTensorEx> t(count > 0 ? count : 0);
  for (int i = 0; i < count; i++) t[i] = CnbOptTensorEx{tensors[i], CNB_RULE_SGD, 0, nullptr, 0.f, 1.f};
  cnb_opt_update_multi(t.data(), count);
}
void cnb_sgd_momentum_multi(const CnbSgdTensor* tensors, int count) {
  std::vector<CnbOptTensor> t(count > 0 ? count : 0);
  for (int i = 0; i < count; i++) {
    const CnbSgdTensor& s = tensors[i];
    t[i] = CnbOptTensor{s.w, s.hist, s.grad, s.n, s.lr, s.momentum, s.l2, 0.f, 1, CNB_NORM_NONE, 0.f};
  }
  cnb_sgd_update_multi(t.data(), count);
}
void cnb_sgd_momentum(float* w, float* hist, const float* grad, long long n, float lr, float momentum, float l2) {
  const CnbOptTensor t = {w, hist, grad, n, lr, momentum, l2, 0.f, 1, CNB_NORM_NONE, 0.f};
  cnb_sgd_update_multi(&t, 1);
}

// ---- batch normalisation.  The reductions fill the machine at both ends of the layer shapes: a few channels of ~1.5 M
// values (row slices, about 8 blocks per SM in all) and thousands of channels of 128 values (one block per channel).
static float* bn_scratch(size_t floats) { static GrowingScratch s; return s.get(floats); }   // ordered on the caller's stream
void cnb_bn_stats(const float* x, long long n, int channels, float eps, float bn_f, float* batch_mu, float* batch_sigma,
                  float* run_mu, float* run_sigma) {
  if (n <= 0 || channels <= 0) return;
  CNB_REQUIRE(channels <= 65535 && (run_mu == nullptr) == (run_sigma == nullptr), "cnb_bn_stats");
  for (float* v : {batch_mu, batch_sigma, run_mu, run_sigma}) bf16_note_write(v, channels);
  const int slices = bn_slices(n, channels);
  const bool vec = n % 4 == 0 && aligned16(x);
  float* part = bn_scratch((size_t)slices * channels);
  const float inv_n = 1.f / (float)n;
  colsum("bn_mean", SumOp{x}, MeanFin{batch_mu, inv_n}, part, n, channels, slices, vec);
  colsum("bn_sigma", SqDevOp{x, batch_mu}, SigmaFin{batch_mu, batch_sigma, run_mu, run_sigma, inv_n, eps, bn_f}, part, n,
         channels, slices, vec);
}
void cnb_bn_apply(const float* x, float* y, long long n, int channels, const float* gamma, const float* beta, const float* mu,
                  const float* sigma, int relu) {
  write_pass("bn_apply", y, n > 0 && channels > 0 ? n * channels : 0, true, [&](__nv_bfloat16* out16) {
    CNB_REQUIRE(channels <= 65535, "cnb_bn_apply");
    const bool vec = bn_vec(n, x, y);
    const dim3 grid = bn_grid(n, channels, vec);
    if (relu) bn_channel_kernel<<<grid, 256, 0, state().stream>>>(x, y, n, vec, BnApplyOp<kActRelu>{gamma, beta, mu, sigma}, out16);
    else bn_channel_kernel<<<grid, 256, 0, state().stream>>>(x, y, n, vec, BnApplyOp<kActNone>{gamma, beta, mu, sigma}, out16);
  });
}
// the gradient means are reduced first: the elementwise pass reads them
void cnb_bn_backward(float* deriv, const float* x, long long n, int channels, const float* gamma, const float* mu,
                     const float* sigma, int train, float* grad_gamma, float* grad_beta) {
  write_pass("bn_backward", deriv, n > 0 && channels > 0 ? n * channels : 0, true, [&](__nv_bfloat16* out16) {
    CNB_REQUIRE(channels <= 65535, "cnb_bn_backward");
    const bool vec = bn_vec(n, x, deriv);
    bf16_note_write(grad_gamma, channels);
    bf16_note_write(grad_beta, channels);
    const int slices = bn_slices(n, channels);
    float* part = bn_scratch((size_t)2 * slices * channels);
    colsum("bn_grad", BnGradOp{deriv, x, mu, sigma}, BnGradFin{grad_gamma, grad_beta, 1.f / (float)n}, part, n, channels,
           slices, vec);
    bn_channel_kernel<<<bn_grid(n, channels, vec), 256, 0, state().stream>>>(
        x, deriv, n, vec, BnBackOp{gamma, mu, sigma, grad_gamma, grad_beta, train}, out16);
  });
}

}  // extern "C"
