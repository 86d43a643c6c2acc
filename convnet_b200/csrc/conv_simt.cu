// conv_simt.cu — fp32 CUDA-core implicit-GEMM convolution (fprop / dgrad / wgrad).
//
// This is the exact-fp32 path: it serves (a) precision mode FP32 (run_grad_check,
// the reference's own 1e-4 kernel tolerance, py/test_conv.py:387) and (b) every
// shape the tensor-core path does not take (batch not a multiple of 4, untied
// filters, tiny channel counts).  No im2col buffer is materialised (the
// reference's kExpand/kWriteRows/kReadRows/kContract passes,
// cudamat_conv_gemm.cu:78-116,353-436, disappear) and dgrad is a deterministic
// gather instead of the reference's atomicAdd scatter.
//
// One templated 128x128x8 register-tiled SGEMM core; the three ops differ only in
// how a GEMM coordinate maps to memory (the `Problem` functors below).
#include <algorithm>

#include "conv_kernels.h"

namespace cnb {

constexpr int BM = 128, BN = 128, BK = 8, TM = 8, TN = 8, THREADS = 256;

// ---- problem functors --------------------------------------------------------------
// fprop:  D[m, o] = sum_k A[m, k] * B[k, o],  m = n + N*module, k = x + kx*(y + ky*c)
struct FpropProblem {
  const float* __restrict__ img; const float* __restrict__ flt; float* out;
  int N, W, H, modX, modules, Cout, kx, ky, sx, sy, px, py, K;
  long long M;                  // N * modules
  long long flt_z, img_z, out_z;  // per-blockIdx.z strides (untied module / 3-D frame)
  int z_is_module;              // untied: z = module and M = N
  float st, so;
  const float* bias; int act;   // fused epilogue (convnet_b200_fuse_next_act); untied: one bias per output feature
  __device__ __forceinline__ long long rows() const { return M; }
  __device__ __forceinline__ int cols() const { return Cout; }
  __device__ __forceinline__ int depth() const { return K; }
  struct Row { int n, sX, sY; };
  __device__ __forceinline__ Row row(long long m, int z) const {
    int n, mod;
    if (z_is_module) { n = (int)m; mod = z; } else { n = (int)(m % N); mod = (int)(m / N); }
    Row r; r.n = n; r.sX = (mod % modX) * sx + px; r.sY = (mod / modX) * sy + py; return r;
  }
  __device__ __forceinline__ float loadA(const Row& r, int k, int z) const {
    const int x = k % kx, t = k / kx, y = t % ky, c = t / ky;
    const int X = r.sX + x, Y = r.sY + y;
    if ((unsigned)X >= (unsigned)W || (unsigned)Y >= (unsigned)H) return 0.f;
    return __ldg(img + (z_is_module ? 0 : z * img_z) + r.n + (long long)N * (X + (long long)W * (Y + (long long)H * c)));
  }
  __device__ __forceinline__ float loadB(int k, int o, int z) const {
    return __ldg(flt + (z_is_module ? z * flt_z : 0) + o + (long long)Cout * k);
  }
  __device__ __forceinline__ void store(long long m, int o, float acc, int z) const {
    float* t = out + (z_is_module ? (long long)z * N : z * out_z) + m + (long long)N * modules * o;
    float r = (st == 0.f) ? so * acc : st * (*t) + so * acc;
    if (bias) r += __ldg(bias + (z_is_module ? z + (long long)modules * o : o));
    if (act) r = act_apply(r, act);
    *t = r;
  }
};

// dgrad (gather): D[m, c] = sum_k A[m, k] * B[k, c], m = n + N*(X + W*Y), k = o + Cout*(x + kx*y)
struct DgradProblem {
  const float* __restrict__ der; const float* __restrict__ flt; float* out;
  int N, W, H, modX, modY, modules, Cout, Cin, kx, ky, sx, sy, px, py, K;
  long long M;                  // N * W * H
  long long der_z, out_z;       // 3-D frame strides (sequential launches use z = 0)
  int untied;
  float st, so;
  const float* mask; int mask_act;   // fused activation derivative act_deriv(., mask, mask_act): same layout as out
  __device__ __forceinline__ long long rows() const { return M; }
  __device__ __forceinline__ int cols() const { return Cin; }
  __device__ __forceinline__ int depth() const { return K; }
  struct Row { int n, X, Y; };
  __device__ __forceinline__ Row row(long long m, int) const {
    Row r; r.n = (int)(m % N); const int p = (int)(m / N); r.X = p % W; r.Y = p / W; return r;
  }
  // module touched by tap (x, y) at input pixel (X, Y), or -1
  __device__ __forceinline__ int module_of(const Row& r, int x, int y) const {
    const int ax = r.X - px - x, ay = r.Y - py - y;
    if (ax < 0 || ay < 0) return -1;
    const int mx = ax / sx, my = ay / sy;
    if (mx * sx != ax || my * sy != ay || mx >= modX || my >= modY) return -1;
    return mx + modX * my;
  }
  __device__ __forceinline__ float loadA(const Row& r, int k, int z) const {
    const int o = k % Cout, tap = k / Cout, x = tap % kx, y = tap / kx;
    const int mod = module_of(r, x, y);
    if (mod < 0) return 0.f;
    return __ldg(der + z * der_z + r.n + (long long)N * (mod + (long long)modules * o));
  }
  __device__ __forceinline__ float loadB(int k, int c, int) const {
    const int o = k % Cout, tap = k / Cout;
    return __ldg(flt + o + (long long)Cout * (tap + (long long)kx * ky * c));
  }
  __device__ __forceinline__ void store(long long m, int c, float acc, int z) const {
    float* t = out + z * out_z + m + M * c;
    float r = (st == 0.f) ? so * acc : st * (*t) + so * acc;
    if (mask) r = act_deriv(r, __ldg(mask + z * out_z + m + M * c), mask_act);
    *t = r;
  }
};

// wgrad: P[z][o, k] = sum_r A[o, r] * B[r, k],  r = n + N*(module within chunk z)
// chunk z = (frame f, module rectangle); written to a partial buffer, reduced afterwards.
struct WgradProblem {
  const float* __restrict__ img; const float* __restrict__ der; float* part;
  float* out; float st, so;       // part == nullptr: block z is written straight to out + z*Cout*K
  int N, W, H, modX, modules, Cout, kx, ky, sx, sy, px, py, K;
  int chunksX, chunksPerFrame, rectW, rectH, modY;     // chunk -> module rectangle
  long long img_f, der_f;                              // 3-D frame strides
  __device__ __forceinline__ long long rows() const { return Cout; }
  __device__ __forceinline__ int cols() const { return K; }
  struct Row { int o; };
  __device__ __forceinline__ Row row(long long m, int) const { Row r; r.o = (int)m; return r; }
  __device__ __forceinline__ void rect(int z, int& f, int& mx0, int& my0, int& w, int& h) const {
    f = z / chunksPerFrame; const int c = z % chunksPerFrame;
    mx0 = (c % chunksX) * rectW; my0 = (c / chunksX) * rectH;
    w = min(rectW, modX - mx0); h = min(rectH, modY - my0);
  }
  __device__ __forceinline__ int depth_z(int z) const {
    int f, mx0, my0, w, h; rect(z, f, mx0, my0, w, h); return N * w * h;
  }
  // reduction index r -> (n, module)
  __device__ __forceinline__ void decode(int r, int z, int& n, int& mx, int& my, int& f) const {
    int mx0, my0, w, h; rect(z, f, mx0, my0, w, h);
    n = r % N; const int q = r / N; mx = mx0 + q % w; my = my0 + q / w;
  }
  __device__ __forceinline__ float loadA(const Row& row, int r, int z) const {
    int n, mx, my, f; decode(r, z, n, mx, my, f);
    return __ldg(der + f * der_f + n + (long long)N * (mx + modX * my + (long long)modules * row.o));
  }
  __device__ __forceinline__ float loadB(int r, int k, int z) const {
    int n, mx, my, f; decode(r, z, n, mx, my, f);
    const int x = k % kx, t = k / kx, y = t % ky, c = t / ky;
    const int X = mx * sx + px + x, Y = my * sy + py + y;
    if ((unsigned)X >= (unsigned)W || (unsigned)Y >= (unsigned)H) return 0.f;
    return __ldg(img + f * img_f + n + (long long)N * (X + (long long)W * (Y + (long long)H * c)));
  }
  __device__ __forceinline__ void store(long long o, int k, float acc, int z) const {
    const long long idx = (long long)z * Cout * K + o + (long long)Cout * k;
    if (part) { part[idx] = acc; return; }
    out[idx] = (st == 0.f) ? so * acc : st * out[idx] + so * acc;
  }
};

// untied dgrad, one module per launch: D[n, k] = sum_o der[n, mod, o] * w_mod[o, k], scattered
// into that module's window (launches are stream-ordered, so overlapping windows do not race).
struct LocalDownProblem {
  const float* __restrict__ der; const float* __restrict__ flt; float* out;
  int N, W, H, modules, Cout, kx, ky, K, sX, sY, mod;
  float so;
  __device__ __forceinline__ long long rows() const { return N; }
  __device__ __forceinline__ int cols() const { return K; }
  __device__ __forceinline__ int depth() const { return Cout; }
  struct Row { int n; };
  __device__ __forceinline__ Row row(long long m, int) const { Row r; r.n = (int)m; return r; }
  __device__ __forceinline__ float loadA(const Row& r, int o, int) const {
    return __ldg(der + r.n + (long long)N * (mod + (long long)modules * o));
  }
  __device__ __forceinline__ float loadB(int o, int k, int) const {
    return __ldg(flt + o + (long long)Cout * k);
  }
  __device__ __forceinline__ void store(long long n, int k, float acc, int) const {
    const int x = k % kx, t = k / kx, y = t % ky, c = t / ky;
    const int X = sX + x, Y = sY + y;
    if ((unsigned)X >= (unsigned)W || (unsigned)Y >= (unsigned)H) return;
    out[n + (long long)N * (X + (long long)W * (Y + (long long)H * c))] += so * acc;
  }
};

template <class P> __device__ __forceinline__ int depth_of(const P& p, int) { return p.depth(); }
template <> __device__ __forceinline__ int depth_of<WgradProblem>(const WgradProblem& p, int z) { return p.depth_z(z); }

// ---- the SGEMM core ----------------------------------------------------------------
template <class P>
__global__ void __launch_bounds__(THREADS) simt_gemm_kernel(P p) {
  __shared__ float As[BK][BM + 4];
  __shared__ float Bs[BK][BN + 4];
  const int z = blockIdx.z;
  const long long m0 = (long long)blockIdx.x * BM;
  const int n0 = blockIdx.y * BN;
  const int tid = threadIdx.x;
  const int tx = tid % 16, ty = tid / 16;          // 16 x 16 threads, each TM x TN
  const long long Mrows = p.rows();
  const int Ncols = p.cols();
  const int depth = depth_of(p, z);

  // loader mapping: A tile BK x BM = 1024 elements -> 4 per thread; row index fastest (coalesced)
  const int a_m = tid % BM;                         // 0..127
  const int a_k0 = tid / BM;                        // 0..1  (+2*i)
  const bool a_ok = (m0 + a_m) < Mrows;
  typename P::Row arow = p.row(a_ok ? m0 + a_m : 0, z);
  const int b_n = tid % BN;
  const int b_k0 = tid / BN;
  const bool b_ok = (n0 + b_n) < Ncols;

  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; i++)
#pragma unroll
    for (int j = 0; j < TN; j++) acc[i][j] = 0.f;

  float ra[4], rb[4];
  auto gload = [&](int k0) {
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const int k = k0 + a_k0 + 2 * i;
      ra[i] = (a_ok && k < depth) ? p.loadA(arow, k, z) : 0.f;
      const int kb = k0 + b_k0 + 2 * i;
      rb[i] = (b_ok && kb < depth) ? p.loadB(kb, n0 + b_n, z) : 0.f;
    }
  };
  gload(0);
  for (int k0 = 0; k0 < depth; k0 += BK) {
#pragma unroll
    for (int i = 0; i < 4; i++) {
      As[a_k0 + 2 * i][a_m] = ra[i];
      Bs[b_k0 + 2 * i][b_n] = rb[i];
    }
    __syncthreads();
    if (k0 + BK < depth) gload(k0 + BK);
#pragma unroll
    for (int kk = 0; kk < BK; kk++) {
      float a[TM], b[TN];
#pragma unroll
      for (int i = 0; i < TM; i++) a[i] = As[kk][tx + 16 * i];
#pragma unroll
      for (int j = 0; j < TN; j++) b[j] = Bs[kk][ty + 16 * j];
#pragma unroll
      for (int i = 0; i < TM; i++)
#pragma unroll
        for (int j = 0; j < TN; j++) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int j = 0; j < TN; j++) {
    const int n = n0 + ty + 16 * j;
    if (n >= Ncols) continue;
#pragma unroll
    for (int i = 0; i < TM; i++) {
      const long long m = m0 + tx + 16 * i;      // consecutive tx -> consecutive rows: coalesced
      if (m < Mrows) p.store(m, n, acc[i][j], z);
    }
  }
}

template <class P>
static void launch(const P& p, long long M, int Ncols, int Z) {
  dim3 grid((unsigned)ceil_div<long long>(M, BM), (unsigned)ceil_div(Ncols, BN), (unsigned)Z);
  simt_gemm_kernel<P><<<grid, THREADS, 0, state().stream>>>(p);
  count_launch();
  CNB_LAUNCH_CHECK("conv_simt");
}

// ---- scale / reduce helpers --------------------------------------------------------
__global__ void scale_kernel(float* a, long long n, float s) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    a[i] = (s == 0.f) ? 0.f : a[i] * s;
}

void scale_buffer(float* a, long long n, float s) {
  if (s == 1.f || n <= 0) return;
  if (s == 0.f) { CNB_CUDA_CHECK(cudaMemsetAsync(a, 0, sizeof(float) * n, state().stream)); return; }
  const int blocks = (int)std::min<long long>(ceil_div<long long>(n, 256), 4 * num_sms());
  scale_kernel<<<blocks, 256, 0, state().stream>>>(a, n, s);
  count_launch();
  CNB_LAUNCH_CHECK("scale");
}

// out[g][i] = st*out[g][i] + so * sum_{j<per} part[(g*per + j)][i]      (deterministic order)
__global__ void reduce_partials_kernel(const float* __restrict__ part, float* out, long long elems,
                                       int groups, int per, float st, float so) {
  const long long total = elems * groups;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const long long g = idx / elems, i = idx % elems;
    float s = 0.f;
    for (int j = 0; j < per; j++) s += part[(g * per + j) * elems + i];
    out[idx] = (st == 0.f) ? so * s : st * out[idx] + so * s;
  }
}

// groups == 1, everything 16-byte aligned: four floats per thread, no index arithmetic
__global__ void __launch_bounds__(256) reduce_partials_v4_kernel(const float4* __restrict__ part, float4* out, long long elems4,
                                                                 int per, float st, float so) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < elems4; i += (long long)gridDim.x * blockDim.x) {
    float4 s = part[i];
    for (int j = 1; j < per; j++) {
      const float4 v = part[i + j * elems4];
      s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
    }
    s.x *= so; s.y *= so; s.z *= so; s.w *= so;
    if (st != 0.f) { const float4 o = out[i]; s.x += st * o.x; s.y += st * o.y; s.z += st * o.z; s.w += st * o.w; }
    out[i] = s;
  }
}

void reduce_partials(const float* part, float* out, long long elems, int groups, int per, float st, float so) {
  if (groups == 1 && elems % 4 == 0 && aligned16(part) && aligned16(out)) {
    const long long e4 = elems / 4;
    const int blocks = (int)std::min<long long>(std::max<long long>(ceil_div<long long>(e4, 256), 1), 8LL * num_sms());
    reduce_partials_v4_kernel<<<blocks, 256, 0, state().stream>>>((const float4*)part, (float4*)out, e4, per, st, so);
    count_launch();
    CNB_LAUNCH_CHECK("reduce_partials");
    return;
  }
  const long long total = elems * groups;
  const int blocks = (int)std::min<long long>(ceil_div<long long>(total, 256), 8 * num_sms());
  reduce_partials_kernel<<<blocks, 256, 0, state().stream>>>(part, out, elems, groups, per, st, so);
  count_launch();
  CNB_LAUNCH_CHECK("reduce_partials");
}

// ---- host entry points -------------------------------------------------------------
void simt_conv_up(const ConvGeom& g, const float* images, const float* filters, float* targets,
                  float scaleTargets, float scaleOutput, const Fuse& fuse) {
  FpropProblem p;
  p.bias = fuse.bias ? fuse.bias + (long long)g.cout0 * (g.conv ? 1 : g.modules) : nullptr; p.act = fuse.act;
  p.img = images + (long long)g.cin0 * g.H * g.W * g.N;
  p.flt = filters;
  p.out = targets + (long long)g.cout0 * g.modules * g.N;
  p.N = g.N; p.W = g.W; p.H = g.H; p.modX = g.modX; p.modules = g.modules; p.Cout = g.Cout;
  p.kx = g.kx; p.ky = g.ky; p.sx = g.sx; p.sy = g.sy; p.px = g.px; p.py = g.py; p.K = g.K;
  p.st = scaleTargets; p.so = scaleOutput;
  p.flt_z = (long long)g.Cout * g.K; p.img_z = g.in_frame_step; p.out_z = g.out_frame_step;
  if (g.conv) {
    p.z_is_module = 0; p.M = (long long)g.N * g.modules;
    launch(p, p.M, g.Cout, g.frames);
  } else {
    p.z_is_module = 1; p.M = g.N;
    launch(p, p.M, g.Cout, g.modules);
  }
}

void simt_local_down(const ConvGeom& g, const float* derivs, const float* filters, float* targets,
                     float scaleTargets, float scaleOutput) {
  CNB_REQUIRE(g.frames == 1, "localDown is 2-D only");
  scale_buffer(targets, g.img_total, scaleTargets);
  LocalDownProblem p;
  p.der = derivs + (long long)g.cout0 * g.modules * g.N;
  p.out = targets + (long long)g.cin0 * g.H * g.W * g.N;
  p.N = g.N; p.W = g.W; p.H = g.H; p.modules = g.modules; p.Cout = g.Cout;
  p.kx = g.kx; p.ky = g.ky; p.K = g.K; p.so = scaleOutput;
  for (int m = 0; m < g.modules; m++) {
    p.mod = m; p.flt = filters + (long long)m * g.Cout * g.K;
    p.sX = (m % g.modX) * g.sx + g.px; p.sY = (m / g.modX) * g.sy + g.py;
    launch(p, g.N, g.K, 1);
  }
}

void simt_conv_down(const ConvGeom& g, const float* derivs, const float* filters, float* targets,
                    float scaleTargets, float scaleOutput, const Fuse& fuse) {
  if (!g.conv) { simt_local_down(g, derivs, filters, targets, scaleTargets, scaleOutput); return; }
  DgradProblem p;
  p.mask = nullptr; p.mask_act = 0;
  p.der = derivs + (long long)g.cout0 * g.modules * g.N;
  p.flt = filters;
  p.out = targets + (long long)g.cin0 * g.H * g.W * g.N;
  p.N = g.N; p.W = g.W; p.H = g.H; p.modX = g.modX; p.modY = g.modY; p.modules = g.modules;
  p.Cout = g.Cout; p.Cin = g.Cin; p.kx = g.kx; p.ky = g.ky; p.sx = g.sx; p.sy = g.sy;
  p.px = g.px; p.py = g.py; p.K = g.Cout * g.kx * g.ky; p.untied = 0;
  p.M = (long long)g.N * g.W * g.H;
  p.der_z = 0; p.out_z = 0; p.so = scaleOutput;
  // The reference scales the WHOLE target (all channels, all frames) first (gemm.cu:760, conv3d:98).
  if (g.frames == 1 && g.cin0 == 0 && g.Cin == g.CinT) {
    p.st = scaleTargets;
    p.mask = fuse.act_state; p.mask_act = fuse.state_act;
    launch(p, p.M, g.Cin, 1);
    return;
  }
  const long long in_frame = g.in_frame_step;    // floats per stride_t frames
  scale_buffer(targets, g.img_total, scaleTargets);
  p.st = 1.f;
  for (int f = 0; f < g.frames; f++) {           // sequential: windows of successive frames overlap
    DgradProblem q = p;
    q.der = p.der + f * g.out_frame_step;
    q.out = p.out + f * in_frame;
    launch(q, q.M, g.Cin, 1);
  }
}

// wgrad into `chunks_y x chunks_x` (per frame) partial blocks, then grouped reduction.
//   groups == 1            : everything summed into one [Cout x K] target (ABI-1, and split-R)
//   groups == chunks       : ABI-2 partial sums, one target block per module rectangle
void simt_conv_outp(const ConvGeom& g, const float* images, const float* derivs, float* targets,
                    int rectH, int rectW, bool keep_partials, float scaleTargets, float scaleOutput) {
  WgradProblem p;
  p.img = images + (long long)g.cin0 * g.H * g.W * g.N;
  p.der = derivs + (long long)g.cout0 * g.modules * g.N;
  p.N = g.N; p.W = g.W; p.H = g.H; p.modX = g.modX; p.modY = g.modY; p.modules = g.modules;
  p.Cout = g.Cout; p.kx = g.kx; p.ky = g.ky; p.sx = g.sx; p.sy = g.sy; p.px = g.px; p.py = g.py;
  p.K = g.K;
  p.rectW = rectW; p.rectH = rectH;
  p.chunksX = ceil_div(g.modX, rectW);
  p.chunksPerFrame = p.chunksX * ceil_div(g.modY, rectH);
  p.img_f = g.in_frame_step; p.der_f = g.out_frame_step;
  const int Z = p.chunksPerFrame * g.frames;
  const long long elems = (long long)g.Cout * g.K;
  p.out = targets; p.st = scaleTargets; p.so = scaleOutput; p.part = nullptr;
  if (keep_partials) CNB_REQUIRE(g.frames == 1, "partial-sum wgrad is 2-D only");
  if (keep_partials || Z == 1) {       // every chunk owns its output block: no scratch, no 2nd pass
    launch(p, g.Cout, g.K, Z);
    return;
  }
  p.part = (float*)workspace(sizeof(float) * elems * Z);
  launch(p, g.Cout, g.K, Z);
  reduce_partials(p.part, targets, elems, 1, Z, scaleTargets, scaleOutput);
}

// ---- convInnerpGemm: per filter tap, the inner product of the image patches with the derivative of the same channel ------
// targets[tx + kx*ty] = st * targets[.] + so * sum over images n, modules m and channels c of
//                       image(n, X(m) + tx, Y(m) + ty, c) * derivs(n, m, c)          (zero outside the image)
// which is what the reference computes by expanding the patches (kExpand), multiplying by the derivative
// (kOutpTraceMultiplyImages) and summing with two cuBLAS gemv passes (gemm.cu:963-1115).  Here no patch matrix exists: CTA
// `split` owns a contiguous range of (channel, module) pairs with all their images, every thread keeps the sums of up to
// INNERP_TAPS taps in registers (the derivative is read once per pass over the taps), and a fixed-shape block reduction
// leaves one partial sum per tap: the target itself when there is one CTA, else a partial-sum row that reduce_partials
// adds in split order.  Deterministic, no atomics.
constexpr int INNERP_TAPS = 16;
constexpr int INNERP_THREADS = 256;

struct InnerpArgs {
  const float* img; const float* der; float* out;   // out: the target (splits == 1) or the partial sums [split][taps]
  int N, W, H, modX, modules, kx, ky, sx, sy, px, py, taps;
  long long pairs, per_split;                        // (channel, module) pairs, pairs per CTA
  float st, so;
};

template <int VEC> __device__ __forceinline__ void ip_load(const float* p, float (&v)[VEC]);
template <> __device__ __forceinline__ void ip_load<4>(const float* p, float (&v)[4]) {
  const float4 t = __ldg(reinterpret_cast<const float4*>(p)); v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
}
template <> __device__ __forceinline__ void ip_load<1>(const float* p, float (&v)[1]) { v[0] = __ldg(p); }

template <int VEC>
__global__ void __launch_bounds__(INNERP_THREADS) innerp_kernel(InnerpArgs a, int final_pass) {
  __shared__ float red[INNERP_THREADS / 32][INNERP_TAPS];
  const int NV = a.N / VEC;
  const long long p0 = (long long)blockIdx.x * a.per_split, p1 = min(a.pairs, p0 + a.per_split);
  const long long units = (p1 - p0) * NV;
  for (int t0 = 0; t0 < a.taps; t0 += INNERP_TAPS) {
    float acc[INNERP_TAPS];
#pragma unroll
    for (int t = 0; t < INNERP_TAPS; t++) acc[t] = 0.f;
    for (int u = threadIdx.x; u < (int)units; u += INNERP_THREADS) {
      const long long pair = p0 + u / NV;
      const int nv = u % NV;
      const int c = (int)(pair / a.modules), m = (int)(pair % a.modules);
      const int X0 = (m % a.modX) * a.sx + a.px, Y0 = (m / a.modX) * a.sy + a.py;
      float d[VEC];
      ip_load<VEC>(a.der + (long long)a.N * pair + nv * VEC, d);     // derivs(n, m, c) at n + N*(m + modules*c)
      const float* img = a.img + (long long)a.N * a.W * a.H * c + nv * VEC;
#pragma unroll
      for (int t = 0; t < INNERP_TAPS; t++) {
        const int tap = t0 + t;
        if (tap >= a.taps) break;
        const int ty = tap / a.kx, tx = tap - ty * a.kx;
        const int X = X0 + tx, Y = Y0 + ty;
        if ((unsigned)X >= (unsigned)a.W || (unsigned)Y >= (unsigned)a.H) continue;
        float v[VEC];
        ip_load<VEC>(img + (long long)a.N * (X + (long long)a.W * Y), v);
#pragma unroll
        for (int e = 0; e < VEC; e++) acc[t] += v[e] * d[e];
      }
    }
#pragma unroll
    for (int t = 0; t < INNERP_TAPS; t++)
      for (int o = 16; o > 0; o >>= 1) acc[t] += __shfl_xor_sync(0xffffffffu, acc[t], o);
    if ((threadIdx.x & 31) == 0) {
#pragma unroll
      for (int t = 0; t < INNERP_TAPS; t++) red[threadIdx.x >> 5][t] = acc[t];
    }
    __syncthreads();
    const int tap = t0 + threadIdx.x;
    if (threadIdx.x < INNERP_TAPS && tap < a.taps) {
      float s = 0.f;
      for (int w = 0; w < INNERP_THREADS / 32; w++) s += red[w][threadIdx.x];
      if (final_pass) a.out[tap] = (a.st == 0.f) ? a.so * s : a.st * a.out[tap] + a.so * s;
      else a.out[(long long)blockIdx.x * a.taps + tap] = s;
    }
    __syncthreads();
  }
}

int conv_innerp(const ConvGeom& g, const float* images, const float* derivs, float* targets, float st, float so, int splits) {
  InnerpArgs a;
  a.img = images + (long long)g.cin0 * g.H * g.W * g.N;
  a.der = derivs + (long long)g.cout0 * g.modules * g.N;
  a.N = g.N; a.W = g.W; a.H = g.H; a.modX = g.modX; a.modules = g.modules;
  a.kx = g.kx; a.ky = g.ky; a.sx = g.sx; a.sy = g.sy; a.px = g.px; a.py = g.py; a.taps = g.kx * g.ky;
  a.pairs = (long long)g.Cin * g.modules;
  a.st = st; a.so = so;
  // about 16K image values per CTA, at most two waves of CTAs
  if (splits <= 0)
    splits = (int)std::min<long long>(std::max<long long>(1, ceil_div<long long>(a.pairs * g.N, 16384)), 2LL * num_sms());
  a.per_split = ceil_div<long long>(a.pairs, splits);
  splits = (int)ceil_div<long long>(a.pairs, a.per_split);
  CNB_REQUIRE(a.per_split * g.N < (1LL << 31), "convInnerpGemm: too many images x modules per channel");
  const bool v4 = g.N % 4 == 0 && aligned16(images) && aligned16(derivs) && aligned16(a.img) && aligned16(a.der);
  float* part = splits > 1 ? (float*)workspace(sizeof(float) * (size_t)splits * a.taps) : nullptr;
  a.out = part ? part : targets;
  if (v4) innerp_kernel<4><<<splits, INNERP_THREADS, 0, state().stream>>>(a, part ? 0 : 1);
  else innerp_kernel<1><<<splits, INNERP_THREADS, 0, state().stream>>>(a, part ? 0 : 1);
  count_launch();
  CNB_LAUNCH_CHECK("conv_innerp");
  if (part) reduce_partials(part, targets, a.taps, 1, splits, st, so);
  return splits;
}

}  // namespace cnb
