// conv_tc.cu — convolution fprop / dgrad / wgrad as implicit GEMMs on the Hopper tensor cores, fed by TMA straight from
// the caller's CHWN buffers (fp32, or their bf16 copies).  No im2col buffer, no layout conversion pass, no atomics.
//
// Layout insight (DESIGN.md §3): in the reference layout the IMAGE index n is the contiguous axis of every activation
// tensor (SURVEY.md Appendix A).  A box of 64 consecutive images (bf16; 32 in fp32) x K channels at one pixel is therefore
// a ready-made MN-major SWIZZLE_128B operand tile of K rows of 128 bytes, and zero-fill of out-of-range TMA coordinates
// implements the convolution padding for free.  Filters [K x Cout] (Cout contiguous) are MN-major B for fprop and K-major
// B for dgrad.
//
//   fprop : D[(n,module), o] = sum_{tap,c}  img[n, x(module,tap), y, c] * w[o, tap, c]     A MN-major, B MN-major
//   dgrad : D[(n,pixel), c]  = sum_{tap,o}  der[n, module(pixel,tap), o] * w[o, tap, c]    A MN-major, B K-major
//   wgrad : D[o, c] (per tap)= sum_{module,n} der[n, module, o] * img[n, x, y, c]          A K-major,  B K-major
//
// One persistent CTA per SM, 9 warps: warps 0..7 are two consumer warpgroups (GEMM rows 0-63 and 64-127 of the 128 x 128
// tile), warp 8 is the TMA producer filling a ring of shared-memory stages guarded by mbarriers.
//   bf16 operands: wgmma.mma_async m64n128k16 reads both operands from the swizzled tiles (either major);
//   tf32 operands: mma.sync m16n8k8 with fragments loaded from the same tiles — wgmma takes 32-bit operands from shared
//                  memory only K-major, and the image / filter operands of fprop and dgrad are MN-major.
// Accumulators live in registers; the consumers store a finished tile straight from them (every group of 8 lanes writes
// 8 consecutive images of one channel = one 32-byte sector) while the producer already fills the ring for the next tile.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cudaTypedefs.h>

#include <algorithm>
#include <vector>

#include "conv_kernels.h"
#include "sm90_ptx.cuh"

namespace cnb {

namespace {

constexpr int kConsumerWarps = 8;
constexpr int kThreads = 32 * kConsumerWarps + 32;
constexpr int BM = 128;             // GEMM rows per tile
constexpr int BN_MAX = 128;         // GEMM columns per tile (the wgmma N); narrower tiles leave the extra columns unstored
constexpr int BK = 32;              // fp32 (tf32) elements of K per pipeline stage (4 MMA steps of 8); x-mode constant
constexpr int kMaxStages = 8;
constexpr uint32_t kAStageBytes = BM * 128;       // 16 KiB: 128 rows x 128 B (K-major) or chunks x bk rows x 128 B (MN-major)
constexpr uint32_t kBStageBytes = BN_MAX * 128;   // 16 KiB: room for 128 columns in either major

enum Op { kFprop = 0, kDgrad = 1, kWgrad = 2 };

struct TcParams {
  // operand element type: tf32 = the caller's fp32 buffers as they are; bf16 = bf16 copies made by a conversion pass.
  // A 128-byte smem row holds `chunk` = 32 (tf32) or 64 (bf16) consecutive images / channels; one pipeline stage
  // covers bk = 32 / 64 elements of K (four MMA steps of 8 / 16) and an m-tile is cpt = 4 / 2 chunks of images.
  int bf16, chunk, chunk_shift, cpt, bk, nbc;   // nbc = ceil(N / chunk)
  int N, nb;                        // images, ceil(N/32)
  int W, H, modX, modY, modules;
  int Cin, Cout;                    // channel sub-range sizes
  int kx, ky, sx, sy, px, py, taps;
  int frames, frame0;               // fprop/wgrad: number of frames; dgrad: the single frame handled by this launch
  int BN, stages;
  int m_tiles, n_tiles, num_tiles;
  int kc_blocks;                    // ceil(K-side channels / bk)
  // "x mode" for tiny channel counts (Cin < 8, e.g. the RGB first layer): the kx taps of a filter row (padded to 8)
  // take the place of the channel block.  fprop: one K block = (channel c, 4 filter rows) = 4x8 K rows;
  // wgrad: the N tile is (x_ct channels) x (ky rows) x 8 taps, reduced over ALL modules at once.
  int x_mode, x_yblocks, x_ct;
  uint32_t b_tx_bytes;              // bytes the B-operand TMA(s) of one stage actually deliver
  // merged requests: when N % 128 == 0 (2-D) the chunks of an m-tile are one box over a (chunk, ..., N/chunk, ...) view
  // of the tensor; when Cout % chunk == 0 the BN/chunk filter chunks are one box likewise.
  int a_merged, b_merged;
  int total_chunks;                 // fprop: nbc*modules*frames ; dgrad: nbc*W*H   (< 2^31, checked on the host)
  int splits, units_per_split;      // wgrad: (frame, module-row) units per reduction split;
                                    // fprop/dgrad of 1x1 / FC shapes with few tiles: K blocks per split (split-K)
  long long part_stride;            // fprop/dgrad split-K: floats between the partial outputs of consecutive splits
  float* out;
  __nv_bfloat16* out16;             // optional bf16 twin of `out` (same indexing): convnet_b200_emit_bf16_next
  float st, so;
  const float* bias; int relu;      // fused fprop epilogue: + bias[o], then max(., 0)
  const float* mask;                // fused epilogue: zero where mask <= 0 (same layout as out)
  // fprop: dropout of the (bias + ReLU'd) result, element index = offset from `out` (Fuse::drop_*); drop_scale 0 = none
  float drop_prob, drop_scale;
  unsigned long long drop_seed;
  long long out_frame_step;         // fprop: floats between output frames
  // fprop: where output position (i, j) of the modX x modY grid lands in the target tensor: pixel
  // (i*o_sx + o_x0, j*o_sy + o_y0) of an o_W-wide plane of out_plane pixels.  Plain fprop: identity.  dgrad run as a
  // stride-1 correlation per stride phase (tc_conv_down_as_fprop) writes every o_sx-th pixel.
  int o_sx, o_sy, o_x0, o_y0, o_W;
  long long out_plane;
};

struct __align__(8) SmemCtl {
  uint64_t full[kMaxStages];
  uint64_t empty[kMaxStages];
};

// ------------------------------------------------------------------------------------------------
// tile / k-block enumeration, shared by the producer (which loads) and the consumers (which only count).
// ------------------------------------------------------------------------------------------------
struct Tile {
  int m_tile, n_tile;               // fprop/dgrad
  int tap, o_tile, c_tile, split;   // wgrad
};

template <int OP>
__device__ __forceinline__ Tile decode_tile(const TcParams& p, int t) {
  Tile r;
  r.split = t % p.splits; t /= p.splits;
  if (OP == kWgrad) {
    r.c_tile = t % p.n_tiles; t /= p.n_tiles;
    r.o_tile = t % p.m_tiles; t /= p.m_tiles;
    r.tap = t;
    r.m_tile = r.o_tile; r.n_tile = r.c_tile;
  } else {
    r.n_tile = t % p.n_tiles;
    r.m_tile = t / p.n_tiles;
    r.tap = r.o_tile = r.c_tile = 0;
  }
  return r;
}

// The (up to four) chunks of an fprop/dgrad m-tile: image offset, position (module / pixel) and frame.
struct Chunks {
  int n[4], pos[4], f[4];
  bool ok[4];
};
__device__ __forceinline__ Chunks decode_chunks(const TcParams& p, int m_tile, int per_frame) {
  Chunks c;
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const int q = m_tile * p.cpt + i;
    c.ok[i] = i < p.cpt && q < p.total_chunks;
    const int ib = q % p.nbc, r = q / p.nbc;
    c.n[i] = c.ok[i] ? ib * p.chunk : p.N;   // n >= N: the whole TMA box is out of range -> zero-filled
    c.pos[i] = r % per_frame;
    c.f[i] = c.ok[i] ? r / per_frame : 0;
  }
  return c;
}

// dgrad: module coordinate touched by tap t at input coordinate X, or -1
__device__ __forceinline__ int dgrad_mod(int X, int p, int t, int s, int mods) {
  const int a = X - p - t;
  if (a < 0) return -1;
  const int m = a / s;
  if (m * s != a || m >= mods) return -1;
  return m;
}

// dgrad: per-chunk bit masks of the taps that reach a module along x and along y (kx, ky <= 32)
struct DgradTaps {
  uint32_t xm[4], ym[4];
  __device__ __forceinline__ bool live(int c, int tx, int ty) const { return ((xm[c] >> tx) & (ym[c] >> ty) & 1u) != 0; }
  __device__ __forceinline__ bool any(int tx, int ty) const { return live(0, tx, ty) | live(1, tx, ty) | live(2, tx, ty) | live(3, tx, ty); }
};
__device__ __forceinline__ DgradTaps dgrad_taps(const TcParams& p, const Chunks& ch) {
  DgradTaps d;
#pragma unroll
  for (int c = 0; c < 4; c++) {
    d.xm[c] = d.ym[c] = 0;
    if (!ch.ok[c]) continue;
    const int X = ch.pos[c] % p.W, Y = ch.pos[c] / p.W;
    for (int t = 0; t < p.kx; t++) d.xm[c] |= (dgrad_mod(X, p.px, t, p.sx, p.modX) >= 0 ? 1u : 0u) << t;
    for (int t = 0; t < p.ky; t++) d.ym[c] |= (dgrad_mod(Y, p.py, t, p.sy, p.modY) >= 0 ? 1u : 0u) << t;
  }
  return d;
}
__device__ __forceinline__ int dgrad_live_taps(const TcParams& p, const DgradTaps& d) {
  int live = 0;
  for (int ty = 0; ty < p.ky; ty++)
    for (int tx = 0; tx < p.kx; tx++) live += d.any(tx, ty) ? 1 : 0;
  return live;
}

// wgrad: the reduction of one tile runs over rows r = f*modY + my in [r0, r1) and, inside a row, over the
// modules mx in [mx_lo, mx_hi] whose tap lands inside the image (the others contribute zeros and are skipped).
struct WgradSpan { int r0, r1, mx_lo, mx_hi, live_rows; };
__device__ __forceinline__ bool wgrad_row_live(const TcParams& p, int r, int ty) {
  const int Y = (r % p.modY) * p.sy + p.py + ty;
  return (unsigned)Y < (unsigned)p.H;
}
__device__ __forceinline__ WgradSpan wgrad_span(const TcParams& p, const Tile& t) {
  WgradSpan s;
  const int tx = t.tap % p.kx, ty = t.tap / p.kx;
  s.r0 = t.split * p.units_per_split;
  s.r1 = min(s.r0 + p.units_per_split, p.modY * p.frames);
  const int lo = -(p.px + tx);                             // mx*sx >= lo
  s.mx_lo = lo <= 0 ? 0 : (lo + p.sx - 1) / p.sx;
  const int hi = p.W - 1 - p.px - tx;                      // mx*sx <= hi
  s.mx_hi = hi < 0 ? -1 : min(hi / p.sx, p.modX - 1);
  s.live_rows = 0;
  if (s.mx_hi >= s.mx_lo)
    for (int r = s.r0; r < s.r1; r++) s.live_rows += wgrad_row_live(p, r, ty) ? 1 : 0;
  return s;
}

// k-blocks of a tile: exactly the stages the producer fills for it
template <int OP>
__device__ __forceinline__ int tile_kblocks(const TcParams& p, const Tile& tile) {
  if (OP == kFprop) {
    const int kcb = p.splits > 1 ? min(p.units_per_split, p.kc_blocks - tile.split * p.units_per_split) : p.kc_blocks;
    return p.x_mode ? p.Cin * p.x_yblocks : p.taps * kcb;
  } else if (OP == kDgrad) {
    const DgradTaps own = dgrad_taps(p, decode_chunks(p, tile.m_tile, p.W * p.H));
    const int kcb = p.splits > 1 ? min(p.units_per_split, p.kc_blocks - tile.split * p.units_per_split) : p.kc_blocks;
    return max(dgrad_live_taps(p, own), 1) * kcb;
  } else if (p.x_mode) {
    const int r0 = tile.split * p.units_per_split, r1 = min(r0 + p.units_per_split, p.modY * p.frames);
    return (r1 - r0) * p.modX * p.nb;
  } else {
    const WgradSpan sp = wgrad_span(p, tile);
    return max(sp.live_rows * (sp.mx_hi - sp.mx_lo + 1), 1) * p.nbc;
  }
}

// byte offset of element (row, k) of a 32-bit SWIZZLE_128B tile.  K-major: one 128-byte row per GEMM row, 32 K elements
// in it; MN-major: [32-row chunk][K rows][128 B].  The swizzle XORs the 16-byte unit with the 128-byte line index mod 8.
__device__ __forceinline__ uint32_t off_kmajor(int row, int k) {
  return (uint32_t)(row * 128 + ((((k >> 2) ^ row) & 7) << 4) + ((k & 3) << 2));
}
__device__ __forceinline__ uint32_t off_mnmajor(int row, int k) {
  return (uint32_t)((row >> 5) * (BK * 128) + k * 128 + (((((row & 31) >> 2) ^ k) & 7) << 4) + ((row & 3) << 2));
}

// ------------------------------------------------------------------------------------------------
template <int OP, bool BF16>
__global__ void __launch_bounds__(kThreads, 1)
tc_conv_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB, const __grid_constant__ TcParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smemA = smem;
  uint8_t* smemB = smem + (size_t)p.stages * kAStageBytes;
  SmemCtl* ctl = reinterpret_cast<SmemCtl*>(smemB + (size_t)p.stages * kBStageBytes);

  // warp index through a shuffle: provably warp-uniform, which keeps the role branches and their loops on the uniform path
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.stages; s++) { ptx::mbar_init(&ctl->full[s], 1); ptx::mbar_init(&ctl->empty[s], kConsumerWarps); }
    ptx::fence_barrier_init();
    ptx::tma_prefetch_desc(&mapA);
    ptx::tma_prefetch_desc(&mapB);
  }
  __syncthreads();
  ptx::pdl_launch_dependents();       // the kernel queued behind this one may start its prologue (it waits for this grid's end)
  ptx::pdl_wait();                    // ... as this one's just overlapped its predecessor's tail; from here on: global memory

  if (warp == kConsumerWarps) {
    // =============================== TMA producer (one lane) ===============================
    if (lane != 0) return;
    int stage = 0; uint32_t phase = 0;
    const uint32_t tx_bytes = kAStageBytes + p.b_tx_bytes;
    for (int t = blockIdx.x; t < p.num_tiles; t += gridDim.x) {
      const Tile tile = decode_tile<OP>(p, t);
      auto begin_stage = [&]() -> uint8_t* {
        ptx::mbar_wait(&ctl->empty[stage], phase ^ 1);
        ptx::mbar_arrive_expect_tx(&ctl->full[stage], tx_bytes);
        return smemA + (size_t)stage * kAStageBytes;
      };
      auto lda5 = [&](const void* m, void* dst, int c0, int c1, int c2, int c3, int c4) {
        ptx::tma_load_5d(m, &ctl->full[stage], dst, c0, c1, c2, c3, c4);
      };
      auto lda4 = [&](const void* m, void* dst, int c0, int c1, int c2, int c3) {
        ptx::tma_load_4d(m, &ctl->full[stage], dst, c0, c1, c2, c3);
      };
      auto lda3 = [&](const void* m, void* dst, int c0, int c1, int c2) {
        ptx::tma_load_3d(m, &ctl->full[stage], dst, c0, c1, c2);
      };
      auto end_stage = [&]() { if (++stage == p.stages) { stage = 0; phase ^= 1; } };

      if (OP == kFprop) {
        const Chunks ch = decode_chunks(p, tile.m_tile, p.modules);
        int cX[4], cY[4];
#pragma unroll
        for (int c = 0; c < 4; c++) {
          cX[c] = (ch.pos[c] % p.modX) * p.sx + p.px;
          cY[c] = (ch.pos[c] / p.modX) * p.sy + p.py;
        }
        if (p.x_mode) {
          for (int c = 0; c < p.Cin; c++)
            for (int yb = 0; yb < p.x_yblocks; yb++) {
              uint8_t* a = begin_stage();
              uint8_t* b = smemB + (size_t)stage * kBStageBytes;
              if (p.a_merged) {                // dims (n_lo, x, y, n_hi, c): one 16 KiB request
                lda5(&mapA, a, 0, cX[0], cY[0] + 4 * yb, ch.n[0] >> 5, c);
              } else {
#pragma unroll
                for (int q = 0; q < 4; q++)    // 8 consecutive x pixels x 4 filter rows of channel c = 32 K rows
                  lda5(&mapA, a + q * (BK * 128), ch.n[q], c, cX[q], cY[q] + 4 * yb, ch.f[q]);
              }
              if (p.b_merged) {                // dims (o_lo, tx, ty, o_hi, c)
                lda5(&mapB, b, 0, 0, 4 * yb, tile.n_tile * (p.BN >> 5), c);
              } else {
                for (int j = 0; j < p.BN / 32; j++)   // taps >= kx and rows >= ky are out of range -> zero weights
                  lda4(&mapB, b + j * (BK * 128), tile.n_tile * p.BN + j * 32, 0, 4 * yb, c);
              }
              end_stage();
            }
        } else {
          // split-K (host: only when taps == 1): this tile reduces K blocks [cb0, cb1)
          const int cb0 = p.splits > 1 ? tile.split * p.units_per_split : 0;
          const int cb1 = p.splits > 1 ? min(cb0 + p.units_per_split, p.kc_blocks) : p.kc_blocks;
          for (int ty = 0; ty < p.ky; ty++)
            for (int tx = 0; tx < p.kx; tx++) {
              const int tap = tx + p.kx * ty;
              for (int cb = cb0; cb < cb1; cb++) {
                uint8_t* a = begin_stage();
                uint8_t* b = smemB + (size_t)stage * kBStageBytes;
                if (p.a_merged) {                // dims (n_lo, c, n_hi, x, y): one 16 KiB request
                  lda5(&mapA, a, 0, cb * p.bk, ch.n[0] >> p.chunk_shift, cX[0] + tx, cY[0] + ty);
                } else {
#pragma unroll
                  for (int c = 0; c < 4; c++)
                    if (c < p.cpt) lda5(&mapA, a + c * (p.bk * 128), ch.n[c], cb * p.bk, cX[c] + tx, cY[c] + ty, ch.f[c]);
                }
                const int o0 = tile.n_tile * p.BN;
                if (p.b_merged) {                // dims (o_lo, c, o_hi, tap)
                  lda4(&mapB, b, 0, cb * p.bk, o0 >> p.chunk_shift, tap);
                } else {
                  for (int j = 0; j < ((p.BN + p.chunk - 1) >> p.chunk_shift); j++)
                    lda3(&mapB, b + j * (p.bk * 128), o0 + j * p.chunk, tap, cb * p.bk);
                }
                end_stage();
              }
            }
        }
      } else if (OP == kDgrad) {
        const Chunks ch = decode_chunks(p, tile.m_tile, p.W * p.H);
        const DgradTaps taps = dgrad_taps(p, ch);
        const bool none = dgrad_live_taps(p, taps) == 0;    // then one all-zero k-block group keeps the count uniform
        int cX[4], cY[4];
#pragma unroll
        for (int c = 0; c < 4; c++) { cX[c] = ch.pos[c] % p.W; cY[c] = ch.pos[c] / p.W; }
        const int ob0 = p.splits > 1 ? tile.split * p.units_per_split : 0;
        const int ob1 = p.splits > 1 ? min(ob0 + p.units_per_split, p.kc_blocks) : p.kc_blocks;
        for (int ty = 0; ty < p.ky; ty++)
          for (int tx = 0; tx < p.kx; tx++) {
            if (!(taps.any(tx, ty) || (none && tx == 0 && ty == 0))) continue;
            int mx[4], my[4];
#pragma unroll
            for (int c = 0; c < 4; c++) {
              const bool lv = ch.ok[c] && taps.live(c, tx, ty);
              mx[c] = lv ? (cX[c] - p.px - tx) / p.sx : -1;      // -1: out of range -> zeros
              my[c] = lv ? (cY[c] - p.py - ty) / p.sy : -1;
            }
            const int tap = tx + p.kx * ty;
            for (int ob = ob0; ob < ob1; ob++) {
              uint8_t* a = begin_stage();
              uint8_t* b = smemB + (size_t)stage * kBStageBytes;
              if (p.a_merged) {                // all chunks sit on the same pixel: dims (n_lo, o, n_hi, mx, my)
                lda5(&mapA, a, 0, ob * p.bk, ch.n[0] >> p.chunk_shift, mx[0], my[0]);
              } else {
#pragma unroll
                for (int c = 0; c < 4; c++)
                  if (c < p.cpt) lda5(&mapA, a + c * (p.bk * 128), ch.n[c], ob * p.bk, mx[c], my[c], p.frame0);
              }
              lda3(&mapB, b, ob * p.bk, tap, tile.n_tile * p.BN);
              end_stage();
            }
          }
      } else if (p.x_mode) {
        // reduction over every module of this split's rows; B holds x_ct channels x ky rows x 8 taps
        const int r0 = tile.split * p.units_per_split, r1 = min(r0 + p.units_per_split, p.modY * p.frames);
        const uint32_t c_bytes = (uint32_t)p.ky * 8 * 128;
        for (int r = r0; r < r1; r++) {
          const int f = r / p.modY, my = r % p.modY;
          for (int mx = 0; mx < p.modX; mx++)
            for (int ib = 0; ib < p.nb; ib++) {
              uint8_t* a = begin_stage();
              uint8_t* b = smemB + (size_t)stage * kBStageBytes;
              lda5(&mapA, a, ib * 32, mx, my, tile.o_tile * BM, f);
              for (int c = 0; c < p.x_ct; c++)
                lda5(&mapB, b + c * c_bytes, ib * 32, mx * p.sx + p.px, my * p.sy + p.py, tile.c_tile * p.x_ct + c, f);
              end_stage();
            }
        }
      } else {
        const WgradSpan sp = wgrad_span(p, tile);
        const int tx = tile.tap % p.kx, ty = tile.tap / p.kx;
        if (sp.live_rows == 0 || sp.mx_hi < sp.mx_lo) {   // nothing to sum: one zero k-block group
          for (int ib = 0; ib < p.nbc; ib++) {
            uint8_t* a = begin_stage();
            uint8_t* b = smemB + (size_t)stage * kBStageBytes;
            lda5(&mapA, a, ib * p.chunk, 0, 0, tile.o_tile * BM, 0);
            lda5(&mapB, b, ib * p.chunk, -1, -1, tile.c_tile * p.BN, 0);
            end_stage();
          }
        } else {
          for (int r = sp.r0; r < sp.r1; r++) {
            if (!wgrad_row_live(p, r, ty)) continue;
            const int f = r / p.modY, my = r % p.modY;
            const int Y = my * p.sy + p.py + ty;
            for (int mx = sp.mx_lo; mx <= sp.mx_hi; mx++) {
              const int X = mx * p.sx + p.px + tx;
              for (int ib = 0; ib < p.nbc; ib++) {
                uint8_t* a = begin_stage();
                uint8_t* b = smemB + (size_t)stage * kBStageBytes;
                lda5(&mapA, a, ib * p.chunk, mx, my, tile.o_tile * BM, f);
                lda5(&mapB, b, ib * p.chunk, X, Y, tile.c_tile * p.BN, f);
                end_stage();
              }
            }
          }
        }
      }
    }
    return;
  }

  // =============================== consumers: MMA + epilogue ===================================
  const int g = lane >> 2, tq = lane & 3;
  const int row0 = warp * 16 + g;                  // this thread's GEMM rows in the tile: row0 and row0 + 8
  int stage = 0; uint32_t phase = 0;
  for (int t = blockIdx.x; t < p.num_tiles; t += gridDim.x) {
    const Tile tile = decode_tile<OP>(p, t);
    const int nkb = tile_kblocks<OP>(p, tile);
    float acc[BN_MAX / 8][4];
#pragma unroll
    for (int j = 0; j < BN_MAX / 8; j++)
#pragma unroll
      for (int e = 0; e < 4; e++) acc[j][e] = 0.f;

    if constexpr (BF16) {
      // warpgroup w multiplies GEMM rows 64w..64w+63: the second 64-image chunk (MN-major A) or rows 64.. (K-major A),
      // 8 KiB into the stage either way
      constexpr bool a_mn = (OP != kWgrad), b_mn = (OP == kFprop);
      constexpr uint32_t a_step = a_mn ? 2048u : 32u, b_step = b_mn ? 2048u : 32u;
      const uint64_t da0 = ptx::gmma_desc(ptx::smem_u32(smemA) + (uint32_t)(warp >> 2) * 8192u, a_mn ? 8192u : 16u, 1024u);
      const uint64_t db0 = ptx::gmma_desc(ptx::smem_u32(smemB), b_mn ? 8192u : 16u, 1024u);
      int prev = -1;
      ptx::wgmma_fence_operands(acc);
      for (int kb = 0; kb < nkb; kb++) {
        ptx::mbar_wait(&ctl->full[stage], phase);
        ptx::wgmma_fence();
        const uint64_t da = da0 + ((uint32_t)stage * kAStageBytes >> 4), db = db0 + ((uint32_t)stage * kBStageBytes >> 4);
#pragma unroll
        for (int ks = 0; ks < 4; ks++)
          ptx::wgmma_m64n128k16_bf16<a_mn ? 1 : 0, b_mn ? 1 : 0>(acc, da + (ks * a_step >> 4), db + (ks * b_step >> 4));
        ptx::wgmma_commit();
        ptx::wgmma_wait<1>();                        // the previous stage's MMAs have retired: its slot can be refilled
        if (prev >= 0 && lane == 0) ptx::mbar_arrive(&ctl->empty[prev]);
        prev = stage;
        if (++stage == p.stages) { stage = 0; phase ^= 1; }
      }
      ptx::wgmma_wait<0>();
      ptx::wgmma_fence_operands(acc);
      if (prev >= 0 && lane == 0) ptx::mbar_arrive(&ctl->empty[prev]);
    } else {
      const uint32_t sA = ptx::smem_u32(smemA), sB = ptx::smem_u32(smemB);
      constexpr bool a_mn = (OP != kWgrad), b_mn = (OP == kFprop);
      for (int kb = 0; kb < nkb; kb++) {
        ptx::mbar_wait(&ctl->full[stage], phase);
        const uint32_t A = sA + (uint32_t)stage * kAStageBytes, B = sB + (uint32_t)stage * kBStageBytes;
#pragma unroll
        for (int ks = 0; ks < 4; ks++) {
          const int k0 = ks * 8 + tq, k1 = k0 + 4;
          const uint32_t a0 = ptx::lds32(A + (a_mn ? off_mnmajor(row0, k0) : off_kmajor(row0, k0)));
          const uint32_t a1 = ptx::lds32(A + (a_mn ? off_mnmajor(row0 + 8, k0) : off_kmajor(row0 + 8, k0)));
          const uint32_t a2 = ptx::lds32(A + (a_mn ? off_mnmajor(row0, k1) : off_kmajor(row0, k1)));
          const uint32_t a3 = ptx::lds32(A + (a_mn ? off_mnmajor(row0 + 8, k1) : off_kmajor(row0 + 8, k1)));
#pragma unroll
          for (int j = 0; j < BN_MAX / 8; j++) {
            if (j * 8 >= p.BN) break;
            const int n = j * 8 + g;
            const uint32_t b0 = ptx::lds32(B + (b_mn ? off_mnmajor(n, k0) : off_kmajor(n, k0)));
            const uint32_t b1 = ptx::lds32(B + (b_mn ? off_mnmajor(n, k1) : off_kmajor(n, k1)));
            ptx::mma_tf32_16x8x8(acc[j], a0, a1, a2, a3, b0, b1);
          }
        }
        __syncwarp();
        if (lane == 0) ptx::mbar_arrive(&ctl->empty[stage]);
        if (++stage == p.stages) { stage = 0; phase ^= 1; }
      }
    }

    // =============================== epilogue ===================================
    float* rowp[2] = {nullptr, nullptr};
    long long col_stride = 0;
    int ncols_valid = 0;
#pragma unroll
    for (int h = 0; h < 2; h++) {
      const int r = row0 + 8 * h;
      if (OP == kFprop || OP == kDgrad) {
        const int q = tile.m_tile * p.cpt + (r >> p.chunk_shift);
        const int per_frame = (OP == kFprop) ? p.modules : p.W * p.H;
        if (q < p.total_chunks) {
          const int ib = q % p.nbc, rr = q / p.nbc, pos = rr % per_frame, f = rr / per_frame;
          const int n = ib * p.chunk + (r & (p.chunk - 1));
          if (n < p.N) {
            if (OP == kFprop) {
              const int i = pos % p.modX, j = pos / p.modX;
              const long long pix = (long long)(i * p.o_sx + p.o_x0) + (long long)p.o_W * (j * p.o_sy + p.o_y0);
              col_stride = (long long)p.N * p.out_plane;
              rowp[h] = p.out + f * p.out_frame_step + n + (long long)p.N * pix;
            } else {
              col_stride = (long long)p.N * per_frame;
              rowp[h] = p.out + n + (long long)p.N * pos;
            }
            rowp[h] += col_stride * ((long long)tile.n_tile * p.BN) + tile.split * p.part_stride;
          }
        }
      } else {
        const int o = tile.o_tile * BM + r;
        if (o < p.Cout) {
          rowp[h] = p.out + (long long)tile.split * p.Cout * p.taps * p.Cin + o;
          if (!p.x_mode) {
            col_stride = (long long)p.Cout * p.taps;
            rowp[h] += (long long)p.Cout * tile.tap + col_stride * ((long long)tile.c_tile * p.BN);
          }
        }
      }
    }
    if (OP == kFprop || OP == kDgrad) ncols_valid = min(p.BN, (OP == kFprop ? p.Cout : p.Cin) - tile.n_tile * p.BN);
    else if (p.x_mode) ncols_valid = min(p.BN, p.x_ct * p.ky * 8);
    else ncols_valid = min(p.BN, p.Cin - tile.c_tile * p.BN);
    const bool direct_scale = (p.splits == 1);
    const float so_eff = direct_scale ? p.so : 1.f;
    const bool rmw = direct_scale && p.st != 0.f;
    const float* bias = (OP == kFprop && p.bias) ? p.bias + tile.n_tile * p.BN : nullptr;
#pragma unroll
    for (int h = 0; h < 2; h++) {
      float* const rp = rowp[h];
      if (rp == nullptr) continue;
#pragma unroll
      for (int j = 0; j < BN_MAX / 8; j++)
#pragma unroll
        for (int e = 0; e < 2; e++) {
          const int col = j * 8 + 2 * tq + e;
          if (col >= ncols_valid) continue;
          const float v = acc[j][2 * h + e];
          float* dst;
          if (OP == kWgrad && p.x_mode) {
            // column = tap tx + 8*(row ty + ky*channel): scattered to dW[o, tx + kx*(ty + ky*c)]
            const int tx = col & 7, rr = col >> 3, ty = rr % p.ky, c = tile.c_tile * p.x_ct + rr / p.ky;
            if (tx >= p.kx || c >= p.Cin) continue;
            dst = rp + (long long)p.Cout * (tx + p.kx * (ty + p.ky * c));
          } else {
            dst = rp + col_stride * col;
          }
          float r = so_eff * v;
          if (rmw) r += p.st * (*dst);
          if (OP == kFprop) {
            if (bias) r += __ldg(bias + col);
            if (p.relu) r = fmaxf(r, 0.f);
            if (p.drop_scale != 0.f) r *= dropout_keep(p.drop_seed + (unsigned long long)(dst - p.out), p.drop_prob, p.drop_scale);
          }
          if (p.mask && !(__ldg(p.mask + (dst - p.out)) > 0.f)) r = 0.f;
          *dst = r;
          if (p.out16) p.out16[dst - p.out] = __float2bfloat16_rn(r);
        }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
PFN_cuTensorMapEncodeTiled_v12000 encode_fn() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
  if (!fn) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    CNB_CUDA_CHECK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres));
    CNB_REQUIRE(qres == cudaDriverEntryPointSuccess && ptr != nullptr, "cuTensorMapEncodeTiled");
    fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(ptr);
  }
  return fn;
}

// operand element type of one launch (see TcParams)
struct Elem { int bf16, esz, chunk, shift, bk; };
inline Elem elem_for(bool bf16) { return bf16 ? Elem{1, 2, 64, 6, 64} : Elem{0, 4, 32, 5, 32}; }

// tensor map over fp32 or bf16 data; dims[0] is the contiguous axis; strides in ELEMENTS for dims 1..rank-1.
// Every box lands in shared memory with the 128-byte swizzle the kernel's operand reads assume.
bool make_map(CUtensorMap* map, const void* base, const Elem& e, int rank, const long long* dims, const long long* strides,
              const int* box) {
  cuuint64_t gdim[5], gstr[4];
  cuuint32_t bdim[5], estr[5];
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0) return false;
  for (int i = 0; i < rank; i++) {
    if (dims[i] <= 0 || dims[i] > 0xFFFFFFFFLL) return false;
    gdim[i] = (cuuint64_t)dims[i];
    bdim[i] = (cuuint32_t)box[i];
    estr[i] = 1;
    if (box[i] > 256) return false;
    if (i > 0) {
      const long long bytes = strides[i - 1] * e.esz;
      if (bytes % 16 != 0 || bytes <= 0 || bytes >= (1LL << 40)) return false;
      gstr[i - 1] = (cuuint64_t)bytes;
    }
  }
  CUresult r = encode_fn()(map, e.bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, (cuuint32_t)rank,
                           const_cast<void*>(base), gdim, gstr, bdim, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                           CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    fprintf(stderr, "convnet_b200: cuTensorMapEncodeTiled failed (%d)\n", (int)r);
    return false;
  }
  return true;
}

int pick_bn(int cols, int granule) {              // N-tile: as wide as possible, <= BN_MAX, balanced across tiles
  const int tiles = ceil_div(cols, BN_MAX);
  const int bn = ceil_div(ceil_div(cols, tiles), granule) * granule;
  return std::min(BN_MAX, std::max(granule, bn));
}

size_t smem_bytes_for(int stages) {
  return 1024 + (size_t)stages * (kAStageBytes + kBStageBytes) + sizeof(SmemCtl) + 16;
}

int pick_stages() {
  int s = kMaxStages;
  while (s > 2 && smem_bytes_for(s) > 225 * 1024) s--;
  return s;
}

template <int OP, bool BF16>
void launch_one(const CUtensorMap& a, const CUtensorMap& b, const TcParams& p, size_t smem) {
  // the attribute belongs to the (function, device) pair: set it once per device this process launches on
  static unsigned long long attr_devices = 0;
  const int dev = current_device();
  if (dev >= 64 || !((attr_devices >> dev) & 1ULL)) {
    CNB_CUDA_CHECK(cudaFuncSetAttribute(tc_conv_kernel<OP, BF16>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    if (dev < 64) attr_devices |= 1ULL << dev;
  }
  const int grid = std::min(p.num_tiles, num_sms());
  launch_pdl(tc_conv_kernel<OP, BF16>, dim3((unsigned)grid), dim3(kThreads), smem, state().stream, a, b, p);
}

template <int OP>
void launch(const CUtensorMap& a, const CUtensorMap& b, TcParams& p) {
  p.stages = pick_stages();
  const size_t smem = smem_bytes_for(p.stages);
  if (p.bf16) launch_one<OP, true>(a, b, p, smem);
  else launch_one<OP, false>(a, b, p, smem);
  count_launch();
  CNB_LAUNCH_CHECK("tc_conv");
}

bool tc_enabled() {
  static int en = -1;
  if (en < 0) { const char* e = getenv("CONVNET_B200_DISABLE_TC"); en = (e && e[0] == '1') ? 0 : 1; }
  return en == 1 && state().precision >= kPrecTF32;
}

void fill_common(TcParams& p, const ConvGeom& g, const Elem& e) {
  p.bf16 = e.bf16; p.chunk = e.chunk; p.chunk_shift = e.shift; p.cpt = BM / e.chunk; p.bk = e.bk;
  p.N = g.N; p.nb = ceil_div(g.N, 32); p.nbc = ceil_div(g.N, e.chunk);
  p.W = g.W; p.H = g.H; p.modX = g.modX; p.modY = g.modY; p.modules = g.modules;
  p.Cin = g.Cin; p.Cout = g.Cout;
  p.kx = g.kx; p.ky = g.ky; p.sx = g.sx; p.sy = g.sy; p.px = g.px; p.py = g.py; p.taps = g.kx * g.ky;
  p.frames = g.frames; p.frame0 = 0;
  p.splits = 1; p.units_per_split = 0; p.part_stride = 0;
  p.x_mode = 0; p.x_yblocks = 0; p.x_ct = 0; p.b_tx_bytes = 0;
  p.a_merged = 0; p.b_merged = 0;
  p.bias = nullptr; p.relu = 0; p.mask = nullptr; p.out16 = nullptr;
  p.drop_prob = 0.f; p.drop_scale = 0.f; p.drop_seed = 0;
  p.o_sx = p.o_sy = 1; p.o_x0 = p.o_y0 = 0; p.o_W = g.modX; p.out_plane = g.modules;
  p.out_frame_step = g.out_frame_step;
  p.total_chunks = 0;
  p.st = 0.f; p.so = 1.f; p.out = nullptr;
}

// image-like tensor (N, W, H, C[, frames]) as a 5-D map ordered (n, c, x, y, f) or (n, x, y, c, f)
bool image_map(CUtensorMap* m, const void* base, const Elem& e, const ConvGeom& g, int Wd, int Hd, int C,
               long long frame_step, bool channel_second, int box_c) {
  const long long N = g.N;
  if (channel_second) {
    const long long dims[5] = {N, C, Wd, Hd, g.frames};
    const long long str[4] = {N * Wd * Hd, N, N * Wd, frame_step};
    const int box[5] = {e.chunk, box_c, 1, 1, 1};
    return make_map(m, base, e, 5, dims, str, box);
  }
  const long long dims[5] = {N, Wd, Hd, C, g.frames};
  const long long str[4] = {N, N * Wd, N * Wd * Hd, frame_step};
  const int box[5] = {e.chunk, 1, 1, box_c, 1};
  return make_map(m, base, e, 5, dims, str, box);
}

// (n_lo = chunk, channel / x / y ..., n_hi = N/chunk) view for one-request A tiles; `x_mode`: box {32, 8x, 4y, 4 n_hi, 1c}
bool merged_image_map(CUtensorMap* m, const void* base, const Elem& e, const ConvGeom& g, int Wd, int Hd, int C, bool x_mode) {
  const long long N = g.N;
  if (x_mode) {
    const long long dims[5] = {32, Wd, Hd, N / 32, C};
    const long long str[4] = {N, N * Wd, 32, N * Wd * Hd};
    const int box[5] = {32, 8, 4, 4, 1};
    return make_map(m, base, e, 5, dims, str, box);
  }
  const long long dims[5] = {e.chunk, C, N / e.chunk, Wd, Hd};
  const long long str[4] = {N * Wd * Hd, e.chunk, N, N * Wd};
  const int box[5] = {e.chunk, e.bk, BM / e.chunk, 1, 1};
  return make_map(m, base, e, 5, dims, str, box);
}

// MN-major filter operand [K = (tap, c)] x [columns], columns contiguous: dims (col, tap, c), or (col_lo, c, col_hi, tap)
// when `merged` (one request per stage).  `cols` = the column count of the whole tensor, `bn` = columns per tile.
bool filter_map(CUtensorMap* m, const void* base, const Elem& e, long long cols, long long taps, long long K_c, int bn,
                bool merged) {
  if (merged) {
    const long long dims[4] = {e.chunk, K_c, cols / e.chunk, taps};
    const long long str[3] = {cols * taps, e.chunk, cols};
    const int box[4] = {e.chunk, e.bk, bn / e.chunk, 1};
    return make_map(m, base, e, 4, dims, str, box);
  }
  const long long dims[3] = {cols, taps, K_c};
  const long long str[2] = {cols, cols * taps};
  const int box[3] = {e.chunk, 1, e.bk};
  return make_map(m, base, e, 3, dims, str, box);
}

inline size_t align_up(size_t v) { return (v + 1023) & ~size_t(1023); }

// ---- split-K for 1x1 / FC shapes: too few output tiles to fill the GPU, long K ------------------------
// out = st*out + so * sum_s part[s]  (+ bias[channel], ReLU | zero where mask <= 0): the fused epilogue moves here
__global__ void __launch_bounds__(256) reduce_split_kernel(const float4* __restrict__ part, float4* out, long long elems4,
                                                           long long stride4, int splits, float st, float so,
                                                           const float* __restrict__ bias, long long per_channel4, int relu,
                                                           const float4* __restrict__ mask) {
  pdl_wait();
  pdl_trigger();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < elems4; i += (long long)gridDim.x * blockDim.x) {
    float4 s = part[i];
    for (int k = 1; k < splits; k++) {
      const float4 v = part[i + k * stride4];
      s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
    }
    s.x *= so; s.y *= so; s.z *= so; s.w *= so;
    if (st != 0.f) { const float4 o = out[i]; s.x += st * o.x; s.y += st * o.y; s.z += st * o.z; s.w += st * o.w; }
    if (bias) { const float b = __ldg(bias + i / per_channel4); s.x += b; s.y += b; s.z += b; s.w += b; }
    if (relu) { s.x = fmaxf(s.x, 0.f); s.y = fmaxf(s.y, 0.f); s.z = fmaxf(s.z, 0.f); s.w = fmaxf(s.w, 0.f); }
    if (mask) {
      const float4 m = mask[i];
      if (!(m.x > 0.f)) s.x = 0.f;
      if (!(m.y > 0.f)) s.y = 0.f;
      if (!(m.z > 0.f)) s.z = 0.f;
      if (!(m.w > 0.f)) s.w = 0.f;
    }
    out[i] = s;
  }
}
void reduce_split(const float* part, float* out, long long elems, int splits, float st, float so, const float* bias,
                  long long per_channel, int relu, const float* mask) {
  const long long e4 = elems / 4;
  const int grid = (int)std::min<long long>(std::max<long long>(ceil_div<long long>(e4, 256), 1), 8LL * num_sms());
  launch_pdl(reduce_split_kernel, dim3((unsigned)grid), dim3(256), 0, state().stream, (const float4*)part, (float4*)out, e4, e4, splits,
             st, so, bias, per_channel / 4, relu, (const float4*)mask);
  count_launch();
  CNB_LAUNCH_CHECK("reduce_split");
}
// how many K splits a fprop/dgrad launch should use (1 = none): only 1x1 / FC shapes that leave most SMs idle
int pick_ksplit(const TcParams& p, const ConvGeom& g, long long out_elems) {
  if (p.x_mode || p.taps != 1 || g.frames != 1 || out_elems % 4 != 0) return 1;
  if (p.num_tiles * 2 > num_sms() || p.kc_blocks < 8) return 1;
  const int want = std::min(num_sms() / p.num_tiles, p.kc_blocks / 4);
  return std::max(want, 1);
}
inline bool aligned16(const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; }

}  // namespace

// ---- fprop ---------------------------------------------------------------------------------------
// `bf` selects bf16 operands (CONVNET_B200_PRECISION=bf16): images and filters are first rounded to bf16 copies in
// library scratch (unless the caller keeps staged copies), then the bf16 flavour of the kernel runs wgmma on them.
static bool tc_conv_up_impl(const ConvGeom& g, const float* images, const float* filters, float* targets, float st, float so,
                            const Fuse& fuse, bool bf) {
  const Elem e = elem_for(bf);
  if (g.N % 4 != 0 || g.Cout % 4 != 0) return false;                        // TMA stride alignment
  const bool x_mode = g.Cin < 8;                                            // tiny channel counts: taps take the K block
  if (x_mode && (g.kx > 8 || g.ky > 8)) return false;
  if (bf && (x_mode || g.N % 8 != 0 || g.Cout % 8 != 0 || !aligned16(images) || !aligned16(filters))) return false;
  // few GEMM rows (FC layers at training batch sizes): the call streams the weights once and is HBM-bound on them; a bf16
  // conversion pass inside the call would read them a second time, so such shapes take bf16 only when the caller keeps a
  // staged bf16 copy of the weights (the training host does: cnb_sgd_momentum refreshes it in the same pass that updates
  // them) — then the call streams HALF the bytes
  if (bf && (long long)g.N * g.modules * g.frames < 1024 && !bf16_staged(filters, (long long)g.Cout * g.K)) return false;
  TcParams p; fill_common(p, g, e);
  p.BN = pick_bn(g.Cout, e.chunk);
  p.kc_blocks = ceil_div(g.Cin, e.bk);
  p.x_mode = x_mode ? 1 : 0;
  p.x_yblocks = ceil_div(g.ky, 4);
  const long long chunks = (long long)p.nb * g.modules * g.frames;
  if (chunks * 4 >= (1LL << 31)) return false;
  p.total_chunks = p.nbc * g.modules * g.frames;
  p.m_tiles = ceil_div(p.total_chunks, p.cpt);
  p.n_tiles = ceil_div(g.Cout, p.BN);
  p.num_tiles = p.m_tiles * p.n_tiles;
  // MN-major B is staged in whole chunks (BN is a multiple of the chunk)
  p.b_tx_bytes = (uint32_t)p.BN * 128;
  float* const out = targets + (long long)g.cout0 * g.modules * g.N;
  const float* const bias = fuse.bias ? fuse.bias + g.cout0 : nullptr;
  const long long out_elems = (long long)g.Cout * g.modules * g.N;
  const int ks = pick_ksplit(p, g, out_elems);
  if (ks > 1) {
    p.units_per_split = ceil_div(p.kc_blocks, ks);
    p.splits = ceil_div(p.kc_blocks, p.units_per_split);
    p.part_stride = out_elems;
    p.num_tiles *= p.splits;
  }
  const size_t part_bytes = p.splits > 1 ? align_up(sizeof(float) * out_elems * p.splits) : 0;
  p.out = out;
  p.st = st; p.so = so;
  p.bias = bias; p.relu = fuse.relu;
  CUtensorMap ma, mb;
  const long long img_off = (long long)g.cin0 * g.H * g.W * g.N;
  const void* img = images + img_off;
  const void* flt = filters;
  const long long taps = (long long)g.kx * g.ky;
  uint8_t* ws = nullptr;
  if (bf) {
    const __nv_bfloat16* si = bf16_staged(images, g.img_total);
    const __nv_bfloat16* sf = bf16_staged(filters, (long long)g.Cout * g.K);
    const size_t ib = si ? 0 : align_up((size_t)g.img_total * 2), fb = sf ? 0 : align_up((size_t)g.Cout * g.K * 2);
    if (part_bytes + ib + fb) ws = (uint8_t*)workspace(part_bytes + ib + fb);
    if (!si) { to_bf16(images, (__nv_bfloat16*)(ws + part_bytes), g.img_total); si = (const __nv_bfloat16*)(ws + part_bytes); }
    if (!sf) { to_bf16(filters, (__nv_bfloat16*)(ws + part_bytes + ib), (long long)g.Cout * g.K); sf = (const __nv_bfloat16*)(ws + part_bytes + ib); }
    img = si + img_off;
    flt = sf;
  } else if (part_bytes) {
    ws = (uint8_t*)workspace(part_bytes);
  }
  if (p.splits > 1) { p.out = (float*)ws; p.bias = nullptr; p.relu = 0; }   // partial sums; the epilogue moves to reduce_split
  // bf16 twin of the output from the same registers: only when this launch writes the final value of EVERY element
  const bool emit = fuse.out16 != nullptr && p.splits == 1 && g.cout0 == 0 && g.Cout == g.CoutT;
  if (emit) p.out16 = fuse.out16;
  // dropout in the epilogue: the element index is the offset from the start of the WHOLE target tensor
  const bool drop = fuse.drop_scale != 0.f && p.splits == 1 && g.frames == 1 && g.cout0 == 0 && g.Cout == g.CoutT;
  if (drop) { p.drop_prob = fuse.drop_prob; p.drop_scale = fuse.drop_scale; p.drop_seed = fuse.drop_seed; }
  p.a_merged = (g.frames == 1 && g.N % 128 == 0) ? 1 : 0;
  p.b_merged = (g.Cout % e.chunk == 0) ? 1 : 0;
  // frames of a 3-D conv start in_frame_step floats apart and see Cin (= Cin3d*kt) channels
  if (x_mode) {
    const long long N = g.N;
    if (p.a_merged) {
      if (!merged_image_map(&ma, img, e, g, g.W, g.H, g.Cin, true)) return false;
    } else {
      const long long adims[5] = {N, g.Cin, g.W, g.H, g.frames};
      const long long astr[4] = {N * g.W * g.H, N, N * g.W, g.in_frame_step};
      const int abox[5] = {32, 1, 8, 4, 1};                     // 8 x-taps x 4 filter rows of one channel
      if (!make_map(&ma, img, e, 5, adims, astr, abox)) return false;
    }
    if (p.b_merged) {
      const long long bdims[5] = {32, g.kx, g.ky, g.Cout / 32, g.Cin};
      const long long bstr[4] = {g.Cout, (long long)g.Cout * g.kx, 32, (long long)g.Cout * taps};
      const int bbox[5] = {32, 8, 4, p.BN / 32, 1};
      if (!make_map(&mb, flt, e, 5, bdims, bstr, bbox)) return false;
    } else {
      const long long bdims[4] = {g.Cout, g.kx, g.ky, g.Cin};
      const long long bstr[3] = {g.Cout, (long long)g.Cout * g.kx, (long long)g.Cout * taps};
      const int bbox[4] = {32, 8, 4, 1};
      if (!make_map(&mb, flt, e, 4, bdims, bstr, bbox)) return false;
    }
  } else {
    if (p.a_merged) {
      if (!merged_image_map(&ma, img, e, g, g.W, g.H, g.Cin, false)) return false;
    } else if (!image_map(&ma, img, e, g, g.W, g.H, g.Cin, g.in_frame_step, true, e.bk)) return false;
    if (!filter_map(&mb, flt, e, g.Cout, taps, g.Cin, p.BN, p.b_merged)) return false;
  }
  launch<kFprop>(ma, mb, p);
  if (emit && fuse.emitted) *fuse.emitted = true;
  if (drop && fuse.dropped) *fuse.dropped = true;
  if (p.splits > 1) reduce_split((const float*)ws, out, out_elems, p.splits, st, so, bias, (long long)g.modules * g.N, fuse.relu, nullptr);
  state().last_conv_path = bf ? kPathTcBf16 : kPathTcTf32;
  return true;
}
bool tc_conv_up(const ConvGeom& g, const float* images, const float* filters, float* targets, float st, float so,
                const Fuse& fuse) {
  if (!tc_enabled() || !g.conv) return false;
  if (want_bf16() && tc_conv_up_impl(g, images, filters, targets, st, so, fuse, true)) return true;
  return tc_conv_up_impl(g, images, filters, targets, st, so, fuse, false);
}


// ---- dgrad in fprop form ---------------------------------------------------------------------------------------------
// dInput[n, x, y, c] = sum_{o, taps} der[n, module, o] * w[o, tap, c] is, for the input pixels of one stride phase, a STRIDE-1
// correlation of the derivative with the phase's flipped taps (stage.cu: dgrad_weights).  In that form it is exactly the fprop
// GEMM — A = derivative (MN-major, one request per tile), B = filter bank [c][tap''][o] (MN-major) — with no dead taps to
// walk, where the gather form skips them per tile.  One launch per stride phase; the epilogue writes every sx-th / sy-th pixel.
// does the phase-decomposed dgrad (below) take this call?  `banks` receives the phases
static bool dgrad_as_fprop_eligible(const ConvGeom& g, const float* derivs, const float* filters, DgradBanks* banks) {
  if (!g.conv || g.frames != 1) return false;
  if (g.cin0 != 0 || g.Cin != g.CinT || g.cout0 != 0 || g.Cout != g.CoutT) return false;
  if (g.N % 128 != 0 || g.Cin % 32 != 0 || g.Cout % 8 != 0 || !aligned16(derivs) || !aligned16(filters)) return false;
  if ((long long)g.N * g.W * g.H < 1024) return false;                      // FC-shaped: weight-streaming bound, stays tf32
  if (dgrad_phases(g, banks) <= 0) return false;
  for (int i = 0; i < banks->count; i++) if (banks->phase[i].ku == 0 || banks->phase[i].kv == 0) return false;
  return true;
}

void tc_conv_down_prestage(const ConvGeom& g, const float* derivs, const float* filters) {
  DgradBanks banks;
  if (!tc_enabled() || !g.conv || !want_bf16() || !dgrad_as_fprop_eligible(g, derivs, filters, &banks)) return;
  dgrad_weights(filters, g, banks);
}

static bool tc_conv_down_as_fprop(const ConvGeom& g, const float* derivs, const float* filters, float* targets, float so,
                                  const Fuse& fuse) {
  DgradBanks banks;
  if (!dgrad_as_fprop_eligible(g, derivs, filters, &banks)) return false;
  const Elem e = elem_for(true);
  // the derivative as bf16 (staged by the producer, or converted here)
  const __nv_bfloat16* sd = bf16_staged(derivs, g.out_total);
  if (!sd) {
    __nv_bfloat16* tmp = (__nv_bfloat16*)workspace(align_up((size_t)g.out_total * 2));
    to_bf16(derivs, tmp, g.out_total);
    sd = tmp;
  }
  const __nv_bfloat16* bank = dgrad_weights(filters, g, banks);
  for (int i = 0; i < banks.count; i++) {
    const DgradPhase& P = banks.phase[i];
    TcParams p; fill_common(p, g, e);
    // the GEMM of this phase: rows = (image, phase pixel), K = (tap'', o), columns = input channels
    p.modX = P.Wp; p.modY = P.Hp; p.modules = P.Wp * P.Hp;
    p.W = g.modX; p.H = g.modY;                        // the tensor A is read from (the derivative grid)
    p.kx = P.ku; p.ky = P.kv; p.taps = P.ku * P.kv; p.sx = p.sy = 1; p.px = P.px; p.py = P.py;
    p.Cin = g.Cout; p.Cout = g.Cin;
    p.BN = pick_bn(g.Cin, 64);
    p.kc_blocks = ceil_div(g.Cout, e.bk);
    p.total_chunks = p.nbc * p.modules;
    p.m_tiles = ceil_div(p.total_chunks, p.cpt);
    p.n_tiles = ceil_div(g.Cin, p.BN);
    p.num_tiles = p.m_tiles * p.n_tiles;
    p.b_tx_bytes = (uint32_t)p.BN * 128;
    p.out = targets; p.st = 0.f; p.so = so;
    p.mask = fuse.relu_mask; p.out16 = fuse.out16;
    p.o_sx = g.sx; p.o_sy = g.sy; p.o_x0 = P.a; p.o_y0 = P.b; p.o_W = g.W; p.out_plane = (long long)g.W * g.H;
    p.a_merged = 1;
    p.b_merged = (g.Cin % 64 == 0) ? 1 : 0;
    CUtensorMap fa, fb;
    if (!merged_image_map(&fa, sd, e, g, g.modX, g.modY, g.Cout, false) ||
        !filter_map(&fb, bank + P.offset, e, g.Cin, p.taps, g.Cout, p.BN, p.b_merged)) {
      CNB_REQUIRE(i == 0, "dgrad-as-fprop: tensor map failed after the first phase");
      return false;
    }
    launch<kFprop>(fa, fb, p);
  }
  if (fuse.out16 && fuse.emitted) *fuse.emitted = true;
  state().last_conv_path = kPathTcBf16;
  return true;
}

// ---- dgrad ---------------------------------------------------------------------------------------
static bool tc_conv_down_impl(const ConvGeom& g, const float* derivs, const float* filters, float* targets, float st, float so,
                              const Fuse& fuse, bool bf) {
  const Elem e = elem_for(bf);
  if (g.N % 4 != 0 || g.Cout % 4 != 0 || g.Cout < 8 || g.Cin < 8) return false;
  if (bf && (g.N % 8 != 0 || g.Cout % 8 != 0 || !aligned16(derivs) || !aligned16(filters))) return false;
  if (bf && (long long)g.N * g.W * g.H < 1024 && !bf16_staged(filters, (long long)g.Cout * g.K)) return false;   // see tc_conv_up_impl
  TcParams p; fill_common(p, g, e);
  p.BN = pick_bn(g.Cin, 16);
  p.kc_blocks = ceil_div(g.Cout, e.bk);
  const long long chunks = (long long)p.nb * g.W * g.H;
  if (chunks * 4 >= (1LL << 31) || g.kx > 32 || g.ky > 32) return false;
  p.total_chunks = p.nbc * g.W * g.H;
  p.m_tiles = ceil_div(p.total_chunks, p.cpt);
  p.n_tiles = ceil_div(g.Cin, p.BN);
  p.num_tiles = p.m_tiles * p.n_tiles;
  p.so = so;
  p.b_tx_bytes = (uint32_t)p.BN * 128;
  const bool whole = (g.frames == 1 && g.cin0 == 0 && g.Cin == g.CinT);
  const long long out_elems = (long long)g.Cin * g.W * g.H * g.N;
  const int ks = whole ? pick_ksplit(p, g, out_elems) : 1;
  if (ks > 1) {
    p.units_per_split = ceil_div(p.kc_blocks, ks);
    p.splits = ceil_div(p.kc_blocks, p.units_per_split);
    p.part_stride = out_elems;
    p.num_tiles *= p.splits;
  }
  const size_t part_bytes = p.splits > 1 ? align_up(sizeof(float) * out_elems * p.splits) : 0;
  CUtensorMap ma, mb;
  const long long der_off = (long long)g.cout0 * g.modules * g.N;
  const void* der = derivs + der_off;
  const void* flt = filters;
  uint8_t* ws = nullptr;
  if (bf) {
    const __nv_bfloat16* sd = bf16_staged(derivs, g.out_total);
    const __nv_bfloat16* sf = bf16_staged(filters, (long long)g.Cout * g.K);
    const size_t db = sd ? 0 : align_up((size_t)g.out_total * 2), fb = sf ? 0 : align_up((size_t)g.Cout * g.K * 2);
    if (part_bytes + db + fb) ws = (uint8_t*)workspace(part_bytes + db + fb);
    if (!sd) { to_bf16(derivs, (__nv_bfloat16*)(ws + part_bytes), g.out_total); sd = (const __nv_bfloat16*)(ws + part_bytes); }
    if (!sf) { to_bf16(filters, (__nv_bfloat16*)(ws + part_bytes + db), (long long)g.Cout * g.K); sf = (const __nv_bfloat16*)(ws + part_bytes + db); }
    der = sd + der_off;
    flt = sf;
  } else if (part_bytes) {
    ws = (uint8_t*)workspace(part_bytes);
  }
  p.a_merged = (g.frames == 1 && g.N % 128 == 0) ? 1 : 0;
  if (p.a_merged) {
    if (!merged_image_map(&ma, der, e, g, g.modX, g.modY, g.Cout, false)) return false;
  } else if (!image_map(&ma, der, e, g, g.modX, g.modY, g.Cout, g.out_frame_step, true, e.bk)) return false;
  {
    const long long dims[3] = {g.Cout, (long long)g.kx * g.ky, g.Cin};
    const long long str[2] = {g.Cout, (long long)g.Cout * g.kx * g.ky};
    const int box[3] = {e.chunk, 1, p.BN};
    if (!make_map(&mb, flt, e, 3, dims, str, box)) return false;
  }
  float* out = targets + (long long)g.cin0 * g.H * g.W * g.N;
  if (whole && p.splits > 1) {
    p.st = 0.f; p.out = (float*)ws; p.mask = nullptr;
    launch<kDgrad>(ma, mb, p);
    reduce_split((const float*)ws, out, out_elems, p.splits, st, so, nullptr, 1, 0, fuse.relu_mask);
  } else if (whole) {
    p.st = st; p.out = out; p.mask = fuse.relu_mask ? fuse.relu_mask + (long long)g.cin0 * g.H * g.W * g.N : nullptr;
    p.out16 = fuse.out16;                              // `whole`: every element gets its final value here
    launch<kDgrad>(ma, mb, p);
    if (fuse.out16 && fuse.emitted) *fuse.emitted = true;
  } else {
    // the reference scales the WHOLE target first (gemm.cu:760, conv3d_gemm.cu:98); frame windows overlap,
    // so frames are accumulated by stream-ordered launches
    scale_buffer(targets, g.img_total, st);
    p.st = 1.f;
    for (int f = 0; f < g.frames; f++) {
      p.frame0 = f; p.out = out + f * g.in_frame_step;
      launch<kDgrad>(ma, mb, p);
    }
  }
  state().last_conv_path = bf ? kPathTcBf16 : kPathTcTf32;
  return true;
}
bool tc_conv_down(const ConvGeom& g, const float* derivs, const float* filters, float* targets, float st, float so,
                  const Fuse& fuse) {
  if (!tc_enabled() || !g.conv) return false;
  if (want_bf16() && st == 0.f && tc_conv_down_as_fprop(g, derivs, filters, targets, so, fuse)) return true;
  if (want_bf16() && tc_conv_down_impl(g, derivs, filters, targets, st, so, fuse, true)) return true;
  return tc_conv_down_impl(g, derivs, filters, targets, st, so, fuse, false);
}

// ---- wgrad ---------------------------------------------------------------------------------------
static bool tc_conv_outp_impl(const ConvGeom& g, const float* images, const float* derivs, float* targets, float st, float so,
                              bool bf) {
  const Elem e = elem_for(bf);
  if (g.N % 4 != 0 || g.Cout < 8) return false;
  const bool x_mode = g.Cin < 8;
  if (x_mode && (g.kx > 8 || g.ky > 8)) return false;
  if (bf && (x_mode || g.N % 8 != 0 || !aligned16(images) || !aligned16(derivs))) return false;
  // few reduction rows (FC layers: K = batch): the call is bound by WRITING dW, and the operands a bf16 pass would convert
  // are tiny — such shapes take bf16 only in the whole-batch-tile layout the training step uses
  if (bf && (long long)g.N * g.modules * g.frames < 1024 && !(g.frames == 1 && g.N % 128 == 0 && g.Cin % 32 == 0)) return false;
  TcParams p; fill_common(p, g, e);
  p.kc_blocks = 0;
  p.m_tiles = ceil_div(g.Cout, BM);
  if (x_mode) {
    p.x_mode = 1;
    p.x_ct = std::min(g.Cin, BN_MAX / (8 * g.ky));   // channels per N tile: x_ct * ky * 8 columns
    p.BN = ceil_div(p.x_ct * g.ky * 8, 16) * 16;
    p.n_tiles = ceil_div(g.Cin, p.x_ct);
    p.b_tx_bytes = (uint32_t)p.x_ct * g.ky * 8 * 128;
  } else {
    p.BN = pick_bn(g.Cin, 16);
    p.n_tiles = ceil_div(g.Cin, p.BN);
    p.b_tx_bytes = (uint32_t)p.BN * 128;
  }
  const int units = g.modY * g.frames;               // reduction units = module rows
  const long long base_tiles = (long long)(x_mode ? 1 : p.taps) * p.m_tiles * p.n_tiles;
  // reduction splits: minimise  waves x (rows per tile x time of a row + epilogue)  +  the partial-sum reduction pass.
  // Times in microseconds, coarse: one k-block ~0.3 us, a tile epilogue ~1.5 us, the reduction streams (splits + 1) x |dW|
  // floats at ~3 TB/s.
  int splits;
  {
    const long long slots = num_sms();
    const double row_us = 0.3 * g.modX * std::max(1, p.nbc / 2);
    const double dw_bytes = 4.0 * g.Cout * g.K;
    const int cap = (int)std::max<long long>(1, std::min<long long>(units, (4LL * num_sms()) / std::max<long long>(base_tiles, 1)));
    double best = 1e30; splits = 1;
    for (int sp = 1; sp <= cap; sp++) {
      const int ups = ceil_div(units, sp), real = ceil_div(units, ups);
      const long long waves = ceil_div<long long>(base_tiles * real, slots);
      const double cost = (double)waves * (ups * row_us + 1.5) + (real > 1 ? dw_bytes * (real + 1) / 3e6 : 0.0);
      if (cost < best - 1e-9) { best = cost; splits = real; }
    }
  }
  const long long elems = (long long)g.Cout * g.K;
  while (splits > 1 && elems * splits * 4 > (1LL << 30)) splits--;
  p.units_per_split = ceil_div(units, splits);
  p.splits = ceil_div(units, p.units_per_split);
  p.num_tiles = (int)(base_tiles * p.splits);
  p.st = st; p.so = so;
  CUtensorMap ma, mb;
  const long long img_off = (long long)g.cin0 * g.H * g.W * g.N, der_off = (long long)g.cout0 * g.modules * g.N;
  const void* img = images + img_off;
  const void* der = derivs + der_off;
  const size_t part_bytes = p.splits > 1 ? align_up(sizeof(float) * elems * p.splits) : 0;
  uint8_t* ws = nullptr;
  if (bf) {
    const __nv_bfloat16* si = bf16_staged(images, g.img_total);
    const __nv_bfloat16* sd = bf16_staged(derivs, g.out_total);
    const size_t ib = si ? 0 : align_up((size_t)g.img_total * 2), db = sd ? 0 : align_up((size_t)g.out_total * 2);
    if (part_bytes + ib + db) ws = (uint8_t*)workspace(part_bytes + ib + db);
    if (!si) { to_bf16(images, (__nv_bfloat16*)(ws + part_bytes), g.img_total); si = (const __nv_bfloat16*)(ws + part_bytes); }
    if (!sd) { to_bf16(derivs, (__nv_bfloat16*)(ws + part_bytes + ib), g.out_total); sd = (const __nv_bfloat16*)(ws + part_bytes + ib); }
    img = si + img_off;
    der = sd + der_off;
  } else if (part_bytes) {
    ws = (uint8_t*)workspace(part_bytes);
  }
  if (!image_map(&ma, der, e, g, g.modX, g.modY, g.Cout, g.out_frame_step, false, BM)) return false;
  if (x_mode) {
    const long long N = g.N;
    const long long dims[5] = {N, g.W, g.H, g.Cin, g.frames};
    const long long str[4] = {N, N * g.W, N * g.W * g.H, g.in_frame_step};
    const int box[5] = {32, 8, g.ky, 1, 1};                   // 8 x-taps x ky rows of one channel: ky*8 GEMM columns
    if (!make_map(&mb, img, e, 5, dims, str, box)) return false;
  } else if (!image_map(&mb, img, e, g, g.W, g.H, g.Cin, g.in_frame_step, false, p.BN)) return false;
  p.out = p.splits == 1 ? targets : (float*)ws;
  launch<kWgrad>(ma, mb, p);
  if (p.splits > 1) reduce_partials((const float*)ws, targets, elems, 1, p.splits, st, so);
  state().last_conv_path = bf ? kPathTcBf16 : kPathTcTf32;
  return true;
}
bool tc_conv_outp(const ConvGeom& g, const float* images, const float* derivs, float* targets, float st, float so) {
  if (!tc_enabled() || !g.conv) return false;
  if (want_bf16() && tc_conv_outp_impl(g, images, derivs, targets, st, so, true)) return true;
  return tc_conv_outp_impl(g, images, derivs, targets, st, so, false);
}

}  // namespace cnb
