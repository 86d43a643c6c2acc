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
// One persistent CTA per SM, 12 or 16 warps: warps 0..7 are two consumer warpgroups (GEMM rows 0-63 and 64-127 of the
// 128 x 128 tile), warp 8 is the TMA producer filling a ring of shared-memory stages guarded by mbarriers, the SW = 3
// or 7 warps after it store the fprop / dgrad output tiles (the launch plan picks SW: pick_store_warps).
//   bf16 operands: wgmma.mma_async m64n128k16 reads both operands from the swizzled tiles (either major);
//   tf32 operands: wgmma takes 32-bit operands from shared memory only K-major, so
//     wgrad (both operands K-major): wgmma m64n128k8 on the tiles, as bf16;
//     x-mode fprop (Cin < 8): wgmma m64nNk8 with A (the MN-major image tile) loaded into registers and B the n-tile's
//                  filter bank, written K-major into shared memory once per CTA and kept there;
//     other fprop / dgrad (MN-major operands): mma.sync m16n8k8 with fragments loaded from the tiles.
// Accumulators live in registers.  fprop / dgrad: the consumers copy a finished tile into a shared-memory staging tile and
// go on to the next tile's k-blocks; the store warps apply the epilogue and write it with 16-byte stores (one warp
// instruction = 128 consecutive images of one channel).  wgrad: the consumers store their tile straight from registers.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cudaTypedefs.h>

#include <algorithm>
#include <type_traits>
#include <vector>

#include "conv_kernels.h"
#include "sm90_ptx.cuh"

namespace cnb {

namespace {

constexpr int kConsumerWarps = 8;
// Threads of a CTA with SW store warps: 384 (ptxas caps a thread at 168 registers) or 512 (128 registers)
template <int SW> constexpr int kThreadsFor = 32 * (kConsumerWarps + 1 + SW);
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
  // x-mode fprop: B is no ring but the filter bank of the tile's n-tile, resident in shared memory after the A ring
  // (bank_bytes = Cin * x_yblocks * BN * 128), filled from the caller's filters `xw` ([c][ty][tx][o], o contiguous)
  const float* xw;
  uint32_t bank_bytes;              // 0: the B half of the ring follows the A ring
  uint32_t epi_bytes;               // fprop / dgrad: the staging tile (BM x BN fp32) after the ring or bank; wgrad: the
                                    // consumer warps' transpose areas (kWgradStageBytes), or 0 for the scalar stores
  uint32_t b_tx_bytes;              // bytes the B-operand TMA(s) of one stage actually deliver
  // merged requests: when N % 128 == 0 (2-D) the chunks of an m-tile are one box over a (chunk, ..., N/chunk, ...) view
  // of the tensor; when Cout % chunk == 0 the BN/chunk filter chunks are one box likewise.
  int a_merged, b_merged;
  // untied filters (localUp / localDown / localOutp): one [K x Cout] bank per module, banks consecutive, and the B tensor
  // map has a module dimension.  Only with N % 128 == 0 (2-D), so that every fprop / dgrad m-tile lies in ONE module /
  // input pixel.  wgrad: `split` is the module, the reduction runs over the images alone.
  int untied;
  int total_chunks;                // fprop: nbc*modules*frames ; dgrad: nbc*W*H   (< 2^31, checked on the host)
  int splits, units_per_split;      // wgrad: (frame, module-row) units per reduction split;
                                    // fprop/dgrad of 1x1 / FC shapes with few tiles: K blocks per split (split-K)
  long long part_stride;            // fprop/dgrad split-K: floats between the partial outputs of consecutive splits
  float* out;
  __nv_bfloat16* out16;             // optional bf16 twin of `out` (same indexing): convnet_b200_emit_bf16_next
  int vec;                          // out / mask 16-byte and out16 8-byte aligned: the store warps move 4 rows at once
  float st, so;
  const float* bias; int act;       // fused fprop epilogue: + bias[o], then act_apply(., act)
  const float* mask; int mask_act;  // fused epilogue: act_deriv(., mask, mask_act) (mask: same layout as out)
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
  uint64_t epi_full;                // the 8 consumer warps have written the staging tile
  uint64_t epi_empty;               // the store warps have read it
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
  } else if (p.untied) {
    return p.nbc;
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

// ---- x-mode fprop on tf32 wgmma -------------------------------------------------------------------------------------
// The k-block of stage rows 8s .. 8s+7 is k-step s.  Inside a k-step, logical k j of the wgmma sits in stage K row
// 2(j&3) + (j>>2): the A fragment of lane (g, q) is then K rows 2q and 2q+1, and the 16-byte units (row>>2 ^ K row) & 7
// that one load instruction of a warp touches are all distinct — no bank conflicts.  The filter bank follows the same
// permutation.
__device__ __forceinline__ int xmode_k_row(int k) { return (k & ~7) | ((k & 3) << 1) | ((k >> 2) & 1); }

// The n-tile's filter bank, K-major [k-block (c, yb)][BN columns][32 K] with the 128-byte swizzle, written by the 256
// consumer threads: stage K row r of k-block (c, yb) is tap tx = r & 7 of filter row ty = 4 yb + (r >> 3).  The raw fp32
// bits (the tensor core reads their tf32 part, as it does the images), and exact zeros at taps tx >= kx, rows ty >= ky
// and columns beyond Cout: the A box covers 8 x 4 real pixels whatever the kernel size.
__device__ __forceinline__ void xmode_fill_bank(const TcParams& p, uint8_t* bank, int n_tile) {
  const int total = p.Cin * p.x_yblocks * 32 * p.BN;
#pragma unroll 8
  for (int i = threadIdx.x; i < total; i += 32 * kConsumerWarps) {
    const int n = i % p.BN, rest = i / p.BN, k = rest & 31, kb = rest >> 5;
    const int r = xmode_k_row(k), c = kb / p.x_yblocks, ty = 4 * (kb % p.x_yblocks) + (r >> 3), tx = r & 7;
    const int o = n_tile * p.BN + n;
    float v = 0.f;
    if (tx < p.kx && ty < p.ky && o < p.Cout) v = __ldg(p.xw + o + (long long)p.Cout * (tx + p.kx * (ty + p.ky * c)));
    *reinterpret_cast<float*>(bank + (size_t)kb * p.BN * 128 + off_kmajor(n, k)) = v;
  }
}

// The k-blocks of one x-mode fprop tile: per stage, this warp's 16 rows of A into registers, then four wgmma m64nNk8
// against the resident bank, and wgmma.wait_group 0 before the next stage's fragment loads.  (Loading the next fragment
// into a second register buffer while the group is in flight makes ptxas serialize every wgmma — C7513, "non wgmma
// instructions defining input registers ... between start and end of the pipeline stage" — so the overlap comes from
// the other warpgroup instead.)  The slot is released once its MMAs retired.
template <int N>
__device__ __forceinline__ void xmode_fprop_mma(float (&acc)[16][4], const TcParams& p, SmemCtl* ctl, uint32_t sA,
                                                uint32_t bank, int nkb, int& stage, uint32_t& phase, int row0, int tq,
                                                int lane) {
  const uint64_t db0 = ptx::gmma_desc(bank, 16u, 1024u);
  ptx::wgmma_fence_operands(acc);
  for (int kb = 0; kb < nkb; kb++) {
    ptx::mbar_wait(&ctl->full[stage], phase);
    const uint32_t A = sA + (uint32_t)stage * kAStageBytes;
    uint32_t a[4][4];
#pragma unroll
    for (int ks = 0; ks < 4; ks++) {
      const int k0 = ks * 8 + 2 * tq;
      a[ks][0] = ptx::lds32(A + off_mnmajor(row0, k0));
      a[ks][1] = ptx::lds32(A + off_mnmajor(row0 + 8, k0));
      a[ks][2] = ptx::lds32(A + off_mnmajor(row0, k0 + 1));
      a[ks][3] = ptx::lds32(A + off_mnmajor(row0 + 8, k0 + 1));
    }
    ptx::wgmma_fence();                            // orders the fragment writes before the wgmma reads them
    const uint64_t db = db0 + ((uint32_t)kb * (N * 128) >> 4);
#pragma unroll
    for (int ks = 0; ks < 4; ks++) ptx::wgmma_m64nNk8_tf32_rs<N>(acc, a[ks], db + (ks * 32 >> 4));
    ptx::wgmma_commit();
    ptx::wgmma_wait<0>();                          // the fragment registers are free again, and so is the slot
    if (lane == 0) ptx::mbar_arrive(&ctl->empty[stage]);
    if (++stage == p.stages) { stage = 0; phase ^= 1; }
  }
  ptx::wgmma_fence_operands(acc);
}

// ---- fprop / dgrad epilogue: the staging tile and the store warps ---------------------------------------------------
// Byte offset of (row, col) in the staging tile: column-major, 512 bytes per column, the 16-byte unit row / 4 XORed with
// col & 7.  A consumer st.shared of one accumulator (lanes g = 0..7 on 8 consecutive rows, tq = 0..3 on columns 2 tq + e)
// then hits 32 distinct banks, and a store warp's ld.shared.v4 of one column reads 512 contiguous bytes.
__device__ __forceinline__ uint32_t epi_off(int row, int col) {
  return (uint32_t)(col * (BM * 4) + ((((row >> 2) ^ col) & 7) << 4) + (((row >> 2) & ~7) << 4) + ((row & 3) << 2));
}

// ---- wgrad epilogue: each consumer warp writes its 16 rows x BN columns of dW, 32 columns at a time, through a 2 KiB
// area of its own: column-major, 64 bytes per column, the 16-byte unit row / 4 XORed with (col / 2) & 3.  A lane then
// reads 4 consecutive rows (output features o, dW's contiguous axis) of one column with one ld.shared.v4 and writes them
// with one 16-byte store, where a store straight from the accumulators moves 4 bytes per lane.
constexpr int kWgradPassCols = 32;
constexpr uint32_t kWgradWarpBytes = 16 * kWgradPassCols * 4;
constexpr uint32_t kWgradStageBytes = kConsumerWarps * kWgradWarpBytes;
__device__ __forceinline__ uint32_t wgrad_stage_off(int row, int col) {
  return (uint32_t)(col * 64 + ((((row >> 2) ^ (col >> 1)) & 3) << 4) + ((row & 3) << 2));
}

__device__ __forceinline__ float4 ld4(const float* a, bool vec) {
  if (vec) return *reinterpret_cast<const float4*>(a);
  return make_float4(a[0], a[1], a[2], a[3]);
}
__device__ __forceinline__ float4 ldg4(const float* a, bool vec) {
  if (vec) return __ldg(reinterpret_cast<const float4*>(a));
  return make_float4(__ldg(a), __ldg(a + 1), __ldg(a + 2), __ldg(a + 3));
}

// Store warp `sw` (0..SW-1) of the CTA: for each of the CTA's tiles, wait until the consumers have staged it, then write
// columns sw, sw + SW, ... (a warp with no column, when the tile has fewer than SW, only releases the tile).  Lane l
// holds rows 4l .. 4l+3, four consecutive images of one chunk: with N % 4 == 0 they are all valid or all not.  Each
// element gets exactly the arithmetic of the in-register epilogue it replaces.  The loads an element's store depends on
// (old target, ReLU' mask, bias) are issued ahead of the stores they would otherwise wait behind, since a store may
// alias a later load as far as the compiler knows: the bias once per tile, the old target and the mask one batch of
// kEpiCols columns ahead.
template <int OP, bool SIG, int SW>
__device__ __forceinline__ void store_tiles(const TcParams& p, SmemCtl* ctl, uint32_t stg, int sw, int lane) {
  constexpr int kStoreWarps = SW;
  // columns per batch.  Three warps: 8 (4 in the logistic instances, whose arithmetic needs the registers of half the
  // batch); seven: 4, which fits their 128 registers
  constexpr int kEpiCols = (SW == 3 && !SIG) ? 8 : 4;
  const bool vec = p.vec != 0;
  const int lr = 4 * lane;                          // this lane's first row
  const int per_frame = (OP == kFprop) ? p.modules : p.W * p.H;
  const long long col_stride = (long long)p.N * (OP == kFprop ? p.out_plane : (long long)per_frame);
  const bool direct_scale = p.splits == 1;
  const float so_eff = direct_scale ? p.so : 1.f;
  const bool rmw = direct_scale && p.st != 0.f;
  uint32_t phase = 0;
  for (int t = blockIdx.x; t < p.num_tiles; t += gridDim.x) {
    const Tile tile = decode_tile<OP>(p, t);
    long long row = -1;                               // offset of this lane's first row from p.out, -1: no rows
    const int q = tile.m_tile * p.cpt + (lr >> p.chunk_shift);
    if (q < p.total_chunks) {
      const int ib = q % p.nbc, rr = q / p.nbc, pos = rr % per_frame, f = rr / per_frame;
      const int n = ib * p.chunk + (lr & (p.chunk - 1));
      if (n < p.N) {
        if (OP == kFprop) {
          const int i = pos % p.modX, j = pos / p.modX;
          const long long pix = (long long)(i * p.o_sx + p.o_x0) + (long long)p.o_W * (j * p.o_sy + p.o_y0);
          row = f * p.out_frame_step + n + (long long)p.N * pix;
        } else {
          row = n + (long long)p.N * pos;
        }
        row += col_stride * ((long long)tile.n_tile * p.BN) + tile.split * p.part_stride;
      }
    }
    const int ncols = min(p.BN, (OP == kFprop ? p.Cout : p.Cin) - tile.n_tile * p.BN);
    const float* bias = (OP == kFprop && p.bias) ? p.bias + tile.n_tile * p.BN : nullptr;
    int bias_step = 1;
    if (OP == kFprop && p.bias && p.untied) {         // one bias per output feature: bias[module + modules * o]
      bias = p.bias + (tile.m_tile * p.cpt / p.nbc) + (long long)p.modules * tile.n_tile * p.BN;
      bias_step = p.modules;
    }
    const int mine = ncols > sw ? (ncols - sw + kStoreWarps - 1) / kStoreWarps : 0;
    const int batches = (mine + kEpiCols - 1) / kEpiCols;
    // the bias of this warp's (at most 43) columns, loaded once per tile before the wait: lane l holds that of its
    // l-th and (l+32)-th column, and a batch takes them by shuffle.  A bias load inside a batch would wait a full
    // memory round trip behind the previous batch's stores, which the compiler must assume may alias it.
    static_assert(BN_MAX <= 64 * kStoreWarps, "two bias values per lane cover a store warp's columns");
    constexpr bool kBiasHi = BN_MAX > 32 * kStoreWarps;   // seven warps: at most 19 columns, one value per lane
    float bias_lo = 0.f, bias_hi = 0.f;
    if (OP == kFprop && bias) {
      const int ca = sw + kStoreWarps * lane, cb = ca + kStoreWarps * 32;
      if (ca < ncols) bias_lo = __ldg(bias + ca * bias_step);
      if (kBiasHi && cb < ncols) bias_hi = __ldg(bias + cb * bias_step);
    }
    // the loads a batch's arithmetic depends on (old target, ReLU' mask), software-pipelined: batch b+1's are issued
    // after batch b's arithmetic and before its stores, and batch 0's before the wait for the tile.  Issued after the
    // previous batch's stores instead, each batch would wait one full memory round trip.  Batches cover disjoint
    // columns, so a load never reads an element that an earlier store in program order wrote.
    float4 acc[kEpiCols], old[kEpiCols], msk[kEpiCols];
    auto load_batch = [&](int b) {
      const int c0 = sw + kStoreWarps * kEpiCols * b;
#pragma unroll
      for (int k = 0; k < kEpiCols; k++) {
        const int col = c0 + kStoreWarps * k;
        old[k] = msk[k] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (row < 0 || col >= ncols) continue;
        const long long idx = row + col_stride * col;
        if (rmw) old[k] = ld4(p.out + idx, vec);
        if (p.mask) msk[k] = ldg4(p.mask + idx, vec);
      }
    };
    if (batches > 0) load_batch(0);
    ptx::mbar_wait(&ctl->epi_full, phase);
    if (batches == 0 && lane == 0) ptx::mbar_arrive(&ctl->epi_empty);
    // The batches, compiled twice: LEAN, the plain writes of a forward pass (no old target, mask or dropout;
    // 16-byte aligned), and every other call.  Branches on work a call does not do, inside the loop over the
    // elements, cost the store warps a third of conv1 fprop's time on an H100 (DESIGN.md §6).
    auto drain = [&](auto lean) {
      constexpr bool LEAN = decltype(lean)::value;
      for (int b = 0; b < batches; b++) {
        const int c0 = sw + kStoreWarps * kEpiCols * b;
        float bv[kEpiCols];
#pragma unroll
        for (int k = 0; k < kEpiCols; k++) {
          const int col = c0 + kStoreWarps * k;
          acc[k] = col < ncols ? ptx::lds128(stg + epi_off(lr, col)) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
        if (b == batches - 1) {                         // the last read of the staging tile: the consumers may refill it
          __syncwarp();
          if (lane == 0) ptx::mbar_arrive(&ctl->epi_empty);
        }
        if (OP == kFprop && bias) {
#pragma unroll
          for (int k = 0; k < kEpiCols; k++) {          // column c0 + SW k is this warp's (kEpiCols b + k)-th
            const int j = kEpiCols * b + k;
            bv[k] = __shfl_sync(0xffffffffu, (kBiasHi && j >= 32) ? bias_hi : bias_lo, j & 31);
          }
        }
        if (row < 0) continue;
#pragma unroll
        for (int k = 0; k < kEpiCols; k++) {            // the results replace the accumulators in acc
          const int col = c0 + kStoreWarps * k;
          if (col >= ncols) continue;
          const long long idx = row + col_stride * col;
          const float a[4] = {acc[k].x, acc[k].y, acc[k].z, acc[k].w};
          const float o[4] = {old[k].x, old[k].y, old[k].z, old[k].w};
          const float m[4] = {msk[k].x, msk[k].y, msk[k].z, msk[k].w};
          float v[4];
#pragma unroll
          for (int e = 0; e < 4; e++) {
            float r = so_eff * a[e];
            if (!LEAN && rmw) r += p.st * o[e];
            if (OP == kFprop) {
              if (bias) r += bv[k];
              if (SIG) { if (p.act) r = act_apply(r, p.act); }
              else if (p.act) r = fmaxf(r, 0.f);
              if (!LEAN && p.drop_scale != 0.f) r *= dropout_keep(p.drop_seed + (unsigned long long)(idx + e), p.drop_prob, p.drop_scale);
            }
            if (!LEAN) {
              if (SIG) { if (p.mask) r = act_deriv(r, m[e], p.mask_act); }
              else if (p.mask && !(m[e] > 0.f)) r = 0.f;
            }
            v[e] = r;
          }
          acc[k] = make_float4(v[0], v[1], v[2], v[3]);
        }
        if (!LEAN && (rmw || p.mask) && b + 1 < batches) load_batch(b + 1);
#pragma unroll
        for (int k = 0; k < kEpiCols; k++) {
          const int col = c0 + kStoreWarps * k;
          if (col >= ncols) continue;
          const long long idx = row + col_stride * col;
          const float v[4] = {acc[k].x, acc[k].y, acc[k].z, acc[k].w};
          float* const dst = p.out + idx;
          if (LEAN || vec) {
            *reinterpret_cast<float4*>(dst) = acc[k];
          } else {
#pragma unroll
            for (int e = 0; e < 4; e++) dst[e] = v[e];
          }
          if (p.out16) {
            __nv_bfloat16* const d16 = p.out16 + idx;
            const __nv_bfloat162 lo = __floats2bfloat162_rn(v[0], v[1]), hi = __floats2bfloat162_rn(v[2], v[3]);
            if (LEAN || vec) {
              uint2 w;
              w.x = *reinterpret_cast<const uint32_t*>(&lo);
              w.y = *reinterpret_cast<const uint32_t*>(&hi);
              *reinterpret_cast<uint2*>(d16) = w;
            } else {
              d16[0] = lo.x; d16[1] = lo.y; d16[2] = hi.x; d16[3] = hi.y;
            }
          }
        }
      }
    };
    if (!rmw && !p.mask && !(OP == kFprop && p.drop_scale != 0.f) && vec) drain(std::true_type{});
    else drain(std::false_type{});
    phase ^= 1;
  }
}

// ------------------------------------------------------------------------------------------------
// SIG: the epilogue applies the activation code (logistic included); the other instances know only ReLU / ReLU', so the
// logistic arithmetic costs the ReLU and linear layers nothing
template <int OP, bool BF16, bool SIG, int SW>
__global__ void __launch_bounds__(kThreadsFor<SW>, 1)
tc_conv_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB, const __grid_constant__ TcParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smemA = smem;
  uint8_t* smemB = smem + (size_t)p.stages * kAStageBytes;      // the B ring, or the x-mode fprop filter bank
  uint8_t* smemE = smemB + (p.bank_bytes ? (size_t)p.bank_bytes : (size_t)p.stages * kBStageBytes);   // staging tile
  SmemCtl* ctl = reinterpret_cast<SmemCtl*>(smemE + p.epi_bytes);

  // warp index through a shuffle: provably warp-uniform, which keeps the role branches and their loops on the uniform path
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.stages; s++) { ptx::mbar_init(&ctl->full[s], 1); ptx::mbar_init(&ctl->empty[s], kConsumerWarps); }
    ptx::mbar_init(&ctl->epi_full, kConsumerWarps);
    ptx::mbar_init(&ctl->epi_empty, SW);
    ptx::fence_barrier_init();
    ptx::tma_prefetch_desc(&mapA);
    ptx::tma_prefetch_desc(&mapB);
  }
  __syncthreads();
  ptx::pdl_launch_dependents();       // the kernel queued behind this one may start its prologue (it waits for this grid's end)
  ptx::pdl_wait();                    // ... as this one's just overlapped its predecessor's tail; from here on: global memory

  if (warp > kConsumerWarps) {
    // =============================== store warps (fprop / dgrad) ===============================
    if constexpr (OP != kWgrad) store_tiles<OP, SIG, SW>(p, ctl, ptx::smem_u32(smemE), warp - kConsumerWarps - 1, lane);
    return;
  }
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
        if (p.x_mode) {                        // A only: B is the consumers' resident filter bank
          for (int c = 0; c < p.Cin; c++)
            for (int yb = 0; yb < p.x_yblocks; yb++) {
              uint8_t* a = begin_stage();
              if (p.a_merged) {                // dims (n_lo, x, y, n_hi, c): one 16 KiB request
                lda5(&mapA, a, 0, cX[0], cY[0] + 4 * yb, ch.n[0] >> 5, c);
              } else {
#pragma unroll
                for (int q = 0; q < 4; q++)    // 8 consecutive x pixels x 4 filter rows of channel c = 32 K rows
                  lda5(&mapA, a + q * (BK * 128), ch.n[q], c, cX[q], cY[q] + 4 * yb, ch.f[q]);
              }
              end_stage();
            }
        } else {
          // split-K (host: only when taps == 1): this tile reduces K blocks [cb0, cb1)
          const int cb0 = p.splits > 1 ? tile.split * p.units_per_split : 0;
          const int cb1 = p.splits > 1 ? min(cb0 + p.units_per_split, p.kc_blocks) : p.kc_blocks;
          const int mod = ch.pos[0];                  // untied: the module of the whole tile
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
                if (p.b_merged) {                // dims (o_lo, c, o_hi, tap[, module])
                  if (p.untied) lda5(&mapB, b, 0, cb * p.bk, o0 >> p.chunk_shift, tap, mod);
                  else lda4(&mapB, b, 0, cb * p.bk, o0 >> p.chunk_shift, tap);
                } else {
                  for (int j = 0; j < ((p.BN + p.chunk - 1) >> p.chunk_shift); j++) {
                    if (p.untied) lda4(&mapB, b + j * (p.bk * 128), o0 + j * p.chunk, tap, cb * p.bk, mod);
                    else lda3(&mapB, b + j * (p.bk * 128), o0 + j * p.chunk, tap, cb * p.bk);
                  }
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
            // untied: the tile's pixel reaches this tap through one module, whose bank B reads (-1: none -> zeros)
            const int mod = mx[0] >= 0 ? mx[0] + p.modX * my[0] : -1;
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
              if (p.untied) lda4(&mapB, b, ob * p.bk, tap, tile.n_tile * p.BN, mod);
              else lda3(&mapB, b, ob * p.bk, tap, tile.n_tile * p.BN);
              end_stage();
            }
          }
      } else if (p.untied) {
        // dW_module[o, tap, c]: the reduction runs over the images alone; a tap outside the image is zero-filled by TMA
        const int mx = tile.split % p.modX, my = tile.split / p.modX;
        const int X = mx * p.sx + p.px + tile.tap % p.kx, Y = my * p.sy + p.py + tile.tap / p.kx;
        for (int ib = 0; ib < p.nbc; ib++) {
          uint8_t* a = begin_stage();
          uint8_t* b = smemB + (size_t)stage * kBStageBytes;
          lda5(&mapA, a, ib * p.chunk, mx, my, tile.o_tile * BM, 0);
          lda5(&mapB, b, ib * p.chunk, X, Y, tile.c_tile * p.BN, 0);
          end_stage();
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
  int bank_tile = -1;                              // x-mode fprop: the n-tile whose filter bank is in shared memory
  uint32_t epi_phase = 0;                          // fprop / dgrad: parity of the staging tile's handoff
  for (int t = blockIdx.x; t < p.num_tiles; t += gridDim.x) {
    const Tile tile = decode_tile<OP>(p, t);
    const int nkb = tile_kblocks<OP>(p, tile);
    float acc[BN_MAX / 8][4];
#pragma unroll
    for (int j = 0; j < BN_MAX / 8; j++)
#pragma unroll
      for (int e = 0; e < 4; e++) acc[j][e] = 0.f;

    if constexpr (BF16 || OP == kWgrad) {
      // warpgroup w multiplies GEMM rows 64w..64w+63: the second 64-image chunk (MN-major A) or rows 64.. (K-major A),
      // 8 KiB into the stage either way.  tf32 (wgrad only): both operands K-major, the k8 step is +32 B like bf16's k16.
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
        for (int ks = 0; ks < 4; ks++) {
          if constexpr (BF16)
            ptx::wgmma_m64n128k16_bf16<a_mn ? 1 : 0, b_mn ? 1 : 0>(acc, da + (ks * a_step >> 4), db + (ks * b_step >> 4));
          else
            ptx::wgmma_m64n128k8_tf32(acc, da + (ks * a_step >> 4), db + (ks * b_step >> 4));
        }
        ptx::wgmma_commit();
        ptx::wgmma_wait<1>();                        // the previous stage's MMAs have retired: its slot can be refilled
        if (prev >= 0 && lane == 0) ptx::mbar_arrive(&ctl->empty[prev]);
        prev = stage;
        if (++stage == p.stages) { stage = 0; phase ^= 1; }
      }
      ptx::wgmma_wait<0>();
      ptx::wgmma_fence_operands(acc);
      if (prev >= 0 && lane == 0) ptx::mbar_arrive(&ctl->empty[prev]);
    } else if (OP == kFprop && p.x_mode) {
      if (tile.n_tile != bank_tile) {              // uniform over the CTA: every consumer thread sees the same tile
        ptx::bar_sync(1, 32 * kConsumerWarps);     // both warpgroups are past the MMAs that read the previous bank
        xmode_fill_bank(p, smemB, tile.n_tile);
        ptx::fence_proxy_async_smem();             // the generic-proxy stores become visible to wgmma
        ptx::bar_sync(1, 32 * kConsumerWarps);
        bank_tile = tile.n_tile;
      }
      const uint32_t sA = ptx::smem_u32(smemA), bank = ptx::smem_u32(smemB);
      switch (p.BN) {                              // the N sizes x-mode picks (host: tc_conv_up_impl)
        case 32: xmode_fprop_mma<32>(acc, p, ctl, sA, bank, nkb, stage, phase, row0, tq, lane); break;
        case 64: xmode_fprop_mma<64>(acc, p, ctl, sA, bank, nkb, stage, phase, row0, tq, lane); break;
        case 96: xmode_fprop_mma<96>(acc, p, ctl, sA, bank, nkb, stage, phase, row0, tq, lane); break;
        default: xmode_fprop_mma<128>(acc, p, ctl, sA, bank, nkb, stage, phase, row0, tq, lane); break;
      }
    } else {
      // tf32 fprop / dgrad: A MN-major; B MN-major (fprop: the caller's filters) or K-major (dgrad)
      const uint32_t sA = ptx::smem_u32(smemA), sB = ptx::smem_u32(smemB);
      constexpr bool b_mn = (OP == kFprop);
      for (int kb = 0; kb < nkb; kb++) {
        ptx::mbar_wait(&ctl->full[stage], phase);
        const uint32_t A = sA + (uint32_t)stage * kAStageBytes, B = sB + (uint32_t)stage * kBStageBytes;
#pragma unroll
        for (int ks = 0; ks < 4; ks++) {
          const int k0 = ks * 8 + tq, k1 = k0 + 4;
          const uint32_t a0 = ptx::lds32(A + off_mnmajor(row0, k0));
          const uint32_t a1 = ptx::lds32(A + off_mnmajor(row0 + 8, k0));
          const uint32_t a2 = ptx::lds32(A + off_mnmajor(row0, k1));
          const uint32_t a3 = ptx::lds32(A + off_mnmajor(row0 + 8, k1));
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
    if constexpr (OP != kWgrad) {
      // hand the tile to the store warps through the staging tile, then go on to the next tile's k-blocks
      ptx::mbar_wait(&ctl->epi_empty, epi_phase ^ 1);
      // column j*8 + c (c < 8) lies j*8 columns past column c with the same swizzle: four base addresses serve all 64
      uint32_t base[2][2];
#pragma unroll
      for (int h = 0; h < 2; h++)
#pragma unroll
        for (int e = 0; e < 2; e++) base[h][e] = ptx::smem_u32(smemE) + epi_off(row0 + 8 * h, 2 * tq + e);
#pragma unroll
      for (int j = 0; j < BN_MAX / 8; j++) {
        if (j * 8 >= p.BN) break;
#pragma unroll
        for (int h = 0; h < 2; h++)
#pragma unroll
          for (int e = 0; e < 2; e++) ptx::sts32(base[h][e] + j * 8 * BM * 4, acc[j][2 * h + e]);
      }
      __syncwarp();
      if (lane == 0) ptx::mbar_arrive(&ctl->epi_full);
      epi_phase ^= 1;
    } else if (p.epi_bytes) {
      // wgrad, not x-mode, Cout % 4 == 0, dW 16-byte aligned: through this warp's transpose area (wgrad_stage_off).
      // Lane l reads column l / 4 + 8 i of the pass, rows 4 (l & 3) .. + 3: all valid or all not.
      const uint32_t stg = ptx::smem_u32(smemE) + (uint32_t)warp * kWgradWarpBytes;
      const int r4 = 4 * (lane & 3);
      const int o = tile.o_tile * BM + warp * 16 + r4;
      const long long col_stride = (long long)p.Cout * p.taps;
      float* const rp = p.out + (long long)tile.split * p.Cout * p.taps * p.Cin + o + (long long)p.Cout * tile.tap +
                        col_stride * ((long long)tile.c_tile * p.BN);
      const int ncols_valid = min(p.BN, p.Cin - tile.c_tile * p.BN);
      const bool direct_scale = (p.splits == 1) || p.untied;
      const float so_eff = direct_scale ? p.so : 1.f;
      const bool rmw = direct_scale && p.st != 0.f;
#pragma unroll
      for (int pass = 0; pass < BN_MAX / kWgradPassCols; pass++) {
        if (pass * kWgradPassCols >= p.BN) break;
#pragma unroll
        for (int jj = 0; jj < kWgradPassCols / 8; jj++)
#pragma unroll
          for (int h = 0; h < 2; h++)
#pragma unroll
            for (int e = 0; e < 2; e++)
              ptx::sts32(stg + wgrad_stage_off(g + 8 * h, 8 * jj + 2 * tq + e), acc[pass * (kWgradPassCols / 8) + jj][2 * h + e]);
        __syncwarp();
#pragma unroll
        for (int i = 0; i < kWgradPassCols / 8; i++) {
          const int cl = (lane >> 2) + 8 * i, col = pass * kWgradPassCols + cl;
          const float4 a = ptx::lds128(stg + wgrad_stage_off(r4, cl));
          if (o >= p.Cout || col >= ncols_valid) continue;
          float* const dst = rp + col_stride * col;
          const float av[4] = {a.x, a.y, a.z, a.w};
          float ov[4] = {0.f, 0.f, 0.f, 0.f};
          if (rmw) {
            const float4 old = *reinterpret_cast<const float4*>(dst);
            ov[0] = old.x; ov[1] = old.y; ov[2] = old.z; ov[3] = old.w;
          }
          float v[4];
#pragma unroll
          for (int k = 0; k < 4; k++) {
            float r = so_eff * av[k];
            if (rmw) r += p.st * ov[k];
            v[k] = r;
          }
          *reinterpret_cast<float4*>(dst) = make_float4(v[0], v[1], v[2], v[3]);
        }
        __syncwarp();                                // the next pass rewrites the area
      }
    } else {
      // wgrad: dW[o, tap, c] straight from the registers
      float* rowp[2] = {nullptr, nullptr};
      long long col_stride = 0;
#pragma unroll
      for (int h = 0; h < 2; h++) {
        const int o = tile.o_tile * BM + row0 + 8 * h;
        if (o < p.Cout) {
          rowp[h] = p.out + (long long)tile.split * p.Cout * p.taps * p.Cin + o;
          if (!p.x_mode) {
            col_stride = (long long)p.Cout * p.taps;
            rowp[h] += (long long)p.Cout * tile.tap + col_stride * ((long long)tile.c_tile * p.BN);
          }
        }
      }
      const int ncols_valid = p.x_mode ? min(p.BN, p.x_ct * p.ky * 8) : min(p.BN, p.Cin - tile.c_tile * p.BN);
      const bool direct_scale = (p.splits == 1) || p.untied;   // untied wgrad: one dW block per module
      const float so_eff = direct_scale ? p.so : 1.f;
      const bool rmw = direct_scale && p.st != 0.f;
      // where column `col` of a row starting at `rp` lands, or nullptr (x-mode: taps / channels beyond the filter)
      auto dst_of = [&](float* rp, int col) -> float* {
        if (p.x_mode) {
          // column = tap tx + 8*(row ty + ky*channel): scattered to dW[o, tx + kx*(ty + ky*c)]
          const int tx = col & 7, rr = col >> 3, ty = rr % p.ky, c = tile.c_tile * p.x_ct + rr / p.ky;
          if (tx >= p.kx || c >= p.Cin) return nullptr;
          return rp + (long long)p.Cout * (tx + p.kx * (ty + p.ky * c));
        }
        return rp + col_stride * col;
      };
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
            float* const dst = dst_of(rp, col);
            if (dst == nullptr) continue;
            float r = so_eff * acc[j][2 * h + e];
            if (rmw) r += p.st * *dst;
            *dst = r;
          }
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

// dynamic shared memory of a launch with `stages` ring stages: A stages, then B stages or (x-mode fprop) the filter bank,
// then (fprop / dgrad) the staging tile
size_t smem_bytes_for(int stages, uint32_t bank_bytes, uint32_t epi_bytes) {
  const size_t b = bank_bytes ? (size_t)bank_bytes : (size_t)stages * kBStageBytes;
  return 1024 + (size_t)stages * kAStageBytes + b + epi_bytes + sizeof(SmemCtl) + 16;
}
constexpr size_t kSmemBudget = 227 * 1024;        // the most a block may use; launch_one requests it
inline uint32_t epi_bytes_for(int bn) { return (uint32_t)BM * bn * 4; }

int pick_stages(uint32_t bank_bytes, uint32_t epi_bytes) {
  int s = kMaxStages;
  while (s > 2 && smem_bytes_for(s, bank_bytes, epi_bytes) > kSmemBudget) s--;
  return s;
}

// Store warps of an fprop / dgrad launch.  A CTA writes its tiles about as fast as it has warps storing them: on an
// H100, conv1's fprop drains its 595 MB in 0.83 ms with 3 store warps and in 0.53 ms with 7, while sending the same
// stores to a few L2-resident lines, or laying each tile out contiguously, gains far less (DESIGN.md §6).  But
// MMA-bound tiles run 3-5 % slower beside 7 store warps (conv4 fprop; not because 512 threads cap a thread at 128
// registers: the 3-warp kernel built at that cap is as fast as before).  So a plan takes 7 when its tiles are bound by
// their epilogue, or nearly so: when writing a tile's `tile_bytes` takes at least half as long as its `kblocks`
// k-blocks take to multiply.  Times in microseconds, coarse, as in the wgrad split model: one k-block ~0.3 us, the
// tile's traffic at an H100 SM's share of ~3 TB/s (~23 KB/us).
int pick_store_warps(int kblocks, double tile_bytes) {
  const double mma_us = 0.3 * kblocks;
  const double epi_us = tile_bytes / (3e6 / 132);
  return 2.0 * epi_us >= mma_us ? 7 : 3;
}

template <int OP, bool BF16, bool SIG, int SW>
void launch_one(const CUtensorMap& a, const CUtensorMap& b, const TcParams& p, size_t smem) {
  smem_opt_in(tc_conv_kernel<OP, BF16, SIG, SW>, 227 * 1024);
  const int grid = std::min(p.num_tiles, num_sms());
  launch_pdl(tc_conv_kernel<OP, BF16, SIG, SW>, dim3((unsigned)grid), dim3(kThreadsFor<SW>), smem, state().stream, a, b, p);
}

template <int OP>
void launch(const CUtensorMap& a, const CUtensorMap& b, TcParams& p) {
  auto aligned = [](const void* q, uintptr_t a) { return (reinterpret_cast<uintptr_t>(q) & (a - 1)) == 0; };
  // wgrad writes dW 16 bytes per lane through the consumer warps' transpose areas wherever 4 consecutive output
  // features are one aligned float4 (not the x-mode scatter): its tiles carry few k-blocks, and 4-byte stores from the
  // accumulators held fc6's 302 MB dW to 0.9 TB/s on an H100.  The areas cost the ring one of its seven stages.
  if (OP == kWgrad) p.epi_bytes = (!p.x_mode && p.Cout % 4 == 0 && aligned(p.out, 16)) ? kWgradStageBytes : 0u;
  else p.epi_bytes = epi_bytes_for(p.BN);
  p.stages = pick_stages(p.bank_bytes, p.epi_bytes);
  const size_t smem = smem_bytes_for(p.stages, p.bank_bytes, p.epi_bytes);
  // the store warps move 4 rows (16 bytes of out / mask, 8 of out16) per access where the pointers allow it
  p.vec = aligned(p.out, 16) && aligned(p.mask, 16) && aligned(p.out16, 8) ? 1 : 0;
  const bool sig = p.act == kActLogistic || (p.mask && p.mask_act == kActLogistic);
  CNB_REQUIRE(OP != kWgrad || !sig, "tc_conv: wgrad has no activation epilogue");
  void (*run)(const CUtensorMap&, const CUtensorMap&, const TcParams&, size_t) = nullptr;
  // wgrad has no SIG instance, and stores from the MMA warps: its 3 store warps exit at once
  if constexpr (OP != kWgrad) {
    // k-blocks of a full tile (dgrad: every tap live), and the bytes its store warps move
    const int kcb = p.splits > 1 ? p.units_per_split : p.kc_blocks;
    const int kblocks = (OP == kFprop && p.x_mode) ? p.Cin * p.x_yblocks : p.taps * kcb;
    const double bytes = BM * p.BN * (4.0 + (p.out16 ? 2 : 0) + (p.mask ? 4 : 0) + (p.st != 0.f && p.splits == 1 ? 4 : 0));
    if (pick_store_warps(kblocks, bytes) == 7) {
      if (sig) run = p.bf16 ? launch_one<OP, true, true, 7> : launch_one<OP, false, true, 7>;
      else run = p.bf16 ? launch_one<OP, true, false, 7> : launch_one<OP, false, false, 7>;
    } else if (sig) {
      run = p.bf16 ? launch_one<OP, true, true, 3> : launch_one<OP, false, true, 3>;
    }
  }
  if (!run) run = p.bf16 ? launch_one<OP, true, false, 3> : launch_one<OP, false, false, 3>;
  run(a, b, p, smem);
  count_launch();
  CNB_LAUNCH_CHECK("tc_conv");
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
  p.xw = nullptr; p.bank_bytes = 0; p.epi_bytes = 0;
  p.a_merged = 0; p.b_merged = 0;
  p.untied = g.conv ? 0 : 1;
  p.bias = nullptr; p.act = 0; p.mask = nullptr; p.mask_act = 0; p.out16 = nullptr; p.vec = 0;
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
// `modules` > 0: untied, that many consecutive banks, and a trailing module dimension.
bool filter_map(CUtensorMap* m, const void* base, const Elem& e, long long cols, long long taps, long long K_c, int bn,
                bool merged, long long modules = 0) {
  const long long bank = cols * taps * K_c;
  const int extra = modules > 0 ? 1 : 0;
  if (merged) {
    const long long dims[5] = {e.chunk, K_c, cols / e.chunk, taps, modules};
    const long long str[4] = {cols * taps, e.chunk, cols, bank};
    const int box[5] = {e.chunk, e.bk, bn / e.chunk, 1, 1};
    return make_map(m, base, e, 4 + extra, dims, str, box);
  }
  const long long dims[4] = {cols, taps, K_c, modules};
  const long long str[3] = {cols, cols * taps, bank};
  const int box[4] = {e.chunk, 1, e.bk, 1};
  return make_map(m, base, e, 3 + extra, dims, str, box);
}
// floats in the filter tensor of a call: Cout x K, times the modules for untied filters
inline long long filter_elems(const ConvGeom& g) { return (long long)g.Cout * g.K * (g.conv ? 1 : g.modules); }

// fp32 operand of a call: the caller's tensor, its length in floats, and the element the kernel starts reading at
struct Operand { const float* src; long long n; long long off; };
// What the kernels of one call read: operands x and y, and `part_bytes` of partial sums at the start of the workspace.
// bf16: each operand's staged copy, or a copy converted into the workspace behind the partial sums (x first, then y);
// tf32: the fp32 buffers as they are.
struct CallBuffers { const void* x; const void* y; float* part; };
CallBuffers call_buffers(bool bf, size_t part_bytes, const Operand& x, const Operand& y) {
  if (!bf) return {x.src + x.off, y.src + y.off, part_bytes ? (float*)workspace(part_bytes) : nullptr};
  const __nv_bfloat16* sx = bf16_staged(x.src, x.n);
  const __nv_bfloat16* sy = bf16_staged(y.src, y.n);
  const size_t xb = sx ? 0 : align_up((size_t)x.n * 2), yb = sy ? 0 : align_up((size_t)y.n * 2);
  uint8_t* ws = part_bytes + xb + yb ? (uint8_t*)workspace(part_bytes + xb + yb) : nullptr;
  if (!sx) { to_bf16(x.src, (__nv_bfloat16*)(ws + part_bytes), x.n); sx = (const __nv_bfloat16*)(ws + part_bytes); }
  if (!sy) { to_bf16(y.src, (__nv_bfloat16*)(ws + part_bytes + xb), y.n); sy = (const __nv_bfloat16*)(ws + part_bytes + xb); }
  return {sx + x.off, sy + y.off, (float*)ws};
}

// ---- split-K for 1x1 / FC shapes: too few output tiles to fill the GPU, long K ------------------------
// out = st*out + so * sum_s part[s]  (+ bias[channel], act | times mask_act'(mask)): the fused epilogue moves here
__global__ void __launch_bounds__(256) reduce_split_kernel(const float4* __restrict__ part, float4* out, long long elems4,
                                                           long long stride4, int splits, float st, float so,
                                                           const float* __restrict__ bias, long long per_channel4, int act,
                                                           const float4* __restrict__ mask, int mask_act) {
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
    if (act) { s.x = act_apply(s.x, act); s.y = act_apply(s.y, act); s.z = act_apply(s.z, act); s.w = act_apply(s.w, act); }
    if (mask) {
      const float4 m = mask[i];
      s.x = act_deriv(s.x, m.x, mask_act); s.y = act_deriv(s.y, m.y, mask_act);
      s.z = act_deriv(s.z, m.z, mask_act); s.w = act_deriv(s.w, m.w, mask_act);
    }
    out[i] = s;
  }
}
void reduce_split(const float* part, float* out, long long elems, int splits, float st, float so, const float* bias,
                  long long per_channel, int act, const float* mask, int mask_act) {
  const long long e4 = elems / 4;
  const int grid = (int)std::min<long long>(std::max<long long>(ceil_div<long long>(e4, 256), 1), 8LL * num_sms());
  launch_pdl(reduce_split_kernel, dim3((unsigned)grid), dim3(256), 0, state().stream, (const float4*)part, (float4*)out, e4, e4, splits,
             st, so, bias, per_channel / 4, act, (const float4*)mask, mask_act);
  count_launch();
  CNB_LAUNCH_CHECK("reduce_split");
}
// The fprop-form GEMM of a launch (fprop, dgrad, dgrad in fprop form): `total_chunks` image chunks of rows, `cols`
// columns in n-tiles of p.BN, K in blocks of p.bk over `k_channels` channels.
void set_tiles(TcParams& p, int total_chunks, int cols, int k_channels) {
  p.kc_blocks = ceil_div(k_channels, p.bk);
  p.total_chunks = total_chunks;
  p.m_tiles = ceil_div(p.total_chunks, p.cpt);
  p.n_tiles = ceil_div(cols, p.BN);
  p.num_tiles = p.m_tiles * p.n_tiles;
  // MN-major B is staged in whole chunks (BN is a multiple of the chunk); x-mode streams A alone
  p.b_tx_bytes = p.x_mode ? 0u : (uint32_t)p.BN * 128;
}
// Split-K of a fprop/dgrad launch writing out_elems floats, where the caller's layout `allows` it: only 1x1 / FC shapes
// that leave most SMs idle split.  Returns the bytes of partial sums the launch needs (0: no split).
size_t split_k(TcParams& p, const ConvGeom& g, long long out_elems, bool allowed) {
  if (!allowed || p.x_mode || p.taps != 1 || g.frames != 1 || out_elems % 4 != 0) return 0;
  if (p.num_tiles * 2 > num_sms() || p.kc_blocks < 8) return 0;
  const int ks = std::max(std::min(num_sms() / p.num_tiles, p.kc_blocks / 4), 1);
  if (ks > 1) {
    p.units_per_split = ceil_div(p.kc_blocks, ks);
    p.splits = ceil_div(p.kc_blocks, p.units_per_split);
    p.part_stride = out_elems;
    p.num_tiles *= p.splits;
  }
  return p.splits > 1 ? align_up(sizeof(float) * out_elems * p.splits) : 0;
}

}  // namespace

// ---- fprop ---------------------------------------------------------------------------------------
// `bf` selects bf16 operands (CONVNET_B200_PRECISION=bf16): images and filters are first rounded to bf16 copies in
// library scratch (unless the caller keeps staged copies), then the bf16 flavour of the kernel runs wgmma on them.
static ConvOutcome tc_conv_up_impl(const ConvGeom& g, const float* images, const float* filters, float* targets, float st,
                                   float so, const Fuse& fuse, __nv_bfloat16* out16, bool bf) {
  const Elem e = elem_for(bf);
  if (g.N % 4 != 0 || g.Cout % 4 != 0) return {};                           // TMA stride alignment
  const bool x_mode = g.Cin < 8;                                            // tiny channel counts: taps take the K block
  if (x_mode && (g.kx > 8 || g.ky > 8)) return {};
  if (bf && (x_mode || g.N % 8 != 0 || g.Cout % 8 != 0 || !aligned16(images) || !aligned16(filters))) return {};
  if (!g.conv && (g.N % 128 != 0 || g.frames != 1 || x_mode)) return {};     // untied: each m-tile in one module
  const long long flt_n = filter_elems(g);
  // few GEMM rows (FC layers at training batch sizes): the call streams the weights once and is HBM-bound on them; a bf16
  // conversion pass inside the call would read them a second time, so such shapes take bf16 only when the caller keeps a
  // staged bf16 copy of the weights (the training host does: cnb_sgd_momentum refreshes it in the same pass that updates
  // them) — then the call streams HALF the bytes
  if (bf && (long long)g.N * g.modules * g.frames < 1024 && !bf16_staged(filters, flt_n)) return {};
  TcParams p; fill_common(p, g, e);
  p.BN = pick_bn(g.Cout, e.chunk);
  p.x_mode = x_mode ? 1 : 0;
  p.x_yblocks = ceil_div(g.ky, 4);
  if (x_mode) {
    // B is the n-tile's filter bank, resident beside the A ring and the staging tile: it must leave room for >= 3 A
    // stages, else the tile narrows (Cin 7, ky 8 at BN 128) — more n-tiles, the same single launch
    auto bank_bytes = [&](int bn) { return (uint32_t)g.Cin * p.x_yblocks * bn * 128; };
    while (p.BN > 32 && smem_bytes_for(3, bank_bytes(p.BN), epi_bytes_for(p.BN)) > kSmemBudget) p.BN = ceil_div(p.BN / 2, 32) * 32;
    p.bank_bytes = bank_bytes(p.BN);
    p.xw = filters;
  }
  const long long chunks = (long long)p.nb * g.modules * g.frames;
  if (chunks * 4 >= (1LL << 31)) return {};
  set_tiles(p, p.nbc * g.modules * g.frames, g.Cout, g.Cin);
  float* const out = targets + (long long)g.cout0 * g.modules * g.N;
  const float* const bias = fuse.bias ? fuse.bias + (long long)g.cout0 * (g.conv ? 1 : g.modules) : nullptr;
  const long long out_elems = (long long)g.Cout * g.modules * g.N;
  const size_t part_bytes = split_k(p, g, out_elems, g.conv);
  p.out = out;
  p.st = st; p.so = so;
  p.bias = bias; p.act = fuse.act;
  CUtensorMap ma, mb;
  const CallBuffers buf = call_buffers(bf, part_bytes, {images, g.img_total, (long long)g.cin0 * g.H * g.W * g.N},
                                       {filters, flt_n, 0});
  const long long taps = (long long)g.kx * g.ky;
  if (p.splits > 1) { p.out = buf.part; p.bias = nullptr; p.act = 0; }    // partial sums; the epilogue moves to reduce_split
  // bf16 twin of the output from the same registers: only when this launch writes the final value of EVERY element
  const bool emit = out16 != nullptr && p.splits == 1 && g.cout0 == 0 && g.Cout == g.CoutT;
  if (emit) p.out16 = out16;
  // dropout in the epilogue: the element index is the offset from the start of the WHOLE target tensor
  const bool drop = fuse.drop_scale != 0.f && p.splits == 1 && g.frames == 1 && g.cout0 == 0 && g.Cout == g.CoutT;
  if (drop) { p.drop_prob = fuse.drop_prob; p.drop_scale = fuse.drop_scale; p.drop_seed = fuse.drop_seed; }
  p.a_merged = (g.frames == 1 && g.N % 128 == 0) ? 1 : 0;
  p.b_merged = (g.Cout % e.chunk == 0) ? 1 : 0;
  // frames of a 3-D conv start in_frame_step floats apart and see Cin (= Cin3d*kt) channels
  if (x_mode) {
    const long long N = g.N;
    if (p.a_merged) {
      if (!merged_image_map(&ma, buf.x, e, g, g.W, g.H, g.Cin, true)) return {};
    } else {
      const long long adims[5] = {N, g.Cin, g.W, g.H, g.frames};
      const long long astr[4] = {N * g.W * g.H, N, N * g.W, g.in_frame_step};
      const int abox[5] = {32, 1, 8, 4, 1};                     // 8 x-taps x 4 filter rows of one channel
      if (!make_map(&ma, buf.x, e, 5, adims, astr, abox)) return {};
    }
    mb = ma;                                                    // no B map: the kernel reads the filters into its bank
  } else {
    if (p.a_merged) {
      if (!merged_image_map(&ma, buf.x, e, g, g.W, g.H, g.Cin, false)) return {};
    } else if (!image_map(&ma, buf.x, e, g, g.W, g.H, g.Cin, g.in_frame_step, true, e.bk)) return {};
    if (!filter_map(&mb, buf.y, e, g.Cout, taps, g.Cin, p.BN, p.b_merged, g.conv ? 0 : g.modules)) return {};
  }
  launch<kFprop>(ma, mb, p);
  if (p.splits > 1)
    reduce_split(buf.part, out, out_elems, p.splits, st, so, bias, (long long)g.modules * g.N, fuse.act, nullptr, 0);
  return {bf ? kPathTcBf16 : kPathTcTf32, emit, drop};
}
ConvOutcome tc_conv_up(const ConvGeom& g, const float* images, const float* filters, float* targets, float st, float so,
                       const Fuse& fuse, __nv_bfloat16* out16) {
  if (want_bf16()) {
    const ConvOutcome r = tc_conv_up_impl(g, images, filters, targets, st, so, fuse, out16, true);
    if (r.path != kPathNone) return r;
  }
  return tc_conv_up_impl(g, images, filters, targets, st, so, fuse, out16, false);
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
  if (!g.conv || !want_bf16() || !dgrad_as_fprop_eligible(g, derivs, filters, &banks)) return;
  dgrad_weights(filters, g, banks, true);
}

static ConvOutcome tc_conv_down_as_fprop(const ConvGeom& g, const float* derivs, const float* filters, float* targets,
                                         float so, const Fuse& fuse, __nv_bfloat16* out16) {
  DgradBanks banks;
  if (!dgrad_as_fprop_eligible(g, derivs, filters, &banks)) return {};
  const Elem e = elem_for(true);
  // the derivative as bf16 (staged by the producer, or converted here)
  const __nv_bfloat16* sd = bf16_staged(derivs, g.out_total);
  if (!sd) {
    __nv_bfloat16* tmp = (__nv_bfloat16*)workspace(align_up((size_t)g.out_total * 2));
    to_bf16(derivs, tmp, g.out_total);
    sd = tmp;
  }
  const __nv_bfloat16* bank = dgrad_weights(filters, g, banks, false);
  for (int i = 0; i < banks.count; i++) {
    const DgradPhase& P = banks.phase[i];
    TcParams p; fill_common(p, g, e);
    // the GEMM of this phase: rows = (image, phase pixel), K = (tap'', o), columns = input channels
    p.modX = P.Wp; p.modY = P.Hp; p.modules = P.Wp * P.Hp;
    p.W = g.modX; p.H = g.modY;                        // the tensor A is read from (the derivative grid)
    p.kx = P.ku; p.ky = P.kv; p.taps = P.ku * P.kv; p.sx = p.sy = 1; p.px = P.px; p.py = P.py;
    p.Cin = g.Cout; p.Cout = g.Cin;
    p.BN = pick_bn(g.Cin, 64);
    set_tiles(p, p.nbc * p.modules, g.Cin, g.Cout);
    p.out = targets; p.st = 0.f; p.so = so;
    p.mask = fuse.act_state; p.mask_act = fuse.state_act; p.out16 = out16;
    p.o_sx = g.sx; p.o_sy = g.sy; p.o_x0 = P.a; p.o_y0 = P.b; p.o_W = g.W; p.out_plane = (long long)g.W * g.H;
    p.a_merged = 1;
    p.b_merged = (g.Cin % 64 == 0) ? 1 : 0;
    CUtensorMap fa, fb;
    if (!merged_image_map(&fa, sd, e, g, g.modX, g.modY, g.Cout, false) ||
        !filter_map(&fb, bank + P.offset, e, g.Cin, p.taps, g.Cout, p.BN, p.b_merged)) {
      CNB_REQUIRE(i == 0, "dgrad-as-fprop: tensor map failed after the first phase");
      return {};
    }
    launch<kFprop>(fa, fb, p);
  }
  return {kPathTcBf16, out16 != nullptr, false};
}

// ---- dgrad ---------------------------------------------------------------------------------------
static ConvOutcome tc_conv_down_impl(const ConvGeom& g, const float* derivs, const float* filters, float* targets, float st,
                                     float so, const Fuse& fuse, __nv_bfloat16* out16, bool bf) {
  const Elem e = elem_for(bf);
  if (g.N % 4 != 0 || g.Cout % 4 != 0 || g.Cout < 8 || g.Cin < 8) return {};
  if (bf && (g.N % 8 != 0 || g.Cout % 8 != 0 || !aligned16(derivs) || !aligned16(filters))) return {};
  if (!g.conv && (g.N % 128 != 0 || g.frames != 1)) return {};             // untied: each m-tile on one input pixel
  const long long flt_n = filter_elems(g);
  if (bf && (long long)g.N * g.W * g.H < 1024 && !bf16_staged(filters, flt_n)) return {};   // see tc_conv_up_impl
  TcParams p; fill_common(p, g, e);
  p.BN = pick_bn(g.Cin, 16);
  const long long chunks = (long long)p.nb * g.W * g.H;
  if (chunks * 4 >= (1LL << 31) || g.kx > 32 || g.ky > 32) return {};
  set_tiles(p, p.nbc * g.W * g.H, g.Cin, g.Cout);
  p.so = so;
  const bool whole = (g.frames == 1 && g.cin0 == 0 && g.Cin == g.CinT);
  const long long out_elems = (long long)g.Cin * g.W * g.H * g.N;
  const size_t part_bytes = split_k(p, g, out_elems, whole && g.conv);
  CUtensorMap ma, mb;
  const CallBuffers buf = call_buffers(bf, part_bytes, {derivs, g.out_total, (long long)g.cout0 * g.modules * g.N},
                                       {filters, flt_n, 0});
  p.a_merged = (g.frames == 1 && g.N % 128 == 0) ? 1 : 0;
  if (p.a_merged) {
    if (!merged_image_map(&ma, buf.x, e, g, g.modX, g.modY, g.Cout, false)) return {};
  } else if (!image_map(&ma, buf.x, e, g, g.modX, g.modY, g.Cout, g.out_frame_step, true, e.bk)) return {};
  {                                                    // (o, tap, c[, module])
    const long long dims[4] = {g.Cout, (long long)g.kx * g.ky, g.Cin, g.modules};
    const long long str[3] = {g.Cout, (long long)g.Cout * g.kx * g.ky, (long long)g.Cout * g.K};
    const int box[4] = {e.chunk, 1, p.BN, 1};
    if (!make_map(&mb, buf.y, e, g.conv ? 3 : 4, dims, str, box)) return {};
  }
  float* out = targets + (long long)g.cin0 * g.H * g.W * g.N;
  bool emit = false;
  if (whole && p.splits > 1) {
    p.st = 0.f; p.out = buf.part; p.mask = nullptr;
    launch<kDgrad>(ma, mb, p);
    reduce_split(buf.part, out, out_elems, p.splits, st, so, nullptr, 1, 0, fuse.act_state, fuse.state_act);
  } else if (whole) {
    p.st = st; p.out = out; p.mask = fuse.act_state ? fuse.act_state + (long long)g.cin0 * g.H * g.W * g.N : nullptr;
    p.mask_act = fuse.state_act;
    p.out16 = out16;                                   // `whole`: every element gets its final value here
    emit = out16 != nullptr;
    launch<kDgrad>(ma, mb, p);
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
  return {bf ? kPathTcBf16 : kPathTcTf32, emit, false};
}
ConvOutcome tc_conv_down(const ConvGeom& g, const float* derivs, const float* filters, float* targets, float st, float so,
                         const Fuse& fuse, __nv_bfloat16* out16) {
  if (want_bf16()) {
    ConvOutcome r;
    if (st == 0.f) r = tc_conv_down_as_fprop(g, derivs, filters, targets, so, fuse, out16);
    if (r.path == kPathNone) r = tc_conv_down_impl(g, derivs, filters, targets, st, so, fuse, out16, true);
    if (r.path != kPathNone) return r;
  }
  return tc_conv_down_impl(g, derivs, filters, targets, st, so, fuse, out16, false);
}

// ---- wgrad ---------------------------------------------------------------------------------------
static ConvPath tc_conv_outp_impl(const ConvGeom& g, const float* images, const float* derivs, float* targets, float st,
                                  float so, bool bf) {
  const Elem e = elem_for(bf);
  if (g.N % 4 != 0 || g.Cout < 8) return kPathNone;
  const bool x_mode = g.Cin < 8;
  if (x_mode && (g.kx > 8 || g.ky > 8)) return kPathNone;
  if (bf && (x_mode || g.N % 8 != 0 || !aligned16(images) || !aligned16(derivs))) return kPathNone;
  if (!g.conv && (g.N % 128 != 0 || g.frames != 1 || x_mode)) return kPathNone;
  // few reduction rows (FC layers: K = batch): the call is bound by WRITING dW, and the operands a bf16 pass would convert
  // are tiny — such shapes take bf16 only in the whole-batch-tile layout the training step uses
  if (bf && (long long)g.N * g.modules * g.frames < 1024 && !(g.frames == 1 && g.N % 128 == 0 && g.Cin % 32 == 0)) return kPathNone;
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
  if (!g.conv) {                 // untied: one tile per (module, tap, o-tile, c-tile), stored straight into its module's block
    if (base_tiles * g.modules >= (1LL << 31)) return kPathNone;
    p.splits = g.modules; p.units_per_split = 1;
  }
  p.num_tiles = (int)(base_tiles * p.splits);
  p.st = st; p.so = so;
  CUtensorMap ma, mb;
  const bool partials = p.splits > 1 && g.conv;
  const size_t part_bytes = partials ? align_up(sizeof(float) * elems * p.splits) : 0;
  const CallBuffers buf = call_buffers(bf, part_bytes, {images, g.img_total, (long long)g.cin0 * g.H * g.W * g.N},
                                       {derivs, g.out_total, (long long)g.cout0 * g.modules * g.N});
  if (!image_map(&ma, buf.y, e, g, g.modX, g.modY, g.Cout, g.out_frame_step, false, BM)) return kPathNone;
  if (x_mode) {
    const long long N = g.N;
    const long long dims[5] = {N, g.W, g.H, g.Cin, g.frames};
    const long long str[4] = {N, N * g.W, N * g.W * g.H, g.in_frame_step};
    const int box[5] = {32, 8, g.ky, 1, 1};                   // 8 x-taps x ky rows of one channel: ky*8 GEMM columns
    if (!make_map(&mb, buf.x, e, 5, dims, str, box)) return kPathNone;
  } else if (!image_map(&mb, buf.x, e, g, g.W, g.H, g.Cin, g.in_frame_step, false, p.BN)) return kPathNone;
  p.out = partials ? buf.part : targets;
  launch<kWgrad>(ma, mb, p);
  if (partials) reduce_partials(buf.part, targets, elems, 1, p.splits, st, so);
  return bf ? kPathTcBf16 : kPathTcTf32;
}
ConvPath tc_conv_outp(const ConvGeom& g, const float* images, const float* derivs, float* targets, float st, float so) {
  if (want_bf16()) {
    const ConvPath path = tc_conv_outp_impl(g, images, derivs, targets, st, so, true);
    if (path != kPathNone) return path;
  }
  return tc_conv_outp_impl(g, images, derivs, targets, st, so, false);
}

}  // namespace cnb
