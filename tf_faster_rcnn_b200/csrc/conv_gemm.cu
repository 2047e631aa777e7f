// Dense stages of the Faster R-CNN TEST graph as ONE implicit-GEMM kernel for sm_90a:
//   slim.conv2d 3x3 / 1x1 (any stride), slim.fully_connected  (lib/nets/vgg16.py:26-60,
//   resnet_v1 bottlenecks, mobilenet pointwise, lib/nets/network.py:323-378)
//
// Math: D[M=pixels, N=cout] = sum over (filter tap, cin chunk) A_tap[M, k] * W[N, k]^T, fp32-grade through a two-term split
// of both operands and three tensor-core products per pair:  a*b ~= a_hi*b_hi + (a_lo*b_hi + a_hi*b_lo).
//   FRCNN_CONV_F16X3 (default): x_hi = RN_f16(x), x_lo = RN_f16((x - x_hi) * 2^11).  fp16 has tf32's 11-bit significand, so
//     every operand is carried to 2^-22 relative, with wgmma moving 16 k per instruction.  Range: the lo planes are pre-scaled
//     by 2^11 (the cross terms are folded back with one fma by 2^-11), weights are pre-scaled per layer by a power of two so
//     that max|w| sits in [2^13, 2^14) (undone exactly by `out_mult` in the epilogue), activations are converted WITHOUT
//     saturation: 2^-14 <= |x| < 65520 keeps 2^-22 relative (below 2^-14 the hi plane is subnormal and the loss grows to
//     2^-12 at 2^-24); |x| >= 65520, +-Inf and NaN become Inf/NaN and so make the output non-finite, never finite and wrong.
//   FRCNN_CONV_TF32X3: the same split in tf32 (hi = RN_tf32(x), lo = RN_tf32(x - hi), no scaling), 8 k per instruction;
//     2^-22 relative from 2^-115 up to the tf32 overflow; non-finite inputs give non-finite outputs.
//   FRCNN_CONV_F16X1 (throughput mode, NOT fp32-grade): the hi planes only, one product per pair.
//
// Data movement: activations stay plain NHWC fp32 in HBM.  For filter tap (r,s) the A operand of a tile of tn x th x tw
// output pixels is ONE 4-D TMA box {32 ch, tw, th, tn} of the input at offset (w0*stride+s-pad_l, h0*stride+r-pad_t):
// out-of-bounds rows/cols are zero-filled by TMA, which IS the convolution's zero padding -- no im2col buffer ever exists.
// Weights are pre-split (hi/lo planes), K-major, 128-byte rows, SWIZZLE_128B in shared memory: the wgmma B operand.
//
// Operand split in registers: the consumer warpgroups read the raw fp32 A tile from shared memory straight into the wgmma
// A-fragment layout (un-swizzling on the fly), split it into hi / lo fragments, and issue wgmma with A from registers.  No
// split copy of A is ever written back to shared memory.
//
// Accumulation is two-level: the tensor core adds into its fp32 accumulator without round-to-nearest, so its error grows
// with the number of products summed.  Each k-block's hi*hi products (4 instructions) go into a fresh register partial that
// is added into the fp32 accumulator with round-to-nearest adds; the cross terms of the same k-block are then summed into the
// same partial registers and folded in with one fma.  Registers hold 2 x BN/2 fp32 per thread (partial + accumulator).
//
// PERSISTENT: grid = min(#work units, #SMs); producer and consumers walk the same sequence of work units (output tile x
// split-K range); the ring's slots and barrier phases run on across units.
// Roles (384 threads, 1 CTA/SM):
//   warps 0-3, 4-7  consumer warpgroup g owns output rows [64g, 64g + 64) of the 128-row tile and all BN columns:
//                   wait full[s]; A rows -> hi/lo fragments; wgmma hi*hi -> partial -> acc; wgmma cross -> partial -> acc;
//                   arrive empty[s]; per unit: epilogue straight from the accumulator registers
//   warp 8          TMA producer: wait empty[s]; A box(es) + B hi (+ B lo) -> full[s] (tx); warps 9-11 idle (they complete
//                   the warpgroup whose registers setmaxnreg hands to the consumers)
// The two warpgroups share the tensor core: while one promotes its partial or converts the next A tile, the other's wgmmas run.
#include <cuda_fp16.h>
#include "common.cuh"
#include "../../include/frcnn_b200.h"
#include <stdlib.h>
#include <string.h>

namespace frcnn {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 32;                          // fp32 channels of one A box row: 128 B = one swizzle row
constexpr int A_TILE_BYTES = BLOCK_M * BLOCK_K * 4;  // 16 KiB
constexpr int NUM_CONSUMERS = 256;                   // two warpgroups
constexpr int NUM_THREADS = NUM_CONSUMERS + 128;     // + the producer warpgroup (one thread issues; setmaxnreg needs whole warpgroups)
constexpr int REGS_PRODUCER = 40, REGS_CONSUMER = 232;   // 128 x 40 + 256 x 232 <= 64K: partial + accumulator + A fragments, no spills
constexpr int STAGES = 3;                            // depth of the (A, B) shared-memory ring

struct ConvKernelParams {
  float* out;
  const float* residual;
  const float* scale;   // [n_tiles*BN] plan-owned: (scale or 1) * out_mult (out_mult = 2^-wexp undoes the f16 weight scaling, exact)
  const float* shift;   // [n_tiles*BN] plan-owned: shift or 0
  int cout, ho, wo, nimg;
  int tn, th, tw;
  int tiles_h, tiles_w;
  int kh, kw, cin, stride, pad_t, pad_l;
  int act;
  int a_box_bytes;
  // Work units.  Tiles t = mt + m_tiles*nblk.  Units [0, n_full) are whole tiles (direct epilogue).  The remaining
  // `n_tail` tiles -- the ragged last round of the persistent loop, or every tile of a layer too small to fill the GPU --
  // are each split over `splits` units along K: unit n_full + v -> tile n_full + v / splits, split v % splits, which writes
  // its raw partial tile to ws[(v / splits)][v % splits][128][BN]; tail_reduce_kernel sums them in index order and
  // runs the epilogue.
  int kb_per_split;
  int m_tiles, n_tiles, total_units, n_full, splits;
  int raster_n;       // 1: consecutive tile indices walk the N-blocks of one M-tile (activations streamed once), 0: M-tiles first
  float* ws;
  long long* trace;   // debug: clock64() stamps of CTA 0's pipeline hand-offs; normally NULL
  int num_kb_total;   // k-blocks of the whole K loop (64 channels for the f16 modes, 32 for tf32)
  int cin2;           // channels of the second A source (tmA2; pointwise layers only), 0 = none
  // Mean epilogue (pointwise layers only, never split): tile mt's activated rows are summed per group of mean_hw pixels
  // into mean_ws[mt][s][n_tiles*BN] (s = group - first group of the tile, s < mean_segs); mean_finish_kernel adds the
  // partials of each group in tile order and divides by mean_hw into mean_out [pixels / mean_hw][cout].
  float* mean_out;
  float* mean_ws;
  int mean_hw, mean_segs, mean_ld;   // mean_ld = n_tiles * BN
};

// clock64 stamps of CTA 0's pipeline hand-offs: compiled in only in the development build (libfrcnn_b200_wd.so, -DFRCNN_WATCHDOG).
#ifdef FRCNN_WATCHDOG
#define FRCNN_TRACE(slot, kbv)                                                              \
  do {                                                                                      \
    if (p.trace && blockIdx.x == 0 && (kbv) < 64) p.trace[(kbv) * 8 + (slot)] = clock64(); \
  } while (0)
#else
#define FRCNN_TRACE(slot, kbv) do { } while (0)
#endif

template <int MODE> struct KTraits {
  static constexpr bool TF32 = MODE == FRCNN_CONV_TF32X3;
  static constexpr bool X1 = MODE == FRCNN_CONV_F16X1;
  static constexpr int BOXES = TF32 ? 1 : 2;               // 32-channel A boxes per k-block
  static constexpr int A_BYTES = BOXES * A_TILE_BYTES;
  static constexpr float LO_SCALE = TF32 ? 1.f : 0.00048828125f;   // undoes the 2^11 of the fp16 lo planes
};
template <int BN> constexpr int b_plane_bytes() { return BN * 128; }      // [BN][128 B]: 64 fp16 or 32 fp32 per row
template <int BN, int MODE> constexpr int stage_bytes() { return KTraits<MODE>::A_BYTES + 2 * b_plane_bytes<BN>(); }
template <int BN, int MODE> constexpr int smem_bytes() {
  return STAGES * stage_bytes<BN, MODE>() + 1024 /*align slack*/ + 64 /*barriers*/;
}
// mean epilogue: one 64-column slice of the 128-row tile at a time, rows padded against bank conflicts
constexpr int MEAN_COLS = 64, MEAN_LD = MEAN_COLS + 2;
constexpr int MEAN_SMEM = BLOCK_M * MEAN_LD * 4;
static_assert(smem_bytes<128, FRCNN_CONV_F16X3>() + MEAN_SMEM <= 227 * 1024, "ring exceeds the sm_90 shared-memory limit per block");

// Work unit u (persistent loop: u = blockIdx.x, += gridDim.x) -> output tile + split-K range.
struct Unit {
  int w0, h0, n0, nblk, z, kb0, num_kb, slot;   // slot >= 0: tail tile index (raw partial output), -1: whole tile
};
__device__ __forceinline__ Unit decode_unit(const ConvKernelParams& p, int u, int num_kb_total) {
  Unit t;
  int tile;
  if (u < p.n_full) { tile = u; t.z = 0; t.slot = -1; }
  else { const int v = u - p.n_full; t.slot = v / p.splits; t.z = v - t.slot * p.splits; tile = p.n_full + t.slot; }
  // raster order of the tile index: the operand with the larger footprint is walked ONCE, the other one stays L2 resident
  // (decide_geometry sets raster_n)
  int mt;
  if (p.raster_n) { t.nblk = tile % p.n_tiles; mt = tile / p.n_tiles; }
  else { mt = tile % p.m_tiles; t.nblk = tile / p.m_tiles; }
  const int tile_w = mt % p.tiles_w;
  const int tile_h = (mt / p.tiles_w) % p.tiles_h;
  const int tile_n = mt / (p.tiles_w * p.tiles_h);
  t.w0 = tile_w * p.tw; t.h0 = tile_h * p.th; t.n0 = tile_n * p.tn;
  if (t.slot < 0) { t.kb0 = 0; t.num_kb = num_kb_total; }
  else { t.kb0 = t.z * p.kb_per_split; t.num_kb = min(p.kb_per_split, num_kb_total - t.kb0); }
  return t;
}

// ---------------- tile epilogue, straight from the wgmma accumulator registers ----------------
// Accumulator layout (m64nBN, fp32): acc[4j + 0,1] = row r0, columns 8j + 2*q4 + {0,1}; acc[4j + 2,3] = row r0 + 8, same
// columns (r0 = 64*warpgroup + 16*warp + lane/4, q4 = lane % 4).  A warp's store of one j writes 8 rows x 32 contiguous bytes:
// whole 32-byte sectors, no staging through shared memory needed.
template <int ACT>
__device__ __forceinline__ float apply_act(float a) {
  if (ACT == FRCNN_ACT_RELU) return fmaxf(a, 0.f);
  if (ACT == FRCNN_ACT_RELU6) return fminf(fmaxf(a, 0.f), 6.f);
  return a;
}

// y = act(v*scale + shift (+ res)) with one rounding per operation (the oracle's order: tf.nn.batch_normalization /
// bias_add, then the shortcut add, then the activation)
template <bool RES, int ACT>
__device__ __forceinline__ float2 finish2(const float2 v, const float2 sc, const float2 sh, const float2 r) {
  float2 y;
  y.x = __fadd_rn(__fmul_rn(v.x, sc.x), sh.x); y.y = __fadd_rn(__fmul_rn(v.y, sc.y), sh.y);
  if (RES) { y.x = __fadd_rn(y.x, r.x); y.y = __fadd_rn(y.y, r.y); }
  y.x = apply_act<ACT>(y.x); y.y = apply_act<ACT>(y.y);
  return y;
}

// whole tile, cout % 4 == 0: float2 loads / stores (scale / shift are padded to the tile grid, so their loads need no bound).
// The loads of a chunk of EPI_CHUNK column groups are all issued before the first of its stores: the per-group loop would
// otherwise wait one full memory round trip (HBM for the residual) per 8 columns, BN / 8 times per tile, with the tensor
// core idle.  Chunks bound the registers the in-flight loads hold (the partial registers are free here).
constexpr int EPI_CHUNK = 8;
template <int BN, bool RES, int ACT>
__device__ __forceinline__ void epilogue_vec(const ConvKernelParams& p, const float (&acc)[BN / 2], const int cbase,
                                             const int pix0, const int pix1) {
  const int cout = p.cout;
  constexpr int NJ = BN / 8;
  constexpr int CH = NJ < EPI_CHUNK ? NJ : EPI_CHUNK;
  static_assert(NJ % CH == 0, "chunking");
  const float* const res0 = RES ? p.residual + (size_t)(pix0 >= 0 ? pix0 : 0) * cout : nullptr;
  const float* const res1 = RES ? p.residual + (size_t)(pix1 >= 0 ? pix1 : 0) * cout : nullptr;
#pragma unroll
  for (int j0 = 0; j0 < NJ; j0 += CH) {
    if (cbase + 8 * j0 >= cout) break;
    float2 sc[CH], sh[CH], r0[CH], r1[CH];
#pragma unroll
    for (int jj = 0; jj < CH; ++jj) {
      const int c = cbase + 8 * (j0 + jj);
      sc[jj] = ld_nc_f2_pinned(p.scale + c);
      sh[jj] = ld_nc_f2_pinned(p.shift + c);
      if (RES) {
        r0[jj] = ld_nc_f2_pinned_if(res0 + c, pix0 >= 0 && c < cout);
        r1[jj] = ld_nc_f2_pinned_if(res1 + c, pix1 >= 0 && c < cout);
      } else {
        r0[jj] = r1[jj] = sc[jj];
      }
    }
#pragma unroll
    for (int jj = 0; jj < CH; ++jj) {
      const int j = j0 + jj;
      const int c = cbase + 8 * j;
      if (c >= cout) break;
      if (pix0 >= 0)
        *reinterpret_cast<float2*>(p.out + (size_t)pix0 * cout + c) =
            finish2<RES, ACT>(make_float2(acc[4 * j], acc[4 * j + 1]), sc[jj], sh[jj], r0[jj]);
      if (pix1 >= 0)
        *reinterpret_cast<float2*>(p.out + (size_t)pix1 * cout + c) =
            finish2<RES, ACT>(make_float2(acc[4 * j + 2], acc[4 * j + 3]), sc[jj], sh[jj], r1[jj]);
    }
  }
}

// any cout (scalar tails): same arithmetic, run-time flags
template <int BN>
__device__ __forceinline__ void epilogue_generic(const ConvKernelParams& p, const float (&acc)[BN / 2], const int cbase,
                                                 const int pix0, const int pix1) {
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int c = cbase + 8 * j + (e & 1);
      const int pix = e < 2 ? pix0 : pix1;
      if (pix < 0 || c >= p.cout) continue;
      float a = __fadd_rn(__fmul_rn(acc[4 * j + e], p.scale[c]), p.shift[c]);
      if (p.residual) a = __fadd_rn(a, __ldg(p.residual + (size_t)pix * p.cout + c));
      if (p.act == FRCNN_ACT_RELU) a = fmaxf(a, 0.f);
      else if (p.act == FRCNN_ACT_RELU6) a = fminf(fmaxf(a, 0.f), 6.f);
      p.out[(size_t)pix * p.cout + c] = a;
    }
  }
}

template <int BN, bool RES>
__device__ __forceinline__ void epilogue_dispatch(const ConvKernelParams& p, const float (&acc)[BN / 2], const int cbase,
                                                  const int pix0, const int pix1) {
  if (p.act == FRCNN_ACT_RELU) epilogue_vec<BN, RES, FRCNN_ACT_RELU>(p, acc, cbase, pix0, pix1);
  else if (p.act == FRCNN_ACT_RELU6) epilogue_vec<BN, RES, FRCNN_ACT_RELU6>(p, acc, cbase, pix0, pix1);
  else epilogue_vec<BN, RES, FRCNN_ACT_NONE>(p, acc, cbase, pix0, pix1);
}

// NHWC pixel index of tile row `row`, or -1 when the row lies outside the output
__device__ __forceinline__ int tile_pixel(const ConvKernelParams& p, const Unit& t, int row) {
  const int rows_img = p.th * p.tw;
  const int dn = row / rows_img, rem = row % rows_img;
  const int n = t.n0 + dn, h = t.h0 + rem / p.tw, w = t.w0 + rem % p.tw;
  const bool valid = row < p.tn * rows_img && n < p.nimg && h < p.ho && w < p.wo;
  return valid ? (int)(((long long)n * p.ho + h) * p.wo + w) : -1;
}

__device__ __forceinline__ void consumer_bar() { asm volatile("bar.sync 1, %0;" :: "n"(NUM_CONSUMERS) : "memory"); }

// Mean epilogue (flattened pointwise layer: tile row r is pixel w0 + r; cout % 4 == 0).  Per 64-column slice: both
// warpgroups put their activated values into `buf` (the arithmetic of finish2; a slice's loads are all issued together, as
// in epilogue_vec), then thread (slot, col) sums the rows of groups slot, slot + 4, ... of the tile and stores the tile
// partial.  Four interleaved partial sums per group keep the shared-memory loads in flight; the order is fixed
// (deterministic, no atomics) and a group of hw values still takes at most hw - 1 rounded adds over the tiles it spans.
template <int BN>
__device__ __forceinline__ void epilogue_mean(const ConvKernelParams& p, const Unit& t, const float (&acc)[BN / 2], int r0, int q4,
                                              float* buf) {
  constexpr int CH = MEAN_COLS / 8;
  const int nrows = min(p.tw, p.wo - t.w0);
  const int hw = p.mean_hw;
  const int g0 = t.w0 / hw, nseg = (t.w0 + nrows - 1) / hw - g0 + 1;
  const int mt = t.w0 / p.tw;
  const size_t ld = (size_t)p.mean_ld;
  const int tid = threadIdx.x, col = tid % MEAN_COLS;
  const bool v0 = r0 < nrows, v1 = r0 + 8 < nrows;
  const float* const res0 = p.residual ? p.residual + (size_t)(t.w0 + (v0 ? r0 : 0)) * p.cout : nullptr;
  const float* const res1 = p.residual ? p.residual + (size_t)(t.w0 + (v1 ? r0 + 8 : 0)) * p.cout : nullptr;
#pragma unroll
  for (int cc = 0; cc < BN; cc += MEAN_COLS) {
    float2 sc[CH], sh[CH], ra[CH], rb[CH];
#pragma unroll
    for (int jj = 0; jj < CH; ++jj) {
      const int c = t.nblk * BN + cc + 8 * jj + 2 * q4;
      sc[jj] = ld_nc_f2_pinned(p.scale + c);          // padded to the tile grid
      sh[jj] = ld_nc_f2_pinned(p.shift + c);
      ra[jj] = ld_nc_f2_pinned_if(res0 + c, res0 && v0 && c < p.cout);
      rb[jj] = ld_nc_f2_pinned_if(res1 + c, res1 && v1 && c < p.cout);
    }
    consumer_bar();                                     // the previous slice's sums have read buf
#pragma unroll
    for (int jj = 0; jj < CH; ++jj) {
      const int j = cc / 8 + jj;
      float2 y0 = make_float2(__fadd_rn(__fmul_rn(acc[4 * j], sc[jj].x), sh[jj].x), __fadd_rn(__fmul_rn(acc[4 * j + 1], sc[jj].y), sh[jj].y));
      float2 y1 = make_float2(__fadd_rn(__fmul_rn(acc[4 * j + 2], sc[jj].x), sh[jj].x), __fadd_rn(__fmul_rn(acc[4 * j + 3], sc[jj].y), sh[jj].y));
      if (p.residual) {
        y0.x = __fadd_rn(y0.x, ra[jj].x); y0.y = __fadd_rn(y0.y, ra[jj].y);
        y1.x = __fadd_rn(y1.x, rb[jj].x); y1.y = __fadd_rn(y1.y, rb[jj].y);
      }
      if (p.act != FRCNN_ACT_NONE) {
        y0.x = fmaxf(y0.x, 0.f); y0.y = fmaxf(y0.y, 0.f); y1.x = fmaxf(y1.x, 0.f); y1.y = fmaxf(y1.y, 0.f);
        if (p.act == FRCNN_ACT_RELU6) { y0.x = fminf(y0.x, 6.f); y0.y = fminf(y0.y, 6.f); y1.x = fminf(y1.x, 6.f); y1.y = fminf(y1.y, 6.f); }
      }
      *reinterpret_cast<float2*>(buf + r0 * MEAN_LD + 8 * jj + 2 * q4) = y0;
      *reinterpret_cast<float2*>(buf + (r0 + 8) * MEAN_LD + 8 * jj + 2 * q4) = y1;
    }
    consumer_bar();
    for (int s = tid / MEAN_COLS; s < nseg; s += NUM_CONSUMERS / MEAN_COLS) {
      const int g = g0 + s;
      const int rs = max(g * hw - t.w0, 0), re = min((g + 1) * hw - t.w0, nrows);
      const float* b = buf + col;
      float a0 = b[rs * MEAN_LD], a1 = 0.f, a2 = 0.f, a3 = 0.f;
      int r = rs + 1;
      for (; r + 3 < re; r += 4) {
        a1 = __fadd_rn(a1, b[r * MEAN_LD]); a2 = __fadd_rn(a2, b[(r + 1) * MEAN_LD]);
        a3 = __fadd_rn(a3, b[(r + 2) * MEAN_LD]); a0 = __fadd_rn(a0, b[(r + 3) * MEAN_LD]);
      }
      for (; r < re; ++r) a1 = __fadd_rn(a1, b[r * MEAN_LD]);
      p.mean_ws[((size_t)mt * p.mean_segs + s) * ld + (size_t)t.nblk * BN + cc + col] = __fadd_rn(__fadd_rn(a0, a1), __fadd_rn(a2, a3));
    }
  }
}

template <int BN>
__device__ __forceinline__ void epilogue_tile(const ConvKernelParams& p, const Unit& t, const float (&acc)[BN / 2], int r0, int q4,
                                              float* mean_buf) {
  if (p.mean_out) {                                     // mean layers are never split (decide_geometry)
    epilogue_mean<BN>(p, t, acc, r0, q4, mean_buf);
    return;
  }
  if (t.slot >= 0) {
    // split tile: raw partial sums into the tile-local [128][BN] workspace (row-major); tail_reduce_kernel runs the epilogue
    float* const w = p.ws + ((size_t)t.slot * p.splits + t.z) * (size_t)(BLOCK_M * BN) + 2 * q4;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      __stcg(reinterpret_cast<float2*>(w + (size_t)r0 * BN + 8 * j), make_float2(acc[4 * j], acc[4 * j + 1]));
      __stcg(reinterpret_cast<float2*>(w + (size_t)(r0 + 8) * BN + 8 * j), make_float2(acc[4 * j + 2], acc[4 * j + 3]));
    }
    return;
  }
  const int pix0 = tile_pixel(p, t, r0), pix1 = tile_pixel(p, t, r0 + 8);
  const int cbase = t.nblk * BN + 2 * q4;
  if ((p.cout & 3) != 0) {
    // scalar-tail layers are never split (decide_geometry) -- generic path
    epilogue_generic<BN>(p, acc, cbase, pix0, pix1);
    return;
  }
  if (p.residual) epilogue_dispatch<BN, true>(p, acc, cbase, pix0, pix1);
  else epilogue_dispatch<BN, false>(p, acc, cbase, pix0, pix1);
}

template <int BN, int MODE>
__device__ __forceinline__ void wgmma_rs(float (&d)[BN / 2], const uint32_t (&a)[4], uint64_t b_desc, uint32_t scale_d) {
  if (KTraits<MODE>::TF32) wgmma_tf32_rs<BN>(d, a, b_desc, scale_d);
  else wgmma_f16_rs<BN>(d, a, b_desc, scale_d);
}

template <int BN, int MODE>
__global__ void __launch_bounds__(NUM_THREADS, 1)
conv_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmA2,
                 const __grid_constant__ CUtensorMap tmBhi, const __grid_constant__ CUtensorMap tmBlo, const ConvKernelParams p) {
  using T = KTraits<MODE>;
  constexpr int kStage = stage_bytes<BN, MODE>();
  constexpr int kPlane = b_plane_bytes<BN>();
  constexpr int NACC = BN / 2;
  static_assert(BN == 64 || BN == 128, "block_n");

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  // stage s: [A box 0 (| A box 1)] [B hi] [B lo], every part 1024-B aligned (SWIZZLE_128B atoms)
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + STAGES * kStage);   // A and B bytes of the stage landed (tx)
  uint64_t* empty = full + STAGES;                                        // both warpgroups are done with the stage
  // full + 8 (64 B of barriers on): MEAN_SMEM bytes for the mean epilogue, allocated only when it is on

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int num_kb_total = p.num_kb_total;

  if (threadIdx.x == NUM_CONSUMERS) {
    tma_prefetch_desc(&tmA); tma_prefetch_desc(&tmBhi); tma_prefetch_desc(&tmBlo);
    if (p.cin2) tma_prefetch_desc(&tmA2);
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], NUM_CONSUMERS); }
    mbar_fence_init();
  }
  __syncthreads();
  // Programmatic dependent launch: the next kernel of the stream may begin its prologue now; we ourselves touch the previous
  // kernel's outputs only behind pdl_wait() (A loads, residual loads, stores).
  pdl_launch_dependents();
  pdl_wait();

  if (warp >= NUM_CONSUMERS / 32) {
    // ---------------- TMA producer ----------------
    reg_dec<REGS_PRODUCER>();
    if (warp == NUM_CONSUMERS / 32 && lane == 0) {
      const int cchunks = p.cin / BLOCK_K;                        // 32-channel chunks per filter tap
      const int total1 = p.kh * p.kw * cchunks;                   // ... of the first source; then cin2 / 32 of the second
      const int cchunks2 = p.cin2 / BLOCK_K;
      const uint32_t tx = (uint32_t)(T::BOXES * p.a_box_bytes + (T::X1 ? 1 : 2) * kPlane);
      int s = 0; uint32_t ph = 0, kbt = 0;
      for (int u = blockIdx.x; u < p.total_units; u += gridDim.x) {
        const Unit t = decode_unit(p, u, num_kb_total);
#pragma unroll 1
        for (int kb = 0; kb < t.num_kb; ++kb, ++kbt) {
          MBAR_WAIT(&empty[s], ph ^ 1u, 4, kbt);                // both warpgroups have released the stage
          uint8_t* st = smem + s * kStage;
          mbar_expect_tx(&full[s], tx);
#pragma unroll
          for (int i = 0; i < T::BOXES; ++i) {
            const int g32 = (t.kb0 + kb) * T::BOXES + i;           // global 32-channel block -> (filter tap, channel chunk)
            int tap = g32 / cchunks, kc = g32 - tap * cchunks;
            const CUtensorMap* ma = &tmA;
            if (g32 >= total1) {                                  // second source (pointwise: one tap), or the odd tail: a box
              tap = 0;                                            // past the last channel is zero-filled by TMA
              if (cchunks2) { ma = &tmA2; kc = min(g32 - total1, cchunks2); }
              else kc = cchunks;
            }
            const int r = tap / p.kw, sx = tap - r * p.kw;
            tma_load_4d(st + i * A_TILE_BYTES, ma, &full[s], kc * BLOCK_K, t.w0 * p.stride + sx - p.pad_l,
                        t.h0 * p.stride + r - p.pad_t, t.n0);
          }
          const int kcoord = (t.kb0 + kb) * T::BOXES * BLOCK_K;   // K axis of the packed weights = (tap, cin) flattened; past the end: zeros
          tma_load_2d(st + T::A_BYTES, &tmBhi, &full[s], kcoord, t.nblk * BN);
          if (!T::X1) tma_load_2d(st + T::A_BYTES + kPlane, &tmBlo, &full[s], kcoord, t.nblk * BN);
          FRCNN_TRACE(0, kbt);
          if (++s == STAGES) { s = 0; ph ^= 1u; }
        }
      }
    }
    return;
  }

  // ---------------- consumers: split A, wgmma, promote, epilogue ----------------
  reg_inc<REGS_CONSUMER>();
  const int wg = warp >> 2;
  const int q4 = lane & 3;
  const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);       // this thread's tile rows: r0 and r0 + 8
  const uint32_t swz = (uint32_t)(lane >> 2);                   // == r0 & 7 == (r0 + 8) & 7
  // byte offset, inside a stage, of this thread's A element (row r0, fragment column (j, h)) for k-slice j, half h; row r0 + 8
  // is 1024 bytes further.  SWIZZLE_128B: 16-byte chunk c of row r sits at chunk (c ^ (r & 7)).
  uint32_t aoff[4][2];
#pragma unroll
  for (int j = 0; j < 4; ++j)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int ch = T::TF32 ? j * 8 + h * 4 + q4 : (j & 1) * 16 + h * 8 + 2 * q4;
      const int box = T::TF32 ? 0 : j >> 1;
      aoff[j][h] = (uint32_t)(box * A_TILE_BYTES + r0 * 128) + ((((uint32_t)ch >> 2) ^ swz) << 4) + (((uint32_t)ch & 3u) << 2);
    }
  const uint32_t smem0 = smem_u32(smem);
  int s = 0; uint32_t ph = 0, kbt = 0;
  for (int u = blockIdx.x; u < p.total_units; u += gridDim.x) {
    const Unit t = decode_unit(p, u, num_kb_total);
    float acc[NACC], part[NACC];
#pragma unroll
    for (int i = 0; i < NACC; ++i) { acc[i] = 0.f; part[i] = 0.f; }
#pragma unroll 1
    for (int kb = 0; kb < t.num_kb; ++kb, ++kbt) {
      MBAR_WAIT(&full[s], ph, 1, kbt);
      if (threadIdx.x == 0) FRCNN_TRACE(1, kbt);
      const uint32_t sa = smem0 + (uint32_t)(s * kStage);
      // A fragments of the 4 k-slices: {(r0, k), (r0+8, k), (r0, k+off), (r0+8, k+off)} per slice, as hi and lo
      uint32_t ahi[4][4], alo[4][4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
#pragma unroll
        for (int f = 0; f < 4; ++f) {
          const uint32_t addr = sa + aoff[j][f >> 1] + ((f & 1) ? 1024u : 0u);
          if (T::TF32) {
            float x;
            asm volatile("ld.shared.f32 %0, [%1];" : "=f"(x) : "r"(addr));
            // hi through cvt.rna: to_tf32_fast carries a NaN's high mantissa bits into the sign (0x7fffffff, the NaN the
            // device's own arithmetic produces, becomes -0.0) and the NaN would vanish.  lo only needs the finite case: a
            // non-finite x already makes hi non-finite.
            const float hi = to_tf32(x);
            ahi[j][f] = __float_as_uint(hi);
            alo[j][f] = __float_as_uint(to_tf32_fast(__fsub_rn(x, hi)));
          } else {
            float2 x;
            asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(x.x), "=f"(x.y) : "r"(addr));
            const uint32_t h = pack_f16x2_rn(x.x, x.y);
            const float2 fh = __half22float2(*reinterpret_cast<const __half2*>(&h));
            ahi[j][f] = h;
            alo[j][f] = T::X1 ? 0u : pack_f16x2_rn(__fmul_rn(__fsub_rn(x.x, fh.x), 2048.f), __fmul_rn(__fsub_rn(x.y, fh.y), 2048.f));
          }
        }
      }
      const uint64_t bhi = wgmma_sw128_desc(sa + (uint32_t)T::A_BYTES);
      const uint64_t blo = wgmma_sw128_desc(sa + (uint32_t)(T::A_BYTES + kPlane));
      // hi * hi: a fresh partial of this k-block, then one round-to-nearest add per element
#pragma unroll
      for (int i = 0; i < NACC; ++i) reg_fence(part[i]);
      wgmma_fence();
#pragma unroll
      for (int j = 0; j < 4; ++j) wgmma_rs<BN, MODE>(part, ahi[j], bhi + 2u * j, j > 0 ? 1u : 0u);   // +32 B per k-slice
      wgmma_commit();
      wgmma_wait_all();
#pragma unroll
      for (int i = 0; i < NACC; ++i) { reg_fence(part[i]); acc[i] = __fadd_rn(acc[i], part[i]); }
      if (!T::X1) {
        // cross terms a_lo*b_hi + a_hi*b_lo into the same partial registers, folded in with one fma each
        wgmma_fence();
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          wgmma_rs<BN, MODE>(part, alo[j], bhi + 2u * j, j > 0 ? 1u : 0u);
          wgmma_rs<BN, MODE>(part, ahi[j], blo + 2u * j, 1u);
        }
        wgmma_commit();
        wgmma_wait_all();
#pragma unroll
        for (int i = 0; i < NACC; ++i) { reg_fence(part[i]); acc[i] = __fmaf_rn(part[i], T::LO_SCALE, acc[i]); }
      }
      mbar_arrive(&empty[s]);                                   // A is in registers, the wgmmas reading B have completed
      if (threadIdx.x == 0) FRCNN_TRACE(2, kbt);
      if (++s == STAGES) { s = 0; ph ^= 1u; }
    }
    epilogue_tile<BN>(p, t, acc, r0, q4, reinterpret_cast<float*>(full + 8));
  }
}

// Second pass for split tiles: out = act((sum_z ws[slot][z]) * scale + shift (+ residual)), z summed in index order
// (deterministic).  One block per (tail tile, group of 256/(BN/4) rows); thread = (row, 4 channels).
template <int BN>
__global__ void __launch_bounds__(256)
tail_reduce_kernel(const ConvKernelParams p) {
  pdl_launch_dependents();
  pdl_wait();
  constexpr int RPB = 256 / (BN / 4);                 // rows per block: one (row, 4-channel group) per thread
  constexpr int GROUPS = BLOCK_M / RPB;
  const int slot = blockIdx.x / GROUPS, rgroup = blockIdx.x % GROUPS;
  const int tile = p.n_full + slot;
  const int mt = p.raster_n ? tile / p.n_tiles : tile % p.m_tiles, nblk = p.raster_n ? tile % p.n_tiles : tile / p.m_tiles;
  const int tile_w = mt % p.tiles_w, tile_h = (mt / p.tiles_w) % p.tiles_h, tile_n = mt / (p.tiles_w * p.tiles_h);
  const int rows_img = p.th * p.tw;
  constexpr int C4 = BN / 4;
  static_assert(256 % C4 == 0, "each thread keeps one fixed channel group");
  const float* base = p.ws + (size_t)slot * p.splits * (size_t)(BLOCK_M * BN);
  const bool vec_ok = (p.cout & 3) == 0;
  const int cg = threadIdx.x % C4;
  const int c = nblk * BN + cg * 4;
  if (c >= p.cout) return;
  const float4 sc4 = __ldg(reinterpret_cast<const float4*>(p.scale + c)), sh4 = __ldg(reinterpret_cast<const float4*>(p.shift + c));   // padded vectors
  const float sc[4] = {sc4.x, sc4.y, sc4.z, sc4.w}, sh[4] = {sh4.x, sh4.y, sh4.z, sh4.w};
  {
    const int row = rgroup * RPB + threadIdx.x / C4;
    const int dn = row / rows_img, rem = row % rows_img;
    const int n = tile_n * p.tn + dn, h = tile_h * p.th + rem / p.tw, w = tile_w * p.tw + rem % p.tw;
    if (row >= p.tn * rows_img || n >= p.nimg || h >= p.ho || w >= p.wo) return;
    const size_t o = ((((size_t)n * p.ho + h) * p.wo + w)) * p.cout + c;
    float4 rv = make_float4(0.f, 0.f, 0.f, 0.f);
    if (p.residual) {
      if (vec_ok) rv = __ldg(reinterpret_cast<const float4*>(p.residual + o));
      else { float t[4] = {0.f, 0.f, 0.f, 0.f}; for (int e = 0; e < 4; ++e) if (c + e < p.cout) t[e] = __ldg(p.residual + o + e); rv = make_float4(t[0], t[1], t[2], t[3]); }
    }
    float4 a = __ldg(reinterpret_cast<const float4*>(base + (size_t)row * BN) + cg);
    for (int z = 1; z < p.splits; ++z) {
      const float4 b = __ldg(reinterpret_cast<const float4*>(base + ((size_t)z * BLOCK_M + row) * BN) + cg);
      a.x = __fadd_rn(a.x, b.x); a.y = __fadd_rn(a.y, b.y); a.z = __fadd_rn(a.z, b.z); a.w = __fadd_rn(a.w, b.w);
    }
    float y[4] = {a.x, a.y, a.z, a.w};
    const float res[4] = {rv.x, rv.y, rv.z, rv.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      float v = y[e];
      v = __fadd_rn(__fmul_rn(v, sc[e]), sh[e]);
      if (p.residual) v = __fadd_rn(v, res[e]);
      if (p.act == FRCNN_ACT_RELU) v = fmaxf(v, 0.f);
      else if (p.act == FRCNN_ACT_RELU6) v = fminf(fmaxf(v, 0.f), 6.f);
      y[e] = v;
    }
    if (vec_ok) *reinterpret_cast<float4*>(p.out + o) = make_float4(y[0], y[1], y[2], y[3]);
    else for (int e = 0; e < 4; ++e) if (c + e < p.cout) p.out[o + e] = y[e];
  }
}

// Second pass of the mean epilogue: mean_out[g][c] = (tile partials of group g, added in tile order) / mean_hw.  A group's
// pixels lie in one or two tiles when mean_hw <= tile width (more for longer groups); thread = (group, channel).
__global__ void __launch_bounds__(256)
mean_finish_kernel(const ConvKernelParams p) {
  pdl_launch_dependents();
  pdl_wait();
  const long gid = (long)blockIdx.x * blockDim.x + threadIdx.x;
  const int groups = p.wo / p.mean_hw;
  if (gid >= (long)groups * p.cout) return;
  const int c = (int)(gid % p.cout), g = (int)(gid / p.cout);
  const int hw = p.mean_hw;
  const size_t ld = (size_t)p.mean_ld;
  const long p0 = (long)g * hw, p1 = p0 + hw - 1;
  const int m0 = (int)(p0 / p.tw), m1 = (int)(p1 / p.tw);
  float sum = 0.f;
  for (int m = m0; m <= m1; ++m) {
    const int s = g - (int)(((long)m * p.tw) / hw);
    const float v = p.mean_ws[((size_t)m * p.mean_segs + s) * ld + c];
    sum = m == m0 ? v : __fadd_rn(sum, v);
  }
  p.mean_out[(size_t)g * p.cout + c] = __fdiv_rn(sum, (float)hw);
}

// plan creation: the epilogue's per-channel vectors, padded to the tile grid (no bounds tests in the kernel)
__global__ void prep_epilogue_vectors_kernel(const float* scale, const float* shift, float out_mult, int cout, int padded,
                                             float* eff_scale, float* eff_shift) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= padded) return;
  const float sc = (c < cout && scale) ? scale[c] : 1.f;
  eff_scale[c] = __fmul_rn(sc, out_mult);                  // exact: out_mult is a power of two
  eff_shift[c] = (c < cout && shift) ? shift[c] : 0.f;
}

// ---------------------------------------------------------------------------------------------------
// host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(ptr);
  }
  return fn;
}

static int encode_map(CUtensorMap* m, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                      const uint32_t* box, const uint32_t* estr, CUtensorMapDataType dtype = CU_TENSOR_MAP_DATA_TYPE_FLOAT32,
                      CUtensorMapSwizzle swz = CU_TENSOR_MAP_SWIZZLE_128B) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) { set_error("cuTensorMapEncodeTiled entry point unavailable"); return ERR_DRIVER_ENTRY; }
  cuuint64_t gd[5]; cuuint64_t gs[4]; cuuint32_t bx[5]; cuuint32_t es[5];
  for (int i = 0; i < rank; ++i) { gd[i] = dims[i]; bx[i] = box[i]; es[i] = estr[i]; }
  for (int i = 0; i + 1 < rank; ++i) gs[i] = strides_bytes[i];
  CUresult r = fn(m, dtype, (cuuint32_t)rank, const_cast<void*>(base), gd, gs, bx, es,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (CUresult %d) rank=%d dims=[%llu,%llu,%llu,%llu] box=[%u,%u,%u,%u]", (int)r, rank,
              (unsigned long long)dims[0], (unsigned long long)dims[1], rank > 2 ? (unsigned long long)dims[2] : 0ull,
              rank > 3 ? (unsigned long long)dims[3] : 0ull, box[0], box[1], rank > 2 ? box[2] : 0u, rank > 3 ? box[3] : 0u);
    return ERR_CUDA;
  }
  return OK;
}

}  // namespace frcnn

using namespace frcnn;

struct frcnn_conv_plan {
  CUtensorMap tmA, tmA2, tmBhi, tmBlo;   // tmA2: the second A source, or a copy of tmA
  ConvKernelParams kp;
  int block_n, stages, smem;
  int impl;                // FRCNN_CONV_F16X3 | FRCNN_CONV_TF32X3 | FRCNN_CONV_F16X1
  dim3 grid;
  int n_tail;
  float* ws;               // owned workspace of the split tiles 
  float* eff;              // owned epilogue vectors: scale * out_mult | shift, each padded to n_tiles * block_n
  float* mean_ws;          // owned tile partials of the mean epilogue
};

// choose the tile of output pixels (tn x th x tw <= 128) that needs the fewest tiles
static void choose_tile(int n, int ho, int wo, int stride, int* tn, int* th, int* tw) {
  long best_tiles = -1; int bn = 1, bh = 1, bw = 1; int best_rows = 0;
  const int lim = 256 / stride;
  for (int a = 1; a <= n && a <= BLOCK_M; ++a)
    for (int b = 1; b <= ho && a * b <= BLOCK_M && b <= lim; ++b) {
      int c = BLOCK_M / (a * b);
      if (c > wo) c = wo;
      if (c > lim) c = lim;
      if (c < 1) continue;
      // shrink c to the smallest width giving the same tile count (less garbage rows)
      int tiles_w = cdiv(wo, c);
      c = cdiv(wo, tiles_w);
      long tiles = (long)cdiv(n, a) * cdiv(ho, b) * tiles_w;
      int rows = a * b * c;
      if (best_tiles < 0 || tiles < best_tiles || (tiles == best_tiles && rows < best_rows)) {
        best_tiles = tiles; bn = a; bh = b; bw = c; best_rows = rows;
      }
    }
  *tn = bn; *th = bh; *tw = bw;
}

// FRCNN_NO_PDL=1 disables programmatic dependent launch (debug / A-B measurements)
static bool pdl_enabled() {
  static int v = -1;
  if (v < 0) { const char* e = getenv("FRCNN_NO_PDL"); v = (e && e[0] == '1') ? 0 : 1; }
  return v == 1;
}

template <int BN, int MODE>
static int launch(const frcnn_conv_plan* p, cudaStream_t st) {
  static bool attr_done = false;
  if (!attr_done) {
    FRCNN_CUDA(cudaFuncSetAttribute(conv_gemm_kernel<BN, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    smem_bytes<BN, MODE>() + MEAN_SMEM));
    attr_done = true;
  }
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  const bool pdl = pdl_enabled();
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = p->grid; cfg.blockDim = dim3(NUM_THREADS); cfg.stream = st;
  cfg.dynamicSmemBytes = smem_bytes<BN, MODE>() + (p->kp.mean_out ? MEAN_SMEM : 0);
  cfg.attrs = attr; cfg.numAttrs = pdl ? 1 : 0;
  FRCNN_CUDA(cudaLaunchKernelEx(&cfg, conv_gemm_kernel<BN, MODE>, p->tmA, p->tmA2, p->tmBhi, p->tmBlo, p->kp));
  if (p->kp.mean_out) {
    cudaLaunchConfig_t mc{};
    const long n = (long)(p->kp.wo / p->kp.mean_hw) * p->kp.cout;
    mc.gridDim = dim3((unsigned)((n + 255) / 256)); mc.blockDim = dim3(256); mc.dynamicSmemBytes = 0; mc.stream = st;
    mc.attrs = attr; mc.numAttrs = pdl ? 1 : 0;
    FRCNN_CUDA(cudaLaunchKernelEx(&mc, mean_finish_kernel, p->kp));
  }
  if (p->n_tail > 0) {
    cudaLaunchConfig_t rc{};
    rc.gridDim = dim3((unsigned)(p->n_tail * (BLOCK_M / (256 / (BN / 4))))); rc.blockDim = dim3(256); rc.dynamicSmemBytes = 0; rc.stream = st;
    rc.attrs = attr; rc.numAttrs = pdl ? 1 : 0;
    FRCNN_CUDA(cudaLaunchKernelEx(&rc, tail_reduce_kernel<BN>, p->kp));
  }
  return OK;
}

// Host-side work decomposition of one layer (no CUDA calls: unit-testable on a CPU box through frcnn_conv_plan_geometry).
struct Geometry {
  int n, h, w, ho, wo;           // after flattening 1x1/stride-1 layers to one row of n*h*w pixels
  int tn, th, tw, tiles_w, tiles_h, tiles_n;
  long m_tiles;
  int num_kb, bn, n_tiles, kpc;
  long tiles, n_tail;
  int splits, kbs;
  long total_units;
  int grid;
  int raster_n;
};

static int decide_geometry(const frcnn_conv_desc* d, int sms, Geometry* g) {
  FRCNN_REQUIRE(d->cin > 0 && d->cin % BLOCK_K == 0, "cin=%d must be a positive multiple of 32", d->cin);
  FRCNN_REQUIRE(d->kh >= 1 && d->kw >= 1 && d->stride >= 1 && d->stride <= 8, "bad filter geometry");
  FRCNN_REQUIRE(d->n > 0 && d->h > 0 && d->w > 0 && d->ho > 0 && d->wo > 0 && d->cout > 0, "bad shape");
  FRCNN_REQUIRE(sms > 0, "bad SM count");
  g->n = d->n; g->h = d->h; g->w = d->w; g->ho = d->ho; g->wo = d->wo;
  const bool pointwise = d->kh == 1 && d->kw == 1 && d->stride == 1 && d->pad_t == 0 && d->pad_l == 0 && g->ho == g->h && g->wo == g->w;
  const bool mean = d->mean_hw != 0;
  FRCNN_REQUIRE(d->cin2 >= 0 && d->cin2 % BLOCK_K == 0, "cin2=%d must be 0 or a positive multiple of 32", d->cin2);
  FRCNN_REQUIRE(d->cin2 == 0 || pointwise, "a second A source needs a pointwise layer (1x1, stride 1, no padding)");
  FRCNN_REQUIRE(!mean || pointwise, "the mean epilogue needs a pointwise layer (1x1, stride 1, no padding)");
  FRCNN_REQUIRE(!mean || d->cout % 4 == 0, "the mean epilogue needs cout %% 4 == 0 (cout=%d)", d->cout);
  FRCNN_REQUIRE(d->mean_hw >= 0 && (!mean || ((long)d->n * d->h * d->w) % d->mean_hw == 0),
                "mean_hw=%d must be positive and divide the pixel count", d->mean_hw);
  FRCNN_REQUIRE(!mean || d->split_k <= 1, "the mean epilogue is never split along K");
  if (pointwise) {  // flatten all pixels into one row of "width" n*h*w: perfect 128-row tiles
    g->w = g->wo = g->n * g->h * g->w; g->n = 1; g->h = g->ho = 1;
  }
  const int ktot = d->kh * d->kw * d->cin + d->cin2;             // K of the packed weights
  choose_tile(g->n, g->ho, g->wo, d->stride, &g->tn, &g->th, &g->tw);
  g->tiles_w = cdiv(g->wo, g->tw); g->tiles_h = cdiv(g->ho, g->th); g->tiles_n = cdiv(g->n, g->tn);
  g->m_tiles = (long)g->tiles_w * g->tiles_h * g->tiles_n;
  const bool f16 = d->impl != FRCNN_CONV_TF32X3;
  const int ks = f16 ? 2 : 1;                                   // 32-channel blocks per k-block (f16x3: 64-wide k-blocks)
  g->num_kb = cdiv(ktot / BLOCK_K, ks);
  g->kpc = d->kb_per_chunk > 0 ? d->kb_per_chunk : 8 / ks;
  int bn = d->block_n;
  if (bn == 0) {
    long best = -1;
    const int cands[2] = {128, 64};
    for (int i = 0; i < 2; ++i) {
      const int c = cands[i];
      if (c > 64 && c / 2 >= d->cout) continue;        // tile mostly empty
      const long ctas = g->m_tiles * cdiv(d->cout, c);
      const long waves = (ctas + sms - 1) / sms;
      // cost model: a k-block costs about the same whatever block_n is (the 128-row A operand and its split dominate for
      // N <= 128), plus a fixed per-unit cost => fewest rounds wins, widest tile on ties
      const long cost = f16 ? waves * (g->num_kb * 900L + 4000L) : waves * (g->num_kb * 1400L + 6000L);
      if (best < 0 || cost < best) { best = cost; bn = c; }
    }
  }
  FRCNN_REQUIRE(bn == 64 || bn == 128, "block_n must be 64 or 128");
  g->bn = bn;
  g->n_tiles = cdiv(d->cout, bn);
  g->tiles = g->m_tiles * g->n_tiles;
  FRCNN_REQUIRE(g->tiles <= 0x3fffffffL, "too many tiles");
  // ---- whole tiles + K-split tail (see ConvKernelParams) ---------------------------------------------------------------
  long n_tail = 0; int splits = 1;
  const int num_kb = g->num_kb;
  const int max_split = num_kb * ks / 8 < 8 ? num_kb * ks / 8 : 8;   // >= 8 32-wide k-blocks (one chunk) per split, at most 8 splits
  if (d->split_k > 1) {                                         // forced: every tile is split
    n_tail = g->tiles; splits = d->split_k;
  } else if (d->split_k == 0 && max_split >= 2) {
    const long rem = g->tiles % sms;
    // a split unit still pays a per-unit overhead and the reduce pass a launch of its own, so the ragged round is only
    // worth splitting when the K loop is long (>= 48 32-wide k-blocks); layers too small to fill the GPU gain from 16 on.
    if (g->tiles <= sms / 2) { if (num_kb * ks >= 16) { n_tail = g->tiles; splits = (int)(sms / g->tiles); } }   // layer too small to fill the GPU
    else if (g->tiles > sms && rem > 0 && rem <= sms / 2 && num_kb * ks >= 48) { n_tail = rem; splits = (int)(sms / rem); }   // ragged last round
    if (splits > max_split) splits = max_split;
    if (splits < 2) { n_tail = 0; splits = 1; }
  }
  int kbs = cdiv(num_kb, splits);                              // (a unit's last chunk may be shorter than kb_per_chunk)
  splits = cdiv(num_kb, kbs);
  // tail_reduce_kernel reads the padded epilogue vectors as float4; the mean epilogue sums whole tiles
  if (splits < 2 || (d->cout & 3) != 0 || mean) { n_tail = 0; splits = 1; kbs = num_kb; }
  FRCNN_REQUIRE(splits <= 64, "bad split_k");
  g->n_tail = n_tail; g->splits = splits; g->kbs = kbs;
  g->total_units = (g->tiles - n_tail) + n_tail * splits;
  FRCNN_REQUIRE(g->total_units <= 0x7fffffffL, "too many work units");
  g->grid = (int)(g->total_units < sms ? g->total_units : sms);   // persistent: one CTA per SM walks the units
  {
    const char* e = getenv("FRCNN_CONV_RASTER");          // development override: m | n
    const double a_bytes = (double)d->n * d->h * d->w * (d->cin + d->cin2) * 4.0, b_bytes = (double)d->cout * ktot * 4.0;
    g->raster_n = (e && (e[0] == 'm' || e[0] == 'n')) ? (e[0] == 'n') : (a_bytes > b_bytes && g->n_tiles > 1);
  }
  return OK;
}

extern "C" int frcnn_conv_plan_geometry(const frcnn_conv_desc* d, int sm_count, int* out16) {
  FRCNN_REQUIRE(d && out16, "null argument");
  Geometry g;
  int rc = decide_geometry(d, sm_count, &g);
  if (rc) return rc;
  const int v[16] = {g.bn, g.tn, g.th, g.tw, (int)g.m_tiles, g.n_tiles, (int)g.tiles, (int)g.n_tail, g.splits, g.kbs,
                     (int)g.total_units, g.grid, g.num_kb, g.kpc, g.tiles_h, g.tiles_w};
  for (int i = 0; i < 16; ++i) out16[i] = v[i];
  return OK;
}

extern "C" int frcnn_conv_plan_create(frcnn_conv_plan** out, const frcnn_conv_desc* d) {
  FRCNN_REQUIRE(out && d, "null argument");
  FRCNN_REQUIRE(d->in_dev && d->w_hi_dev && d->w_lo_dev && (d->mean_hw ? d->mean_dev != nullptr : d->out_dev != nullptr),
                "null device pointer");
  FRCNN_REQUIRE(d->cin2 == 0 || d->in2_dev, "cin2=%d without in2_dev", d->cin2);
  int sms = 132;
  { int dev = 0; cudaDeviceProp pr; if (cudaGetDevice(&dev) == cudaSuccess && cudaGetDeviceProperties(&pr, dev) == cudaSuccess && pr.multiProcessorCount > 0) sms = pr.multiProcessorCount; }
  Geometry g;
  int grc = decide_geometry(d, sms, &g);
  if (grc) return grc;
  frcnn_conv_plan* p = (frcnn_conv_plan*)aligned_alloc(64, (sizeof(frcnn_conv_plan) + 63) / 64 * 64);
  if (!p) { set_error("out of host memory"); return ERR_ARG; }
  memset(p, 0, sizeof(*p));
  const int bn = g.bn;
  // A: NHWC activations as a rank-4 tensor {C, W, H, N}; traversal stride = conv stride on W and H
  {
    uint64_t dims[4] = {(uint64_t)d->cin, (uint64_t)g.w, (uint64_t)g.h, (uint64_t)g.n};
    uint64_t strides[3] = {(uint64_t)d->cin * 4, (uint64_t)g.w * d->cin * 4, (uint64_t)g.h * g.w * d->cin * 4};
    uint32_t box[4] = {(uint32_t)BLOCK_K, (uint32_t)(g.tw * d->stride), (uint32_t)(g.th * d->stride), (uint32_t)g.tn};
    uint32_t es[4] = {1, (uint32_t)d->stride, (uint32_t)d->stride, 1};
    int rc = encode_map(&p->tmA, d->in_dev, 4, dims, strides, box, es);
    if (rc) { free(p); return rc; }
    p->tmA2 = p->tmA;
    if (d->cin2 > 0) {   // pointwise: same pixel rows, cin2 channels
      uint64_t dims2[4] = {(uint64_t)d->cin2, (uint64_t)g.w, (uint64_t)g.h, (uint64_t)g.n};
      uint64_t strides2[3] = {(uint64_t)d->cin2 * 4, (uint64_t)g.w * d->cin2 * 4, (uint64_t)g.h * g.w * d->cin2 * 4};
      rc = encode_map(&p->tmA2, d->in2_dev, 4, dims2, strides2, box, es);
      if (rc) { free(p); return rc; }
    }
  }
  const bool f16 = d->impl != FRCNN_CONV_TF32X3;
  {
    const uint64_t ktot = (uint64_t)d->kh * d->kw * d->cin + d->cin2;
    uint64_t dims[2] = {ktot, (uint64_t)d->cout};
    uint64_t strides[1] = {ktot * (f16 ? 2 : 4)};
    uint32_t box[2] = {(uint32_t)(f16 ? 2 * BLOCK_K : BLOCK_K), (uint32_t)bn};   // 128-byte rows either way
    uint32_t es[2] = {1, 1};
    const CUtensorMapDataType dt = f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
    const CUtensorMapSwizzle sw = CU_TENSOR_MAP_SWIZZLE_128B;
    int rc = encode_map(&p->tmBhi, d->w_hi_dev, 2, dims, strides, box, es, dt, sw);
    if (!rc) rc = encode_map(&p->tmBlo, d->w_lo_dev, 2, dims, strides, box, es, dt, sw);
    if (rc) { free(p); return rc; }
  }
  ConvKernelParams& k = p->kp;
  k.out = d->out_dev; k.residual = d->residual_dev;
  k.cout = d->cout; k.ho = g.ho; k.wo = g.wo; k.nimg = g.n;
  k.tn = g.tn; k.th = g.th; k.tw = g.tw; k.tiles_h = g.tiles_h; k.tiles_w = g.tiles_w;
  k.kh = d->kh; k.kw = d->kw; k.cin = d->cin; k.stride = d->stride; k.pad_t = d->pad_t; k.pad_l = d->pad_l;
  k.act = d->act;
  k.a_box_bytes = g.tn * g.th * g.tw * BLOCK_K * 4;
  k.trace = nullptr;
  k.num_kb_total = g.num_kb;
  k.m_tiles = (int)g.m_tiles; k.n_tiles = g.n_tiles;
  k.kb_per_split = g.kbs; k.splits = g.splits; k.n_full = (int)(g.tiles - g.n_tail);
  k.total_units = (int)g.total_units;
  k.raster_n = g.raster_n;
  k.cin2 = d->cin2;
  k.mean_out = d->mean_hw ? d->mean_dev : nullptr; k.mean_ws = nullptr; k.mean_hw = d->mean_hw; k.mean_ld = g.n_tiles * bn;
  k.mean_segs = d->mean_hw ? (g.tw < cdiv(g.tw - 1, d->mean_hw) + 1 ? g.tw : cdiv(g.tw - 1, d->mean_hw) + 1) : 0;
  k.ws = nullptr; p->ws = nullptr; p->eff = nullptr; p->mean_ws = nullptr; p->n_tail = (int)g.n_tail;
  {
    // NOTE: the vectors are snapshots of scale_dev / shift_dev taken now (they are weights: constant after load)
    const int padded = g.n_tiles * bn;
    const float om = f16 ? (d->out_mult != 0.f ? d->out_mult : 1.f) : 1.f;
    cudaError_t e = cudaMalloc(&p->eff, (size_t)2 * padded * sizeof(float));
    if (e != cudaSuccess) { free(p); return cuda_fail(e, "epilogue vectors", __FILE__, __LINE__); }
    prep_epilogue_vectors_kernel<<<cdiv(padded, 256), 256>>>(d->scale_dev, d->shift_dev, om, d->cout, padded, p->eff, p->eff + padded);
    e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e != cudaSuccess) { cudaFree(p->eff); free(p); return cuda_fail(e, "prep_epilogue_vectors", __FILE__, __LINE__); }
    k.scale = p->eff; k.shift = p->eff + padded;
  }
  if (g.n_tail > 0) {
    cudaError_t e = cudaMalloc(&p->ws, (size_t)g.n_tail * g.splits * BLOCK_M * bn * sizeof(float));
    if (e != cudaSuccess) { cudaFree(p->eff); free(p); return cuda_fail(e, "split-tile workspace", __FILE__, __LINE__); }
    k.ws = p->ws;
  }
  if (d->mean_hw) {
    cudaError_t e = cudaMalloc(&p->mean_ws, (size_t)g.m_tiles * k.mean_segs * k.mean_ld * sizeof(float));
    if (e != cudaSuccess) { cudaFree(p->eff); free(p); return cuda_fail(e, "mean workspace", __FILE__, __LINE__); }
    k.mean_ws = p->mean_ws;
  }
  p->grid = dim3((unsigned)g.grid, 1, 1);
  p->block_n = bn;
  p->impl = f16 ? (d->impl == FRCNN_CONV_F16X1 ? FRCNN_CONV_F16X1 : FRCNN_CONV_F16X3) : FRCNN_CONV_TF32X3;
  p->stages = STAGES;
  p->smem = f16 ? (bn == 128 ? smem_bytes<128, FRCNN_CONV_F16X3>() : smem_bytes<64, FRCNN_CONV_F16X3>())
              : (bn == 128 ? smem_bytes<128, FRCNN_CONV_TF32X3>() : smem_bytes<64, FRCNN_CONV_TF32X3>());
  if (d->mean_hw) p->smem += MEAN_SMEM;
  *out = p;
  return OK;
}

extern "C" int frcnn_conv_plan_run(const frcnn_conv_plan* p, void* stream) {
  FRCNN_REQUIRE(p, "null plan");
  cudaStream_t st = (cudaStream_t)stream;
  if (p->impl == FRCNN_CONV_F16X3) return p->block_n == 128 ? launch<128, FRCNN_CONV_F16X3>(p, st) : launch<64, FRCNN_CONV_F16X3>(p, st);
  if (p->impl == FRCNN_CONV_F16X1) return p->block_n == 128 ? launch<128, FRCNN_CONV_F16X1>(p, st) : launch<64, FRCNN_CONV_F16X1>(p, st);
  return p->block_n == 128 ? launch<128, FRCNN_CONV_TF32X3>(p, st) : launch<64, FRCNN_CONV_TF32X3>(p, st);
}

extern "C" int frcnn_conv_plan_info(const frcnn_conv_plan* p, int* block_n, int* tile_n, int* tile_h, int* tile_w,
                                    int* grid_m, int* grid_n, int* stages, int* smem) {
  FRCNN_REQUIRE(p, "null plan");
  if (block_n) *block_n = p->block_n;
  if (tile_n) *tile_n = p->kp.tn;
  if (tile_h) *tile_h = p->kp.th;
  if (tile_w) *tile_w = p->kp.tw;
  if (grid_m) *grid_m = p->kp.m_tiles;
  if (grid_n) *grid_n = p->kp.n_tiles;
  if (stages) *stages = p->n_tail > 0 ? p->kp.splits : 1;   /* "splits" of the tail tiles */
  if (smem) *smem = p->smem;
  return OK;
}

extern "C" int frcnn_debug_watchdog(unsigned int* out16, int reset) {
  FRCNN_REQUIRE(out16, "null argument");
#ifdef FRCNN_WATCHDOG
  FRCNN_CUDA(cudaMemcpyFromSymbol(out16, g_watchdog, 16 * sizeof(unsigned int)));
  if (reset) { unsigned int z[16] = {0}; FRCNN_CUDA(cudaMemcpyToSymbol(g_watchdog, z, sizeof(z))); }
  return OK;
#else
  (void)reset;
  for (int i = 0; i < 16; ++i) out16[i] = 0;
  out16[15] = 0xffffffffu;   // "not a watchdog build"
  return OK;
#endif
}

extern "C" int frcnn_conv_plan_set_trace(frcnn_conv_plan* p, long long* trace_dev) {
  FRCNN_REQUIRE(p, "null plan");
  p->kp.trace = trace_dev;
  return OK;
}

extern "C" void frcnn_conv_plan_destroy(frcnn_conv_plan* p) {
  if (p && p->ws) cudaFree(p->ws);
  if (p && p->eff) cudaFree(p->eff);
  if (p && p->mean_ws) cudaFree(p->mean_ws);
  free(p);
}
