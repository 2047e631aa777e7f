// Bandwidth-bound stages of the TEST graph as coalesced / float4-vectorised SIMT kernels (fp32).
// Where the oracle (numpy, no FMA) performs separate roundings the kernels use __f*_rn intrinsics so that
// nvcc cannot contract them; reference file:line citations are in include/frcnn_b200.h.
#include <cuda_fp16.h>
#include <math.h>
#include <climits>
#include "common.cuh"
#include "../../include/frcnn_b200.h"

namespace frcnn {

__device__ __forceinline__ float apply_act(float v, int act) {
  if (act == FRCNN_ACT_RELU) return fmaxf(v, 0.f);
  if (act == FRCNN_ACT_RELU6) return fminf(fmaxf(v, 0.f), 6.f);
  return v;
}

// ---- weight packing: HWIO -> [cout][kh*kw*cin] hi/lo tf32 planes ---------------------------------------
__global__ void pack_weights_kernel(const float* __restrict__ w, float* __restrict__ hi, float* __restrict__ lo,
                                    int ktot, int cout) {
  const size_t total = (size_t)ktot * cout;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int k = (int)(i % ktot);
    const int co = (int)(i / ktot);
    const float v = w[(size_t)k * cout + co];
    const float h = to_tf32(v);
    hi[i] = h;
    lo[i] = to_tf32(__fsub_rn(v, h));
  }
}

// fp16 planes for the FP16x3 kernel: hi = RN_f16(w * 2^wexp), lo = RN_f16((w * 2^wexp - hi) * 2^11)  (see conv_gemm.cu)
__global__ void pack_weights_f16_kernel(const float* __restrict__ w, __half* __restrict__ hi, __half* __restrict__ lo,
                                        int ktot, int cout, float wmul) {
  const size_t total = (size_t)ktot * cout;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int k = (int)(i % ktot);
    const int co = (int)(i / ktot);
    const float v = __fmul_rn(w[(size_t)k * cout + co], wmul);
    const __half h = __float2half_rn(v);
    hi[i] = h;
    lo[i] = __float2half_rn(__fmul_rn(__fsub_rn(v, __half2float(h)), 2048.f));
  }
}

// ---- first-layer convolution, cin == 3 ------------------------------------------------------------------
// Block = CF_TH x CF_TW output pixels x all output channels.  The input patch and the whole filter bank sit in shared memory;
// a warp = 32 lanes x PIX pixels each x one group of 32 output channels, so every weight read is a warp-wide broadcast float4
// and each thread keeps 32 * PIX accumulators.  r02: with PIX = 1 the loop issued 9 LDS per 32 FFMA (1 input + 8 weight float4)
// and was bound by the shared-memory pipe (ncu: SM 43 %, 21 TFLOP/s of fp32); PIX = 2 reuses every weight float4 for two pixels
// (10 LDS per 64 FFMA).  The accumulation order per output is unchanged (taps in (r, s, c) order, one fmaf each).
constexpr int CF_TH = 8, CF_TW = 32;
template <int PIX>
__global__ void __launch_bounds__(256, PIX == 2 ? 2 : 1)
conv_first_kernel(const float* __restrict__ in, const float* __restrict__ w, const float* __restrict__ scale,
                  const float* __restrict__ shift, float* __restrict__ out, int h, int wd, int cout, int k, int stride,
                  int pad_t, int pad_l, int ho, int wo, int act, int tiles_x, int tiles_y) {
  extern __shared__ float smem_cf[];
  const int taps = k * k * 3;
  float* wsm = smem_cf;                                   // [k*k*3][cout]
  const int ph = (CF_TH - 1) * stride + k, pw = (CF_TW - 1) * stride + k;
  float* psm = smem_cf + taps * cout;                     // [ph][pw][3]
  const int tile = blockIdx.x;
  const int tx = tile % tiles_x, ty = (tile / tiles_x) % tiles_y, b = tile / (tiles_x * tiles_y);
  const int oy0 = ty * CF_TH, ox0 = tx * CF_TW;
  const int iy0 = oy0 * stride - pad_t, ix0 = ox0 * stride - pad_l;
  for (int i = threadIdx.x; i < taps * cout; i += blockDim.x) wsm[i] = __ldg(w + i);
  for (int i = threadIdx.x; i < ph * pw * 3; i += blockDim.x) {
    const int c = i % 3, x = (i / 3) % pw, y = i / (3 * pw);
    const int iy = iy0 + y, ix = ix0 + x;
    psm[i] = (iy >= 0 && iy < h && ix >= 0 && ix < wd) ? __ldg(in + (((size_t)b * h + iy) * wd + ix) * 3 + c) : 0.f;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int groups = cout >> 5;                           // 32-channel groups (1 or 2)
  const int g = warp % groups;
  const int pblk = warp / groups;                         // block of 32 * PIX pixels inside the tile
  const int nblk = (blockDim.x >> 5) / groups;
  for (int pb = pblk; pb < (CF_TH * CF_TW) / (32 * PIX); pb += nblk) {
    int py[PIX], px[PIX];
#pragma unroll
    for (int q = 0; q < PIX; ++q) {
      const int pix = pb * 32 * PIX + q * 32 + lane;
      py[q] = pix / CF_TW; px[q] = pix % CF_TW;
    }
    float acc[PIX][32];
#pragma unroll
    for (int q = 0; q < PIX; ++q)
#pragma unroll
      for (int i = 0; i < 32; ++i) acc[q][i] = 0.f;
    for (int r = 0; r < k; ++r)
      for (int s2 = 0; s2 < k; ++s2) {
        const float* ip[PIX];
#pragma unroll
        for (int q = 0; q < PIX; ++q) ip[q] = psm + ((py[q] * stride + r) * pw + px[q] * stride + s2) * 3;
        const float* wp = wsm + ((r * k + s2) * 3) * cout + g * 32;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          float x[PIX];
#pragma unroll
          for (int q = 0; q < PIX; ++q) x[q] = ip[q][c];
          const float4* w4 = reinterpret_cast<const float4*>(wp + c * cout);
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float4 wv = w4[j];
#pragma unroll
            for (int q = 0; q < PIX; ++q) {
              acc[q][4 * j + 0] = fmaf(x[q], wv.x, acc[q][4 * j + 0]); acc[q][4 * j + 1] = fmaf(x[q], wv.y, acc[q][4 * j + 1]);
              acc[q][4 * j + 2] = fmaf(x[q], wv.z, acc[q][4 * j + 2]); acc[q][4 * j + 3] = fmaf(x[q], wv.w, acc[q][4 * j + 3]);
            }
          }
        }
      }
#pragma unroll
    for (int q = 0; q < PIX; ++q) {
      const int oy = oy0 + py[q], ox = ox0 + px[q];
      if (oy < ho && ox < wo) {
        float* op = out + (((size_t)b * ho + oy) * wo + ox) * cout + g * 32;
#pragma unroll
        for (int i = 0; i < 32; ++i) {
          float v = acc[q][i];
          const int ch = g * 32 + i;
          if (scale) v = __fmul_rn(v, __ldg(scale + ch));
          if (shift) v = __fadd_rn(v, __ldg(shift + ch));
          acc[q][i] = apply_act(v, act);
        }
#pragma unroll
        for (int i = 0; i < 32; i += 4) *reinterpret_cast<float4*>(op + i) = make_float4(acc[q][i], acc[q][i + 1], acc[q][i + 2], acc[q][i + 3]);
      }
    }
  }
}

// ---- depthwise 3x3 ---------------------------------------------------------------------------------------
__global__ void depthwise3x3_kernel(const float* __restrict__ in, const float* __restrict__ w,
                                    const float* __restrict__ scale, const float* __restrict__ shift,
                                    float* __restrict__ out, int n, int h, int wd, int c, int stride, int pad_t,
                                    int pad_l, int ho, int wo, int act) {
  const int c4 = c >> 2;
  const long total = (long)n * ho * wo * c4;
  const long gid = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (gid >= total) return;
  const int cg = (int)(gid % c4);
  const long pix = gid / c4;
  const int ox = (int)(pix % wo);
  const int oy = (int)((pix / wo) % ho);
  const int b = (int)(pix / ((long)wo * ho));
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    const int iy = oy * stride - pad_t + r;
    if (iy < 0 || iy >= h) continue;
#pragma unroll
    for (int s = 0; s < 3; ++s) {
      const int ix = ox * stride - pad_l + s;
      if (ix < 0 || ix >= wd) continue;
      const float4 x = __ldg(reinterpret_cast<const float4*>(in + (((size_t)b * h + iy) * wd + ix) * c) + cg);
      const float4 k4 = __ldg(reinterpret_cast<const float4*>(w + (size_t)(r * 3 + s) * c) + cg);
      acc.x = fmaf(x.x, k4.x, acc.x); acc.y = fmaf(x.y, k4.y, acc.y);
      acc.z = fmaf(x.z, k4.z, acc.z); acc.w = fmaf(x.w, k4.w, acc.w);
    }
  }
  float v[4] = {acc.x, acc.y, acc.z, acc.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int ch = cg * 4 + i;
    if (scale) v[i] = __fmul_rn(v[i], __ldg(scale + ch));
    if (shift) v[i] = __fadd_rn(v[i], __ldg(shift + ch));
    v[i] = apply_act(v[i], act);
  }
  reinterpret_cast<float4*>(out + (size_t)pix * c)[cg] = make_float4(v[0], v[1], v[2], v[3]);
}

// ---- max pool ----------------------------------------------------------------------------------------------
__global__ void max_pool_kernel(const float* __restrict__ in, float* __restrict__ out, int n, int h, int wd, int c,
                                int k, int stride, int pad_t, int pad_l, int ho, int wo, int pad_neg_inf) {
  const int c4 = c >> 2;
  const long total = (long)n * ho * wo * c4;
  const long gid = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (gid >= total) return;
  const int cg = (int)(gid % c4);
  const long pix = gid / c4;
  const int ox = (int)(pix % wo);
  const int oy = (int)((pix / wo) % ho);
  const int b = (int)(pix / ((long)wo * ho));
  const float ninf = __int_as_float(0xff800000);
  float4 m = make_float4(ninf, ninf, ninf, ninf);
  for (int r = 0; r < k; ++r) {
    const int iy = oy * stride - pad_t + r;
    for (int s = 0; s < k; ++s) {
      const int ix = ox * stride - pad_l + s;
      float4 x;
      if (iy < 0 || iy >= h || ix < 0 || ix >= wd) {
        if (pad_neg_inf) continue;
        x = make_float4(0.f, 0.f, 0.f, 0.f);
      } else {
        x = __ldg(reinterpret_cast<const float4*>(in + (((size_t)b * h + iy) * wd + ix) * c) + cg);
      }
      m.x = fmaxf(m.x, x.x); m.y = fmaxf(m.y, x.y); m.z = fmaxf(m.z, x.z); m.w = fmaxf(m.w, x.w);
    }
  }
  reinterpret_cast<float4*>(out + (size_t)pix * c)[cg] = m;
}

// ---- spatial mean -------------------------------------------------------------------------------------------
__global__ void spatial_mean_kernel(const float* __restrict__ in, float* __restrict__ out, int r, int hw, int c) {
  const int c4 = c >> 2;
  const long gid = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (gid >= (long)r * c4) return;
  const int cg = (int)(gid % c4);
  const int row = (int)(gid / c4);
  const float4* p = reinterpret_cast<const float4*>(in + (size_t)row * hw * c) + cg;
  float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int i = 0; i < hw; ++i) {
    const float4 x = __ldg(p + (size_t)i * c4);
    s.x = __fadd_rn(s.x, x.x); s.y = __fadd_rn(s.y, x.y); s.z = __fadd_rn(s.z, x.z); s.w = __fadd_rn(s.w, x.w);
  }
  const float d = (float)hw;
  reinterpret_cast<float4*>(out + (size_t)row * c)[cg] =
      make_float4(__fdiv_rn(s.x, d), __fdiv_rn(s.y, d), __fdiv_rn(s.z, d), __fdiv_rn(s.w, d));
}

// ---- crop_and_resize (+ 2x2 max) ---------------------------------------------------------------------------
// correctly-rounded fp32 exp (via fp64) for the two box-size terms: the oracle defines exp the same way
__device__ __forceinline__ float exp_cr(float x) { return (float)exp((double)x); }

__device__ __forceinline__ float lerp_rn(float a, float b, float t) { return __fadd_rn(a, __fmul_rn(__fsub_rn(b, a), t)); }

// One block per (RoI, output row): the first threads compute the sampling geometry of that row once (the per-sample
// divisions and float index math used to be redone by every channel thread and made the kernel ALU bound), then all threads
// stream channels: 4 gathers + lerps per sample, float4 wide.
struct CropSample { int top, bot, lef, rig; float yl, xl; int valid; };

__device__ __forceinline__ float4 sample4(const float* __restrict__ feat, int fw, int c, int cg, const CropSample& s) {
  if (!s.valid) return make_float4(0.f, 0.f, 0.f, 0.f);
  const float4 tl = __ldg(reinterpret_cast<const float4*>(feat + ((size_t)s.top * fw + s.lef) * c) + cg);
  const float4 tr = __ldg(reinterpret_cast<const float4*>(feat + ((size_t)s.top * fw + s.rig) * c) + cg);
  const float4 bl = __ldg(reinterpret_cast<const float4*>(feat + ((size_t)s.bot * fw + s.lef) * c) + cg);
  const float4 br = __ldg(reinterpret_cast<const float4*>(feat + ((size_t)s.bot * fw + s.rig) * c) + cg);
  float4 o;
  o.x = lerp_rn(lerp_rn(tl.x, tr.x, s.xl), lerp_rn(bl.x, br.x, s.xl), s.yl);
  o.y = lerp_rn(lerp_rn(tl.y, tr.y, s.xl), lerp_rn(bl.y, br.y, s.xl), s.yl);
  o.z = lerp_rn(lerp_rn(tl.z, tr.z, s.xl), lerp_rn(bl.z, br.z, s.xl), s.yl);
  o.w = lerp_rn(lerp_rn(tl.w, tr.w, s.xl), lerp_rn(bl.w, br.w, s.xl), s.yl);
  return o;
}

constexpr int CROP_MAX_POOLED = 16;

__global__ void __launch_bounds__(256)
crop_pool_kernel(const float* __restrict__ feat, int batch, int fh, int fw, int c, const float* __restrict__ rois, int r, int pooled,
                 int pre_pool, float* __restrict__ out) {
  __shared__ CropSample smp[CROP_MAX_POOLED * 4];           // [px][dy*2+dx] (one entry per px when !pre_pool)
  const int ri = blockIdx.x / pooled, py = blockIdx.x % pooled;
  // crop_and_resize's box_ind = rois[:, 0] (network.py:143): which image of the batch the box is cut from
  const int bi = min(max((int)__ldg(rois + (size_t)ri * 5), 0), batch - 1);
  feat += (size_t)bi * fh * fw * c;
  const int nsub = pre_pool ? 4 : 1;
  if (threadIdx.x < pooled * nsub) {
    const int px = threadIdx.x / nsub, sub = threadIdx.x % nsub;
    const float* roi = rois + (size_t)ri * 5;
    // network.py:146-153: normalise by (dim-1)*16, then crop_and_resize's own un-normalisation -- op by op as the oracle
    const float hh = __fmul_rn(__fsub_rn((float)fh, 1.f), 16.f);
    const float ww = __fmul_rn(__fsub_rn((float)fw, 1.f), 16.f);
    const float x1 = __fdiv_rn(__ldg(roi + 1), ww), y1 = __fdiv_rn(__ldg(roi + 2), hh);
    const float x2 = __fdiv_rn(__ldg(roi + 3), ww), y2 = __fdiv_rn(__ldg(roi + 4), hh);
    const int crop = pre_pool ? 2 * pooled : pooled;
    const float hs = __fdiv_rn(__fmul_rn(__fsub_rn(y2, y1), (float)(fh - 1)), (float)(crop - 1));
    const float ws = __fdiv_rn(__fmul_rn(__fsub_rn(x2, x1), (float)(fw - 1)), (float)(crop - 1));
    const int iy = pre_pool ? 2 * py + (sub >> 1) : py, ix = pre_pool ? 2 * px + (sub & 1) : px;
    const float in_y = __fadd_rn(__fmul_rn(y1, (float)(fh - 1)), __fmul_rn((float)iy, hs));
    const float in_x = __fadd_rn(__fmul_rn(x1, (float)(fw - 1)), __fmul_rn((float)ix, ws));
    CropSample sp;
    sp.valid = !(in_y < 0.f || in_y > (float)(fh - 1) || in_x < 0.f || in_x > (float)(fw - 1));
    const float ty = floorf(in_y), lx = floorf(in_x);
    sp.top = (int)ty; sp.bot = (int)ceilf(in_y); sp.lef = (int)lx; sp.rig = (int)ceilf(in_x);
    sp.yl = __fsub_rn(in_y, ty); sp.xl = __fsub_rn(in_x, lx);
    if (!sp.valid) { sp.top = sp.bot = sp.lef = sp.rig = 0; }
    smp[px * 4 + sub] = sp;
  }
  __syncthreads();
  const int c4 = c >> 2;
  float* orow = out + (size_t)((size_t)ri * pooled + py) * pooled * c;
  for (int i = threadIdx.x; i < pooled * c4; i += blockDim.x) {
    const int px = i / c4, cg = i - px * c4;
    float4 o;
    if (!pre_pool) {
      o = sample4(feat, fw, c, cg, smp[px * 4]);
    } else {
      const float ninf = __int_as_float(0xff800000);
      o = make_float4(ninf, ninf, ninf, ninf);
#pragma unroll
      for (int sub = 0; sub < 4; ++sub) {
        const float4 v = sample4(feat, fw, c, cg, smp[px * 4 + sub]);
        o.x = fmaxf(o.x, v.x); o.y = fmaxf(o.y, v.y); o.z = fmaxf(o.z, v.z); o.w = fmaxf(o.w, v.w);
      }
    }
    reinterpret_cast<float4*>(orow + (size_t)px * c)[cg] = o;
  }
}

// ---- RoIAlign / RoIPool (POOLING_MODE 'align' / 'pool') ------------------------------------------------------
// torchvision.ops.roi_align / roi_pool on NHWC, op by op in fp32 (DESIGN §2 gives the definition the tests pin).
// One block per (RoI, output row) as crop_pool_kernel.
constexpr int ROI_MAX_POOLED = 16;
constexpr int ALIGN_XTAB = 512;     // x-sample entries per pass, (pw, ix) pairs
constexpr int ALIGN_YTAB = 64;      // y-sample entries per pass

// One sample coordinate of one axis: neighbour offsets (row offsets premultiplied by fw), their weights; lo < 0 = the sample
// lies outside [-1, dim] and contributes nothing.
struct __align__(16) AxisSample { int lo, hi; float l, h; };

__device__ __forceinline__ AxisSample align_axis(float v, int dim, int mult) {
  AxisSample s;
  if (v < -1.f || v > (float)dim) { s.lo = s.hi = -1; s.l = s.h = 0.f; return s; }
  if (v <= 0.f) v = 0.f;
  int lo = (int)v, hi;
  if (lo >= dim - 1) { lo = hi = dim - 1; v = (float)lo; } else { hi = lo + 1; }
  s.l = __fsub_rn(v, (float)lo);
  s.h = __fsub_rn(1.f, s.l);
  s.lo = lo * mult; s.hi = hi * mult;
  return s;
}

__device__ __forceinline__ float align_term(float acc, float w1, float w2, float w3, float w4, float v1, float v2, float v3, float v4) {
  return __fadd_rn(acc, __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(w1, v1), __fmul_rn(w2, v2)), __fmul_rn(w3, v3)), __fmul_rn(w4, v4)));
}

// The sample geometry is separable: a y table over (iy) and an x table over (pw, ix), built by the block once per pass; every
// thread then streams float4 channel groups through the samples in (iy, ix) order.  A grid too large for the tables is walked
// in passes that keep that order (whole rows of iy while every ix fits, else one iy row and a range of ix per pass), the
// running sum carried between passes in the output element itself (an fp32 store and reload is exact).
__global__ void __launch_bounds__(256)
roi_align_kernel(const float* __restrict__ feat, int batch, int fh, int fw, int c, const float* __restrict__ rois, int pooled,
                 float scale, int sampling_ratio, int aligned, float* __restrict__ out) {
  __shared__ AxisSample ytab[ALIGN_YTAB];
  __shared__ AxisSample xtab[ALIGN_XTAB];
  const int ri = blockIdx.x / pooled, ph = blockIdx.x % pooled;
  const float* roi = rois + (size_t)ri * 5;
  const int bi = min(max((int)__ldg(roi), 0), batch - 1);
  feat += (size_t)bi * fh * fw * c;
  const float off = aligned ? 0.5f : 0.f;
  const float sx = __fsub_rn(__fmul_rn(__ldg(roi + 1), scale), off), sy = __fsub_rn(__fmul_rn(__ldg(roi + 2), scale), off);
  const float ex = __fsub_rn(__fmul_rn(__ldg(roi + 3), scale), off), ey = __fsub_rn(__fmul_rn(__ldg(roi + 4), scale), off);
  float rw = __fsub_rn(ex, sx), rh = __fsub_rn(ey, sy);
  if (!aligned) { rw = rw < 1.f ? 1.f : rw; rh = rh < 1.f ? 1.f : rh; }    // std::max(v, 1): a NaN stays NaN
  const float bw = __fdiv_rn(rw, (float)pooled), bh = __fdiv_rn(rh, (float)pooled);
  const int gw = sampling_ratio > 0 ? sampling_ratio : (int)ceilf(bw);
  const int gh = sampling_ratio > 0 ? sampling_ratio : (int)ceilf(bh);
  const float cnt = (float)max(gh * gw, 1);
  const float y0 = __fadd_rn(sy, __fmul_rn((float)ph, bh));
  const int c4 = c >> 2, items = pooled * c4;
  float* orow = out + (size_t)blockIdx.x * pooled * c;
  if (gh <= 0 || gw <= 0) {                       // no sample: 0 / count
    for (int i = threadIdx.x; i < items; i += blockDim.x) reinterpret_cast<float4*>(orow)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    return;
  }
  const int xcap = max(ALIGN_XTAB / pooled, 1);
  const bool xsplit = gw > xcap;
  const int ystep = xsplit ? 1 : ALIGN_YTAB, xstep = xsplit ? xcap : gw;
  for (int iy0 = 0; iy0 < gh; iy0 += ystep) {
    for (int ix0 = 0; ix0 < gw; ix0 += xstep) {
      const int ny = min(ystep, gh - iy0), nx = min(xstep, gw - ix0);
      const bool first = iy0 == 0 && ix0 == 0, last = iy0 + ny == gh && ix0 + nx == gw;
      __syncthreads();                            // the previous pass's readers are done with the tables
      for (int k = threadIdx.x; k < ny; k += blockDim.x) {
        const float y = __fadd_rn(y0, __fdiv_rn(__fmul_rn(__fadd_rn((float)(iy0 + k), 0.5f), bh), (float)gh));
        ytab[k] = align_axis(y, fh, fw);
      }
      for (int k = threadIdx.x; k < pooled * nx; k += blockDim.x) {
        const int pw = k / nx, ix = ix0 + k - pw * nx;
        const float x = __fadd_rn(__fadd_rn(sx, __fmul_rn((float)pw, bw)), __fdiv_rn(__fmul_rn(__fadd_rn((float)ix, 0.5f), bw), (float)gw));
        xtab[k] = align_axis(x, fw, 1);
      }
      __syncthreads();
      for (int i = threadIdx.x; i < items; i += blockDim.x) {
        const int pw = i / c4, cg = i - pw * c4;
        float4 acc = first ? make_float4(0.f, 0.f, 0.f, 0.f) : reinterpret_cast<const float4*>(orow)[i];
        const AxisSample* xs = xtab + pw * nx;
        for (int iy = 0; iy < ny; ++iy) {
          const AxisSample ys = ytab[iy];
          if (ys.lo < 0) continue;
          const float4* rlo = reinterpret_cast<const float4*>(feat + (size_t)ys.lo * c) + cg;
          const float4* rhi = reinterpret_cast<const float4*>(feat + (size_t)ys.hi * c) + cg;
          for (int ix = 0; ix < nx; ++ix) {
            const AxisSample xv = xs[ix];
            if (xv.lo < 0) continue;
            const float w1 = __fmul_rn(ys.h, xv.h), w2 = __fmul_rn(ys.h, xv.l), w3 = __fmul_rn(ys.l, xv.h), w4 = __fmul_rn(ys.l, xv.l);
            const float4 v1 = __ldg(rlo + (size_t)xv.lo * c4), v2 = __ldg(rlo + (size_t)xv.hi * c4);
            const float4 v3 = __ldg(rhi + (size_t)xv.lo * c4), v4 = __ldg(rhi + (size_t)xv.hi * c4);
            acc.x = align_term(acc.x, w1, w2, w3, w4, v1.x, v2.x, v3.x, v4.x);
            acc.y = align_term(acc.y, w1, w2, w3, w4, v1.y, v2.y, v3.y, v4.y);
            acc.z = align_term(acc.z, w1, w2, w3, w4, v1.z, v2.z, v3.z, v4.z);
            acc.w = align_term(acc.w, w1, w2, w3, w4, v1.w, v2.w, v3.w, v4.w);
          }
        }
        if (last) acc = make_float4(__fdiv_rn(acc.x, cnt), __fdiv_rn(acc.y, cnt), __fdiv_rn(acc.z, cnt), __fdiv_rn(acc.w, cnt));
        reinterpret_cast<float4*>(orow)[i] = acc;
      }
    }
  }
}

// Max over the bin's cells by '>' from -FLT_MAX in (row, column) order: a NaN never wins, an all-NaN bin gives -FLT_MAX,
// an empty bin gives 0 (torchvision's roi_pool).
__global__ void __launch_bounds__(256)
roi_pool_kernel(const float* __restrict__ feat, int batch, int fh, int fw, int c, const float* __restrict__ rois, int pooled,
                float scale, float* __restrict__ out) {
  const int ri = blockIdx.x / pooled, ph = blockIdx.x % pooled;
  const float* roi = rois + (size_t)ri * 5;
  const int bi = min(max((int)__ldg(roi), 0), batch - 1);
  feat += (size_t)bi * fh * fw * c;
  const int sx = (int)roundf(__fmul_rn(__ldg(roi + 1), scale)), sy = (int)roundf(__fmul_rn(__ldg(roi + 2), scale));
  const int ex = (int)roundf(__fmul_rn(__ldg(roi + 3), scale)), ey = (int)roundf(__fmul_rn(__ldg(roi + 4), scale));
  const float bw = __fdiv_rn((float)max(ex - sx + 1, 1), (float)pooled), bh = __fdiv_rn((float)max(ey - sy + 1, 1), (float)pooled);
  const int h0 = min(max((int)floorf(__fmul_rn((float)ph, bh)) + sy, 0), fh);
  const int h1 = min(max((int)ceilf(__fmul_rn((float)(ph + 1), bh)) + sy, 0), fh);
  const int c4 = c >> 2;
  float* orow = out + (size_t)blockIdx.x * pooled * c;
  for (int i = threadIdx.x; i < pooled * c4; i += blockDim.x) {
    const int pw = i / c4, cg = i - pw * c4;
    const int w0 = min(max((int)floorf(__fmul_rn((float)pw, bw)) + sx, 0), fw);
    const int w1 = min(max((int)ceilf(__fmul_rn((float)(pw + 1), bw)) + sx, 0), fw);
    float4 m;
    if (h1 <= h0 || w1 <= w0) {
      m = make_float4(0.f, 0.f, 0.f, 0.f);
    } else {
      const float lowest = __int_as_float(0xff7fffff);     // -FLT_MAX
      m = make_float4(lowest, lowest, lowest, lowest);
      for (int y = h0; y < h1; ++y) {
        const float4* row = reinterpret_cast<const float4*>(feat + (size_t)y * fw * c) + cg;
        for (int x = w0; x < w1; ++x) {
          const float4 v = __ldg(row + (size_t)x * c4);
          m.x = v.x > m.x ? v.x : m.x; m.y = v.y > m.y ? v.y : m.y; m.z = v.z > m.z ? v.z : m.z; m.w = v.w > m.w ? v.w : m.w;
        }
      }
    }
    reinterpret_cast<float4*>(orow)[i] = m;
  }
}

// ---- RPN decode ---------------------------------------------------------------------------------------------
__global__ void rpn_decode_kernel(const float* __restrict__ rpn, int ld, int delta_col, const float* __restrict__ base, int A, int batch,
                                  int fh, int fw, int feat_stride, float im_h, float im_w, float* __restrict__ scores,
                                  float* __restrict__ props) {
  const int total = batch * fh * fw * A;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int a = i % A, pos = i / A;                    // pos runs over the images of the batch
  const int pin = pos % (fh * fw);
  const int gx = pin % fw, gy = pin / fw;
  const float* row = rpn + (size_t)pos * ld;
  const float bg = __ldg(row + a), fg = __ldg(row + A + a);
  const float m = fmaxf(bg, fg);
  const float e0 = expf(__fsub_rn(bg, m)), e1 = expf(__fsub_rn(fg, m));
  scores[i] = __fdiv_rn(e1, __fadd_rn(e0, e1));
  const float sx = (float)(gx * feat_stride), sy = (float)(gy * feat_stride);
  const float ax1 = __ldg(base + a * 4 + 0) + sx, ay1 = __ldg(base + a * 4 + 1) + sy;
  const float ax2 = __ldg(base + a * 4 + 2) + sx, ay2 = __ldg(base + a * 4 + 3) + sy;
  const float4 d = *reinterpret_cast<const float4*>(row + delta_col + 4 * a);
  const float w = __fadd_rn(__fsub_rn(ax2, ax1), 1.f), h = __fadd_rn(__fsub_rn(ay2, ay1), 1.f);
  const float cx = __fadd_rn(ax1, __fmul_rn(0.5f, w)), cy = __fadd_rn(ay1, __fmul_rn(0.5f, h));
  const float pcx = __fadd_rn(__fmul_rn(d.x, w), cx), pcy = __fadd_rn(__fmul_rn(d.y, h), cy);
  const float pw = __fmul_rn(exp_cr(d.z), w), ph = __fmul_rn(exp_cr(d.w), h);
  const float xmax = __fsub_rn(im_w, 1.f), ymax = __fsub_rn(im_h, 1.f);
  float4 o;
  o.x = fmaxf(fminf(__fsub_rn(pcx, __fmul_rn(0.5f, pw)), xmax), 0.f);
  o.y = fmaxf(fminf(__fsub_rn(pcy, __fmul_rn(0.5f, ph)), ymax), 0.f);
  o.z = fmaxf(fminf(__fadd_rn(pcx, __fmul_rn(0.5f, pw)), xmax), 0.f);
  o.w = fmaxf(fminf(__fadd_rn(pcy, __fmul_rn(0.5f, ph)), ymax), 0.f);
  reinterpret_cast<float4*>(props)[i] = o;
}

// ---- classification tail --------------------------------------------------------------------------------------
// one warp per RoI row: softmax over C logits + de-normalised deltas
__global__ void cls_finish_kernel(const float* __restrict__ head, int ld, int r, int C, float4 stds, float4 means,
                                  float* __restrict__ cls_score, float* __restrict__ cls_prob, float* __restrict__ bbox) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= r) return;
  const float* hr = head + (size_t)row * ld;
  float m = __int_as_float(0xff800000);
  for (int c = lane; c < C; c += 32) m = fmaxf(m, __ldg(hr + c));
  for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  float s = 0.f;
  for (int c = lane; c < C; c += 32) s += expf(__fsub_rn(__ldg(hr + c), m));
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  for (int c = lane; c < C; c += 32) {
    const float x = __ldg(hr + c);
    cls_score[(size_t)row * C + c] = x;
    cls_prob[(size_t)row * C + c] = __fdiv_rn(expf(__fsub_rn(x, m)), s);
  }
  const float sd[4] = {stds.x, stds.y, stds.z, stds.w};
  const float mn[4] = {means.x, means.y, means.z, means.w};
  for (int j = lane; j < 4 * C; j += 32)
    bbox[(size_t)row * 4 * C + j] = __fadd_rn(__fmul_rn(__ldg(hr + C + j), sd[j & 3]), mn[j & 3]);
}

// im_detect tail: thread per (roi, class)
// im_meta [batch][3] = (im_scale, orig_h, orig_w) of every image, read from device memory so that the launch can sit in a
// CUDA graph (r01 passed them by value and had to launch this tail eagerly after the graph)
__global__ void bbox_decode_kernel(const float* __restrict__ rois, const float* __restrict__ deltas, int r, int C, int batch,
                                   const float* __restrict__ im_meta, float* __restrict__ pred) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= r * C) return;
  const int row = i / C;
  const float* roi = rois + (size_t)row * 5;
  const int bi = min(max((int)__ldg(roi), 0), batch - 1);
  const float im_scale = __ldg(im_meta + bi * 3);
  const float ymax = __fsub_rn(__ldg(im_meta + bi * 3 + 1), 1.f), xmax = __fsub_rn(__ldg(im_meta + bi * 3 + 2), 1.f);
  const float x1 = __fdiv_rn(__ldg(roi + 1), im_scale), y1 = __fdiv_rn(__ldg(roi + 2), im_scale);
  const float x2 = __fdiv_rn(__ldg(roi + 3), im_scale), y2 = __fdiv_rn(__ldg(roi + 4), im_scale);
  const float w = __fadd_rn(__fsub_rn(x2, x1), 1.f), h = __fadd_rn(__fsub_rn(y2, y1), 1.f);
  const float cx = __fadd_rn(x1, __fmul_rn(0.5f, w)), cy = __fadd_rn(y1, __fmul_rn(0.5f, h));
  const float4 d = reinterpret_cast<const float4*>(deltas)[i];
  const float pcx = __fadd_rn(__fmul_rn(d.x, w), cx), pcy = __fadd_rn(__fmul_rn(d.y, h), cy);
  const float pw = __fmul_rn(exp_cr(d.z), w), ph = __fmul_rn(exp_cr(d.w), h);
  float4 o;
  o.x = fmaxf(__fsub_rn(pcx, __fmul_rn(0.5f, pw)), 0.f);
  o.y = fmaxf(__fsub_rn(pcy, __fmul_rn(0.5f, ph)), 0.f);
  o.z = fminf(__fadd_rn(pcx, __fmul_rn(0.5f, pw)), xmax);
  o.w = fminf(__fadd_rn(pcy, __fmul_rn(0.5f, ph)), ymax);
  reinterpret_cast<float4*>(pred)[i] = o;
}

// caller boxes (original-image pixels) -> RoI rows (image, x1*s, y1*s, x2*s, y2*s) in blob pixels, thread per (image, row).
// Scale and count are read from device memory, so one captured graph serves every call of the same capacity.  No clipping:
// crop_and_resize extrapolates samples outside the feature map to 0.
__global__ void boxes_to_rois_kernel(const float4* __restrict__ boxes, const int* __restrict__ counts, const float* __restrict__ im_meta,
                                     int batch, int cap, float* __restrict__ rois, int* __restrict__ num_rois) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= batch * cap) return;
  const int b = i / cap, j = i - b * cap;
  const int n = min(max(__ldg(counts + b), 0), cap);
  if (j == 0) num_rois[b] = n;
  float* row = rois + (size_t)i * 5;
  if (j < n) {
    const float s = __ldg(im_meta + b * 3);
    const float4 bx = __ldg(boxes + i);
    row[0] = (float)b; row[1] = __fmul_rn(bx.x, s); row[2] = __fmul_rn(bx.y, s); row[3] = __fmul_rn(bx.z, s); row[4] = __fmul_rn(bx.w, s);
  } else {
    row[0] = row[1] = row[2] = row[3] = row[4] = 0.f;
  }
}

// ---- test-time augmentation: the union of the views' im_detect outputs, ahead of the per-class NMS ------------------------
// The per-view pointers travel inside the kernel's parameter block (__grid_constant__: indexed in place, no local copy), so
// one captured launch serves every call of the same views.
struct AugViews {
  const float* prob[FRCNN_AUG_MAX_VIEWS];    // [batch, rows, C] of the view
  const float4* box[FRCNN_AUG_MAX_VIEWS];    // [batch, rows, C] float4 (x1, y1, x2, y2)
  const int* num[FRCNN_AUG_MAX_VIEWS];       // [batch] valid-row counts
  int rows[FRCNN_AUG_MAX_VIEWS];
  int flip[FRCNN_AUG_MAX_VIEWS];
};

// Thread per (union row, class) of image blockIdx.y; every union row is written exactly once.  View v's valid rows [0, n_v)
// land at [off_v, off_v + n_v), off_v = n_0 + ... + n_{v-1}; the rows past the total are zero.  A mirrored view's boxes are
// un-flipped in original pixels: x1 = (W - x2') - 1, x2 = (W - x1') - 1, two fp32 roundings each, W = im_meta's orig_w.
__global__ void __launch_bounds__(256)
aug_union_kernel(const __grid_constant__ AugViews vw, int nv, int C, int ru, const float* __restrict__ im_meta,
                 float* __restrict__ prob, float4* __restrict__ box, int* __restrict__ num) {
  __shared__ int s_off[FRCNN_AUG_MAX_VIEWS + 1];
  const int b = blockIdx.y;
  if (threadIdx.x == 0) {
    int o = 0;
    for (int v = 0; v < nv; ++v) {
      s_off[v] = o;
      o += min(max(__ldg(vw.num[v] + b), 0), vw.rows[v]);
    }
    s_off[nv] = o;
    if (blockIdx.x == 0) num[b] = o;
  }
  __syncthreads();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= ru * C) return;
  const int u = i / C, c = i - u * C;
  const size_t dst = ((size_t)b * ru + u) * C + c;
  if (u >= s_off[nv]) {
    prob[dst] = 0.f;
    box[dst] = make_float4(0.f, 0.f, 0.f, 0.f);
    return;
  }
  int v = 0;
  while (u >= s_off[v + 1]) ++v;                       // terminates: u < s_off[nv]; views with no rows are stepped over
  const size_t src = ((size_t)b * vw.rows[v] + (u - s_off[v])) * C + c;
  prob[dst] = __ldg(vw.prob[v] + src);
  float4 q = __ldg(vw.box[v] + src);
  if (vw.flip[v]) {
    const float w = __ldg(im_meta + b * 3 + 2);
    const float x1 = __fsub_rn(__fsub_rn(w, q.z), 1.f), x2 = __fsub_rn(__fsub_rn(w, q.x), 1.f);
    q.x = x1;
    q.z = x2;
  }
  box[dst] = q;
}

// ---- image -> blob on the device (SURVEY 8(f) rank 2): mean subtraction + cv2.resize(INTER_LINEAR) restated ----------
// lib/model/test.py:35-36 (float32(pixel) - PIXEL_MEANS, evaluated in double and rounded once, as numpy's in-place
// float32 -= float64 does) followed by OpenCV's float bilinear resize: source coordinate (dx + 0.5) / fx - 0.5 in double,
// floor + fraction in double, clamp; horizontal pass then vertical pass.
// HFLIP: the blob of the mirrored image img[:, ::-1] (test-time augmentation): the same arithmetic on the mirrored source
// grid, whose column sx is the image's column w0 - 1 - sx.
template <bool HFLIP>
__global__ void preprocess_kernel(const unsigned char* __restrict__ img, int h0, int w0, double m0, double m1, double m2,
                                  double inv_fx, double inv_fy, float* __restrict__ blob, int H, int W) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= H * W) return;
  const int dx = i % W, dy = i / W;
  // source coordinate and its fractional part in double, rounded to float once (OpenCV 4.x; measured against cv2 4.13:
  // taking the fraction of the float32 coordinate is off by up to 6e-3 on the blob)
  const double cx = (dx + 0.5) * inv_fx - 0.5, cy = (dy + 0.5) * inv_fy - 0.5;
  int sx = (int)floor(cx);
  float fx = (float)(cx - (double)sx);
  if (sx < 0) { fx = 0.f; sx = 0; }
  if (sx >= w0 - 1) { fx = 0.f; sx = w0 - 1; }
  int sy = (int)floor(cy);
  float fy = (float)(cy - (double)sy);
  if (sy < 0) { fy = 0.f; sy = 0; }
  if (sy >= h0 - 1) { fy = 0.f; sy = h0 - 1; }
  const int sx1 = min(sx + 1, w0 - 1), sy1 = min(sy + 1, h0 - 1);
  const int ix0 = HFLIP ? w0 - 1 - sx : sx, ix1 = HFLIP ? w0 - 1 - sx1 : sx1;
  const float a0 = 1.f - fx, a1 = fx, b0 = 1.f - fy, b1 = fy;
  const double mean[3] = {m0, m1, m2};
  const unsigned char* r0 = img + (size_t)sy * w0 * 3;
  const unsigned char* r1 = img + (size_t)sy1 * w0 * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float v00 = (float)((double)r0[ix0 * 3 + c] - mean[c]), v01 = (float)((double)r0[ix1 * 3 + c] - mean[c]);
    const float v10 = (float)((double)r1[ix0 * 3 + c] - mean[c]), v11 = (float)((double)r1[ix1 * 3 + c] - mean[c]);
    const float t0 = __fadd_rn(__fmul_rn(v00, a0), __fmul_rn(v01, a1));
    const float t1 = __fadd_rn(__fmul_rn(v10, a0), __fmul_rn(v11, a1));
    blob[(size_t)i * 3 + c] = __fadd_rn(__fmul_rn(t0, b0), __fmul_rn(t1, b1));
  }
}

static inline unsigned blocks_for(long total, int threads) { return (unsigned)((total + threads - 1) / threads); }

}  // namespace frcnn

using namespace frcnn;

extern "C" int frcnn_pack_conv_weights(const float* w, void* hi, void* lo, int kh, int kw, int cin, int cout, int wexp, void* stream) {
  FRCNN_REQUIRE(w && hi && lo && kh > 0 && kw > 0 && cin > 0 && cout > 0, "bad argument");
  FRCNN_REQUIRE(wexp >= -100 && wexp <= 100, "pack_conv_weights: wexp=%d out of range", wexp);
  {
    const int ktot = kh * kw * cin;
    const long total = (long)ktot * cout;
    unsigned blocks = blocks_for(total, 256);
    if (blocks > 132 * 16) blocks = 132 * 16;
    pack_weights_f16_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(w, (__half*)hi, (__half*)lo, ktot, cout, ldexpf(1.f, wexp));
    FRCNN_LAUNCH_CHECK();
    return OK;
  }
}

extern "C" int frcnn_pack_conv_weights_tf32(const float* w, float* hi, float* lo, int kh, int kw, int cin, int cout, void* stream) {
  FRCNN_REQUIRE(w && hi && lo && kh > 0 && kw > 0 && cin > 0 && cout > 0, "bad argument");
  const int ktot = kh * kw * cin;
  const long total = (long)ktot * cout;
  unsigned blocks = blocks_for(total, 256);
  if (blocks > 132 * 16) blocks = 132 * 16;
  pack_weights_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(w, hi, lo, ktot, cout);
  FRCNN_LAUNCH_CHECK();
  return OK;
}

extern "C" int frcnn_conv_first(const float* in, const float* w, const float* scale, const float* shift, float* out, int n,
                                int h, int wd, int cout, int k, int stride, int pad_t, int pad_l, int ho, int wo, int act,
                                void* stream) {
  FRCNN_REQUIRE(in && w && out && (cout == 32 || cout == 64), "conv_first: cout must be 32 or 64");
  const int ph = (CF_TH - 1) * stride + k, pw = (CF_TW - 1) * stride + k;
  const size_t smem = ((size_t)k * k * 3 * cout + (size_t)ph * pw * 3) * sizeof(float);
  FRCNN_REQUIRE(smem <= 100 * 1024, "conv_first: %zu B of shared memory needed", smem);
  static size_t attr_smem = 0;
  if (smem > 48 * 1024 && smem > attr_smem) {
    FRCNN_CUDA(cudaFuncSetAttribute(conv_first_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    FRCNN_CUDA(cudaFuncSetAttribute(conv_first_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr_smem = smem;
  }
  const int tiles_x = cdiv(wo, CF_TW), tiles_y = cdiv(ho, CF_TH);
  const unsigned grid = (unsigned)(tiles_x * tiles_y * n);
  if (cout == 64)       // 2 channel groups x 4 pixel blocks of 64 = the 8 warps, two pixels per thread
    conv_first_kernel<2><<<grid, 256, smem, (cudaStream_t)stream>>>(in, w, scale, shift, out, h, wd, cout, k, stride, pad_t, pad_l, ho, wo, act,
                                                                   tiles_x, tiles_y);
  else                  // cout == 32: 8 pixel blocks of 32, one pixel per thread
    conv_first_kernel<1><<<grid, 256, smem, (cudaStream_t)stream>>>(in, w, scale, shift, out, h, wd, cout, k, stride, pad_t, pad_l, ho, wo, act,
                                                                   tiles_x, tiles_y);
  FRCNN_LAUNCH_CHECK();
  return OK;
}

extern "C" int frcnn_depthwise3x3(const float* in, const float* w, const float* scale, const float* shift, float* out, int n,
                                  int h, int wd, int c, int stride, int pad_t, int pad_l, int ho, int wo, int act, void* stream) {
  FRCNN_REQUIRE(in && w && out && c % 4 == 0, "depthwise: c must be a multiple of 4");
  const long total = (long)n * ho * wo * (c / 4);
  depthwise3x3_kernel<<<blocks_for(total, 256), 256, 0, (cudaStream_t)stream>>>(in, w, scale, shift, out, n, h, wd, c, stride,
                                                                              pad_t, pad_l, ho, wo, act);
  FRCNN_LAUNCH_CHECK();
  return OK;
}

extern "C" int frcnn_max_pool(const float* in, float* out, int n, int h, int wd, int c, int k, int stride, int pad_t, int pad_l,
                              int ho, int wo, int pad_is_neg_inf, void* stream) {
  FRCNN_REQUIRE(in && out && c % 4 == 0, "max_pool: c must be a multiple of 4");
  const long total = (long)n * ho * wo * (c / 4);
  max_pool_kernel<<<blocks_for(total, 256), 256, 0, (cudaStream_t)stream>>>(in, out, n, h, wd, c, k, stride, pad_t, pad_l, ho, wo,
                                                                          pad_is_neg_inf);
  FRCNN_LAUNCH_CHECK();
  return OK;
}

extern "C" int frcnn_spatial_mean(const float* in, float* out, int r, int hw, int c, void* stream) {
  FRCNN_REQUIRE(in && out && c % 4 == 0, "spatial_mean: c must be a multiple of 4");
  spatial_mean_kernel<<<blocks_for((long)r * (c / 4), 256), 256, 0, (cudaStream_t)stream>>>(in, out, r, hw, c);
  FRCNN_LAUNCH_CHECK();
  return OK;
}

extern "C" int frcnn_crop_pool(const float* feat, int batch, int fh, int fw, int c, const float* rois, int r, int pooled, int pre_pool,
                               float* out, void* stream) {
  FRCNN_REQUIRE(feat && rois && out && batch > 0 && c % 4 == 0 && pooled > 1 && pooled <= CROP_MAX_POOLED, "crop_pool: bad argument");
  crop_pool_kernel<<<(unsigned)(r * pooled), 256, 0, (cudaStream_t)stream>>>(feat, batch, fh, fw, c, rois, r, pooled, pre_pool, out);
  FRCNN_LAUNCH_CHECK();
  return OK;
}

extern "C" int frcnn_roi_align(const float* feat, int batch, int fh, int fw, int c, const float* rois, int r, int pooled,
                               float spatial_scale, int sampling_ratio, int aligned, float* out, void* stream) {
  FRCNN_REQUIRE(feat && rois && out && batch > 0 && fh > 0 && fw > 0 && c > 0 && c % 4 == 0 && r >= 0 && pooled >= 1 &&
                pooled <= ROI_MAX_POOLED && spatial_scale > 0.f && sampling_ratio >= 0 && sampling_ratio <= FRCNN_ROI_ALIGN_MAX_SAMPLING,
                "roi_align: bad argument");
  if (r == 0) return OK;
  roi_align_kernel<<<(unsigned)(r * pooled), 256, 0, (cudaStream_t)stream>>>(feat, batch, fh, fw, c, rois, pooled, spatial_scale,
                                                                             sampling_ratio, aligned ? 1 : 0, out);
  FRCNN_LAUNCH_CHECK();
  return OK;
}

extern "C" int frcnn_roi_pool(const float* feat, int batch, int fh, int fw, int c, const float* rois, int r, int pooled,
                              float spatial_scale, float* out, void* stream) {
  FRCNN_REQUIRE(feat && rois && out && batch > 0 && fh > 0 && fw > 0 && c > 0 && c % 4 == 0 && r >= 0 && pooled >= 1 &&
                pooled <= ROI_MAX_POOLED && spatial_scale > 0.f, "roi_pool: bad argument");
  if (r == 0) return OK;
  roi_pool_kernel<<<(unsigned)(r * pooled), 256, 0, (cudaStream_t)stream>>>(feat, batch, fh, fw, c, rois, pooled, spatial_scale, out);
  FRCNN_LAUNCH_CHECK();
  return OK;
}

extern "C" int frcnn_rpn_decode(const float* rpn_out, int ld, int delta_col, const float* base_anchors, int num_anchors, int batch, int fh,
                                int fw, int feat_stride, float im_h, float im_w, float* scores, float* props, void* stream) {
  FRCNN_REQUIRE(rpn_out && base_anchors && scores && props && batch > 0, "rpn_decode: bad argument");
  FRCNN_REQUIRE(delta_col >= 2 * num_anchors && ld >= delta_col + 4 * num_anchors && (ld % 4) == 0 && (delta_col % 4) == 0,
                "rpn_decode: ld/delta_col alignment");
  const long total = (long)batch * fh * fw * num_anchors;
  rpn_decode_kernel<<<blocks_for(total, 256), 256, 0, (cudaStream_t)stream>>>(rpn_out, ld, delta_col, base_anchors, num_anchors, batch, fh, fw,
                                                                            feat_stride, im_h, im_w, scores, props);
  FRCNN_LAUNCH_CHECK();
  return OK;
}

extern "C" int frcnn_cls_finish(const float* head_out, int ld, int r, int num_classes, const float* stds4, const float* means4,
                                float* cls_score, float* cls_prob, float* bbox_pred, void* stream) {
  FRCNN_REQUIRE(head_out && stds4 && means4 && cls_score && cls_prob && bbox_pred, "cls_finish: null pointer");
  const float4 sd = make_float4(stds4[0], stds4[1], stds4[2], stds4[3]);
  const float4 mn = make_float4(means4[0], means4[1], means4[2], means4[3]);
  cls_finish_kernel<<<blocks_for((long)r * 32, 256), 256, 0, (cudaStream_t)stream>>>(head_out, ld, r, num_classes, sd, mn, cls_score,
                                                                                   cls_prob, bbox_pred);
  FRCNN_LAUNCH_CHECK();
  return OK;
}

extern "C" int frcnn_bbox_decode(const float* rois, const float* bbox_pred, int r, int num_classes, int batch, const float* im_meta_dev,
                                 float* pred_boxes, void* stream) {
  FRCNN_REQUIRE(rois && bbox_pred && pred_boxes && im_meta_dev && batch > 0, "bbox_decode: bad argument");
  FRCNN_REQUIRE((long long)r * num_classes <= INT_MAX, "bbox_decode: r*C = %lld does not fit in int", (long long)r * num_classes);
  bbox_decode_kernel<<<blocks_for((long)r * num_classes, 256), 256, 0, (cudaStream_t)stream>>>(rois, bbox_pred, r, num_classes, batch,
                                                                                             im_meta_dev, pred_boxes);
  FRCNN_LAUNCH_CHECK();
  return OK;
}

extern "C" int frcnn_boxes_to_rois(const float* boxes, const int* counts, const float* im_meta_dev, int batch, int cap, float* rois,
                                   int* num_rois, void* stream) {
  FRCNN_REQUIRE(boxes && counts && im_meta_dev && rois && num_rois, "boxes_to_rois: null pointer");
  FRCNN_REQUIRE(batch > 0 && cap > 0 && ((uintptr_t)boxes & 15) == 0, "boxes_to_rois: batch>0, cap>0 and 16-byte aligned boxes required");
  boxes_to_rois_kernel<<<blocks_for((long)batch * cap, 256), 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const float4*>(boxes), counts,
                                                                                           im_meta_dev, batch, cap, rois, num_rois);
  FRCNN_LAUNCH_CHECK();
  return OK;
}

template <bool HFLIP>
static int preprocess(const unsigned char* img_dev, int h0, int w0, const double* means3, double fx, double fy, float* blob_dev, int H,
                      int W, void* stream) {
  FRCNN_REQUIRE(img_dev && means3 && blob_dev && h0 > 0 && w0 > 0 && H > 0 && W > 0 && fx > 0 && fy > 0, "preprocess: bad argument");
  preprocess_kernel<HFLIP><<<blocks_for((long)H * W, 256), 256, 0, (cudaStream_t)stream>>>(img_dev, h0, w0, means3[0], means3[1], means3[2],
                                                                                         1.0 / fx, 1.0 / fy, blob_dev, H, W);
  FRCNN_LAUNCH_CHECK();
  return OK;
}

extern "C" int frcnn_preprocess(const unsigned char* img_dev, int h0, int w0, const double* means3, double fx, double fy,
                                float* blob_dev, int H, int W, void* stream) {
  return preprocess<false>(img_dev, h0, w0, means3, fx, fy, blob_dev, H, W, stream);
}

extern "C" int frcnn_preprocess_hflip(const unsigned char* img_dev, int h0, int w0, const double* means3, double fx, double fy,
                                      float* blob_dev, int H, int W, void* stream) {
  return preprocess<true>(img_dev, h0, w0, means3, fx, fy, blob_dev, H, W, stream);
}

extern "C" int frcnn_aug_union(const float* const* cls_prob_views, const float* const* pred_boxes_views, const int* const* num_rois_views,
                               const int* rois_per_view, const int* flip_views, int num_views, int batch, int num_classes,
                               const float* im_meta_dev, float* cls_prob_dev, float* pred_boxes_dev, int* num_rois_dev, void* stream) {
  FRCNN_REQUIRE(cls_prob_views && pred_boxes_views && num_rois_views && rois_per_view && flip_views && im_meta_dev && cls_prob_dev &&
                    pred_boxes_dev && num_rois_dev, "aug_union: null pointer");
  FRCNN_REQUIRE(num_views > 0 && batch > 0 && num_classes > 0, "aug_union: num_views>0, batch>0, num_classes>0 required");
  if (num_views > FRCNN_AUG_MAX_VIEWS) { set_error("aug_union: %d views > capacity %d", num_views, FRCNN_AUG_MAX_VIEWS); return ERR_CAPACITY; }
  FRCNN_REQUIRE(((uintptr_t)pred_boxes_dev & 15) == 0, "aug_union: pred_boxes_dev must be 16-byte aligned");
  AugViews vw = {};
  long ru = 0;
  for (int v = 0; v < num_views; ++v) {
    FRCNN_REQUIRE(cls_prob_views[v] && pred_boxes_views[v] && num_rois_views[v], "aug_union: null pointer of view %d", v);
    FRCNN_REQUIRE(((uintptr_t)pred_boxes_views[v] & 15) == 0, "aug_union: pred_boxes of view %d must be 16-byte aligned", v);
    FRCNN_REQUIRE(rois_per_view[v] > 0 && (flip_views[v] == 0 || flip_views[v] == 1), "aug_union: view %d: rows > 0, flip 0 or 1 required", v);
    vw.prob[v] = cls_prob_views[v];
    vw.box[v] = reinterpret_cast<const float4*>(pred_boxes_views[v]);
    vw.num[v] = num_rois_views[v];
    vw.rows[v] = rois_per_view[v];
    vw.flip[v] = flip_views[v];
    ru += rois_per_view[v];
  }
  FRCNN_REQUIRE(ru * num_classes < (1l << 31), "aug_union: %ld union rows x %d classes too large", ru, num_classes);
  const dim3 grid(blocks_for(ru * num_classes, 256), (unsigned)batch);
  aug_union_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(vw, num_views, num_classes, (int)ru, im_meta_dev, cls_prob_dev,
                                                           reinterpret_cast<float4*>(pred_boxes_dev), num_rois_dev);
  FRCNN_LAUNCH_CHECK();
  return OK;
}
