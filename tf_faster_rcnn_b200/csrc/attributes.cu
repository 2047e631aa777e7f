// Attribute head of the bottom-up regions (frcnn_regions_attr_embed, frcnn_attr_finish; the definition is in
// include/frcnn_b200.h).  The two FCs between these launches run on the conv kernel (frcnn_conv_plan_*).
#include <math.h>
#include <climits>
#include "common.cuh"
#include "../../include/frcnn_b200.h"

namespace frcnn {

constexpr int ATTR_THREADS = 256;            // 8 warps, one row each
constexpr int ATTR_MAX_COLS = 4096;          // classes / attributes per row

// numpy's argmax over one row, merged across a warp: the first NaN column if the row holds one (nan_col), else the first
// column holding the maximum (col, val).  Each lane walks its columns in ascending order and keeps the first it saw, so the
// merge only has to prefer the lower column on ties.
struct ArgMax {
  float val;
  int col;      // INT_MAX: no non-NaN column seen
  float nan_val;
  int nan_col;  // INT_MAX: no NaN seen
};

__device__ __forceinline__ void argmax_add(ArgMax& a, float v, int c) {
  if (isnan(v)) {
    if (a.nan_col == INT_MAX) { a.nan_col = c; a.nan_val = v; }
  } else if (a.col == INT_MAX || v > a.val) {
    a.val = v; a.col = c;
  }
}

__device__ __forceinline__ void argmax_warp(ArgMax& a) {
  for (int o = 16; o; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, a.val, o);
    const int oc = __shfl_xor_sync(0xffffffffu, a.col, o);
    const float onv = __shfl_xor_sync(0xffffffffu, a.nan_val, o);
    const int onc = __shfl_xor_sync(0xffffffffu, a.nan_col, o);
    if (oc != INT_MAX && (a.col == INT_MAX || ov > a.val || (ov == a.val && oc < a.col))) { a.val = ov; a.col = oc; }
    if (onc < a.nan_col) { a.nan_col = onc; a.nan_val = onv; }
  }
}

// one warp per region row (b, k) of [batch, M]: argmax of the RoI's class logits (background included), then its embedding row
__global__ void __launch_bounds__(ATTR_THREADS)
regions_attr_embed_kernel(const float* __restrict__ cls_score, int r, int C, const int* __restrict__ index, const int* __restrict__ count,
                          int batch, int M, const float4* __restrict__ table, int E4, float4* __restrict__ emb) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= batch * M) return;
  const int b = row / M, k = row - b * M;
  const int n = min(max(__ldg(count + b), 0), M);
  const int i = k < n ? __ldg(index + row) : -1;
  float4* out = emb + (size_t)row * E4;
  if (i < 0 || i >= r) {
    for (int j = lane; j < E4; j += 32) out[j] = make_float4(0.f, 0.f, 0.f, 0.f);
    return;
  }
  const float* s = cls_score + ((size_t)b * r + i) * C;
  ArgMax a{0.f, INT_MAX, 0.f, INT_MAX};
  for (int c = lane; c < C; c += 32) argmax_add(a, __ldg(s + c), c);
  argmax_warp(a);
  const int c = a.nan_col != INT_MAX ? a.nan_col : a.col;
  const float4* src = table + (size_t)c * E4;
  for (int j = lane; j < E4; j += 32) out[j] = __ldg(src + j);
}

// one warp per region row: softmax over the A attribute logits with cls_finish_kernel's arithmetic (max, expf of the rounded
// difference, lane sums strided over the row then 5 xor shuffles, one rounded division), then numpy's argmax over columns 1..A-1
// of the probabilities just computed
__global__ void __launch_bounds__(ATTR_THREADS)
attr_finish_kernel(const float* __restrict__ score, int ld, int A, const int* __restrict__ count, int batch, int M,
                   float* __restrict__ prob, int* __restrict__ attr, float* __restrict__ conf) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= batch * M) return;
  const int b = row / M, k = row - b * M;
  float* p = prob + (size_t)row * A;
  if (k >= min(max(__ldg(count + b), 0), M)) {
    for (int c = lane; c < A; c += 32) p[c] = 0.f;
    if (lane == 0) { attr[row] = -1; conf[row] = 0.f; }
    return;
  }
  const float* x = score + (size_t)row * ld;
  float m = __int_as_float(0xff800000);
  for (int c = lane; c < A; c += 32) m = fmaxf(m, __ldg(x + c));
  for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  float s = 0.f;
  for (int c = lane; c < A; c += 32) s += expf(__fsub_rn(__ldg(x + c), m));
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  ArgMax a{0.f, INT_MAX, 0.f, INT_MAX};
  for (int c = lane; c < A; c += 32) {
    const float v = __fdiv_rn(expf(__fsub_rn(__ldg(x + c), m)), s);
    p[c] = v;
    if (c > 0) argmax_add(a, v, c);
  }
  argmax_warp(a);
  if (lane == 0) {
    const bool nan = a.nan_col != INT_MAX;
    attr[row] = nan ? a.nan_col : a.col;
    conf[row] = nan ? a.nan_val : a.val;
  }
}

static inline unsigned warp_blocks(int rows) { return (unsigned)(((long)rows * 32 + ATTR_THREADS - 1) / ATTR_THREADS); }

}  // namespace frcnn

using namespace frcnn;

extern "C" int frcnn_regions_attr_embed(const float* cls_score, int r, int batch, int num_classes, const int* index_dev,
                                        const int* count_dev, int max_regions, const float* embedding, int embed_dim, float* emb_out,
                                        void* stream) {
  FRCNN_REQUIRE(cls_score && index_dev && count_dev && embedding && emb_out, "regions_attr_embed: null pointer");
  FRCNN_REQUIRE(num_classes >= 2 && num_classes <= ATTR_MAX_COLS, "regions_attr_embed: num_classes %d outside [2, %d]", num_classes,
                ATTR_MAX_COLS);
  FRCNN_REQUIRE(batch >= 1 && max_regions >= 1 && r >= max_regions, "regions_attr_embed: need batch >= 1 and 1 <= max_regions <= r, "
                "got batch %d, max_regions %d, r %d", batch, max_regions, r);
  FRCNN_REQUIRE((long long)batch * max_regions <= INT_MAX / 32, "regions_attr_embed: %d x %d region rows too many", batch, max_regions);
  FRCNN_REQUIRE(embed_dim >= 4 && embed_dim % 4 == 0, "regions_attr_embed: embed_dim %d must be a positive multiple of 4", embed_dim);
  FRCNN_REQUIRE((((uintptr_t)embedding | (uintptr_t)emb_out) & 15) == 0, "regions_attr_embed: embedding and emb_out must be 16-byte aligned");
  regions_attr_embed_kernel<<<warp_blocks(batch * max_regions), ATTR_THREADS, 0, (cudaStream_t)stream>>>(
      cls_score, r, num_classes, index_dev, count_dev, batch, max_regions, reinterpret_cast<const float4*>(embedding), embed_dim / 4,
      reinterpret_cast<float4*>(emb_out));
  FRCNN_LAUNCH_CHECK();
  return OK;
}

extern "C" int frcnn_attr_finish(const float* score, int ld, int batch, int max_regions, int num_attributes, const int* count_dev,
                                 float* attr_prob, int* attributes, float* attr_conf, void* stream) {
  FRCNN_REQUIRE(score && count_dev && attr_prob && attributes && attr_conf, "attr_finish: null pointer");
  FRCNN_REQUIRE(num_attributes >= 2 && num_attributes <= ATTR_MAX_COLS, "attr_finish: num_attributes %d outside [2, %d]", num_attributes,
                ATTR_MAX_COLS);
  FRCNN_REQUIRE(batch >= 1 && max_regions >= 1, "attr_finish: need batch >= 1 and max_regions >= 1, got %d, %d", batch, max_regions);
  FRCNN_REQUIRE((long long)batch * max_regions <= INT_MAX / 32, "attr_finish: %d x %d region rows too many", batch, max_regions);
  FRCNN_REQUIRE(ld >= num_attributes, "attr_finish: ld %d < num_attributes %d", ld, num_attributes);
  FRCNN_REQUIRE((((uintptr_t)score | (uintptr_t)attr_prob | (uintptr_t)attr_conf | (uintptr_t)attributes | (uintptr_t)count_dev) & 3) == 0,
                "attr_finish: buffers must be 4-byte aligned");
  attr_finish_kernel<<<warp_blocks(batch * max_regions), ATTR_THREADS, 0, (cudaStream_t)stream>>>(
      score, ld, num_attributes, count_dev, batch, max_regions, attr_prob, attributes, attr_conf);
  FRCNN_LAUNCH_CHECK();
  return OK;
}
