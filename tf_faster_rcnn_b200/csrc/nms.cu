// Both NMS passes of the TEST path + the score sort, for sm_90a.
//   RPN stage   : proposal_layer_tf / proposal_layer / proposal_top_layer (lib/layer_utils/proposal_layer.py:16-83,
//                 proposal_top_layer.py:58-85)                                   -> frcnn_proposals
//   final stage : per-class NMS + max_per_image cap (lib/model/test.py:162-180) -> frcnn_detect_post
//   `_nms` ABI  : lib/nms/gpu_nms.hpp:1-2                                        -> frcnn_nms_host
//
// Algorithm (replaces nms_kernel.cu's N x N/64 bitmask + host sweep, which is O(N^2) work and memory even
// though at most post_nms_top_n boxes survive): candidates are walked in priority order in windows of 1024.
// Per round the CTA (a) tests every candidate of the window against the <=K boxes already kept (kept set in shared
// memory) and compacts the survivors, (b) builds the <=256x256 suppression bitmask among them, (c) one thread resolves
// it sequentially with 4 x 64-bit words; survivors are appended to the kept set.  The walk stops as soon as
// max_out boxes are kept, so the RPN stage touches only the first few thousand of the 17k-50k anchors.
// IoU arithmetic is the oracle's op-by-op fp32 sequence (__f*_rn: no FMA contraction) for all three predicate
// variants (flags), so survivor indices are bit-exact.
#include <cfloat>
#include <climits>

#include "common.cuh"
#include "../../include/frcnn_b200.h"

namespace frcnn {

constexpr int NMS_THREADS = 1024;
constexpr int CHUNK = 256;

__device__ __forceinline__ float box_area(const float4 b, unsigned flags) {
  if (flags & FRCNN_NMS_PLUS_ONE) return __fmul_rn(__fadd_rn(__fsub_rn(b.z, b.x), 1.f), __fadd_rn(__fsub_rn(b.w, b.y), 1.f));
  return __fmul_rn(__fsub_rn(b.z, b.x), __fsub_rn(b.w, b.y));
}

// TF normalises corners with min/max first (boxes are (y1,x1,y2,x2) there; the formula is symmetric in x/y)
__device__ __forceinline__ float4 canon(const float4 b, unsigned flags) {
  if (flags & FRCNN_NMS_PLUS_ONE) return b;
  return make_float4(fminf(b.x, b.z), fminf(b.y, b.w), fmaxf(b.x, b.z), fmaxf(b.y, b.w));
}

__device__ __forceinline__ bool suppresses(const float4 a, float area_a, const float4 b, float area_b, float thr, unsigned flags) {
  float inter;
  if (flags & FRCNN_NMS_PLUS_ONE) {
    const float w = fmaxf(0.f, __fadd_rn(__fsub_rn(fminf(a.z, b.z), fmaxf(a.x, b.x)), 1.f));
    const float h = fmaxf(0.f, __fadd_rn(__fsub_rn(fminf(a.w, b.w), fmaxf(a.y, b.y)), 1.f));
    inter = __fmul_rn(w, h);
  } else {
    if ((flags & FRCNN_NMS_SKIP_DEGENERATE) && (area_a <= 0.f || area_b <= 0.f)) return false;
    const float h = fmaxf(__fsub_rn(fminf(a.w, b.w), fmaxf(a.y, b.y)), 0.f);
    const float w = fmaxf(__fsub_rn(fminf(a.z, b.z), fmaxf(a.x, b.x)), 0.f);
    inter = __fmul_rn(h, w);
  }
  const float ovr = __fdiv_rn(inter, __fsub_rn(__fadd_rn(area_a, area_b), inter));
  return (flags & FRCNN_NMS_INCLUSIVE) ? (ovr >= thr) : (ovr > thr);
}

constexpr int WIDE = 1024;    // candidates filtered against the kept set per round (one per thread)

struct GreedyShared {
  unsigned long long mask[CHUNK][CHUNK / 64];
  float4 cbox[CHUNK];
  float carea[CHUNK];
  int cpos[CHUNK];                 // position (in priority order) of each compacted candidate
  int warp_cnt[WIDE / 32];
  unsigned char chunk_kept[CHUNK];
  int nkept;
  int chunk_nk;
  int n_alive;                     // compacted candidates this round (<= CHUNK)
  int consumed;                    // candidates of the window that are settled after this round
  int tot_alive, last_wn;          // survivors / size of the previous window (drives threads-per-candidate)
};

// CTA-cooperative greedy NMS over `m` candidates given in priority order (blockDim.x == 1024).
//   cand(i) -> float4 box of the i-th candidate;  kept/kept_area: storage for the kept set (shared or global)
//   kept_pos: positions (0..m-1) of survivors.   Number kept is left in sh.nkept (valid after the final barrier).
// Round: (a) a window of up to 1024 candidates is tested against the kept set, one candidate per thread; the survivors are
// compacted in order (at most CHUNK = 256 of them -- the window is cut right after the 256th survivor and the rest is
// re-examined next round), (b) the CHUNK x CHUNK suppression bitmask among the survivors is built, (c) one thread resolves it
// sequentially with 4 x 64-bit words, skipping suppressed candidates with ffs.  With a low keep rate (RPN: most anchors
// overlap something already kept) almost everything dies in (a) and a round settles ~1000 candidates.
template <typename CandFn>
__device__ void block_greedy_nms(CandFn cand, int m, float thr, unsigned flags, int max_out, float4* kept, float* kept_area,
                                 int* kept_pos, GreedyShared& sh) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) { sh.nkept = 0; sh.tot_alive = WIDE; sh.last_wn = WIDE; }
  __syncthreads();
  int base = 0;
  while (base < m) {
    const int nk = sh.nkept;
    if (nk >= max_out) break;
    // threads per candidate: when most of the last window survived (high keep rate) a round can only settle ~256 candidates,
    // so look at 256 with 4 threads each; when few survive, look at 1024 with one thread each.
    const int tpc = (sh.tot_alive * 3 >= sh.last_wn) ? 4 : 1;
    const int wn = min(WIDE / tpc, m - base);
    const int ci = tid / tpc, part = tid % tpc;
    // (a) filter the window against the kept set
    bool dead = false;
    float4 b = make_float4(0.f, 0.f, 0.f, 0.f);
    float ab = 0.f;
    if (ci < wn) {
      b = canon(cand(base + ci), flags);
      ab = box_area(b, flags);
      if (thr >= 0.f)
        for (int k = part; k < nk; k += tpc)
          if (suppresses(kept[k], kept_area[k], b, ab, thr, flags)) { dead = true; break; }
    }
    const unsigned dbal = __ballot_sync(0xffffffffu, dead);
    const bool any_dead = tpc == 1 ? dead : (((dbal >> (lane & ~3)) & 0xFu) != 0u);
    const bool alive = (ci < wn) && part == 0 && !any_dead;       // one representative thread per candidate
    // ordered compaction: exclusive prefix of `alive` over the block
    const unsigned bal = __ballot_sync(0xffffffffu, alive);
    if (lane == 0) sh.warp_cnt[warp] = __popc(bal);
    __syncthreads();
    int before = 0;
    for (int w = 0; w < warp; ++w) before += sh.warp_cnt[w];
    const int idx = before + __popc(bal & ((1u << lane) - 1u));
    if (tid == 0) {
      int tot = 0;
      for (int w = 0; w < WIDE / 32; ++w) tot += sh.warp_cnt[w];
      sh.n_alive = min(tot, CHUNK);
      sh.tot_alive = tot; sh.last_wn = wn;
      if (tot <= CHUNK) sh.consumed = wn;
    }
    if (alive && idx < CHUNK) { sh.cbox[idx] = b; sh.carea[idx] = ab; sh.cpos[idx] = base + ci; }
    if (alive && idx == CHUNK) sh.consumed = ci;           // first survivor that does not fit: the window is cut here
    __syncthreads();
    const int cn = sh.n_alive;
    // (b) suppression bitmask among the survivors: thread (row i, 64-bit word wj); only j > i matters
    if (thr >= 0.f) {
      const int i = tid >> 2, wj = tid & 3;
      if (i < cn) {
        unsigned long long bits = 0ull;
        const float4 a = sh.cbox[i];
        const float aa = sh.carea[i];
        const int j0 = wj * 64;
        for (int j = max(j0, i + 1); j < min(j0 + 64, cn); ++j)
          if (suppresses(a, aa, sh.cbox[j], sh.carea[j], thr, flags)) bits |= 1ull << (j - j0);
        sh.mask[i][wj] = bits;
      }
    }
    __syncthreads();
    // (c) sequential resolve (ffs skips suppressed candidates)
    if (tid == 0) {
      static_assert(CHUNK == 256, "resolve loop is written for 4 x 64-bit words");
      unsigned long long rem[4] = {0ull, 0ull, 0ull, 0ull};
      int k = nk, ck = 0;
#pragma unroll
      for (int w = 0; w < 4; ++w) {
        const int lim = min(64, cn - w * 64);
        if (lim <= 0) break;
        const unsigned long long valid = lim == 64 ? ~0ull : ((1ull << lim) - 1ull);
        unsigned long long todo = ~rem[w] & valid;
        while (todo && k < max_out) {
          const int bit = __ffsll((long long)todo) - 1;
          const int i = w * 64 + bit;
          sh.chunk_kept[ck++] = (unsigned char)i;
          ++k;
          if (thr >= 0.f) {
#pragma unroll
            for (int w2 = 0; w2 < 4; ++w2) if (w2 >= w) rem[w2] |= sh.mask[i][w2];
          }
          todo = (todo & ~rem[w]) & ~((2ull << bit) - 1ull);
        }
      }
      sh.chunk_nk = ck;
    }
    __syncthreads();
    const int ck = sh.chunk_nk;
    if (tid < ck) {
      const int i = sh.chunk_kept[tid];
      kept[nk + tid] = sh.cbox[i];
      kept_area[nk + tid] = sh.carea[i];
      kept_pos[nk + tid] = sh.cpos[i];
    }
    const int consumed = sh.consumed;
    __syncthreads();
    if (tid == 0) sh.nkept = nk + ck;
    base += consumed;
    __syncthreads();
  }
  __syncthreads();
}

// ---- RPN proposal selection ---------------------------------------------------------------------------
constexpr int PROPOSAL_CAP = 1024;   // kept set held in shared memory (post_nms_top_n: 300 / 1000 / 'top' handled separately)

__global__ void __launch_bounds__(NMS_THREADS, 1)
proposals_kernel(const float4* __restrict__ props, const float* __restrict__ scores, const int* __restrict__ order, int n_seg, int m,
                 int max_out, float thr, unsigned flags, float* __restrict__ rois, float* __restrict__ roi_scores,
                 int* __restrict__ keep, int* __restrict__ num) {
  __shared__ GreedyShared sh;
  __shared__ float4 kept[PROPOSAL_CAP];
  __shared__ float kept_area[PROPOSAL_CAP];
  __shared__ int kept_pos[PROPOSAL_CAP];
  // one CTA per image of the batch: segment blockIdx.x of the per-image arrays (order holds segment-local indices)
  const int img = blockIdx.x;
  props += (size_t)img * n_seg; scores += (size_t)img * n_seg; order += (size_t)img * n_seg;
  rois += (size_t)img * max_out * 5; roi_scores += (size_t)img * max_out; keep += (size_t)img * max_out; num += img;
  block_greedy_nms([&](int i) { return __ldg(props + __ldg(order + i)); }, m, thr, flags, max_out, kept, kept_area, kept_pos, sh);
  const int nk = sh.nkept;
  for (int i = threadIdx.x; i < max_out; i += blockDim.x) {
    float* r = rois + (size_t)i * 5;
    if (i < nk) {
      const int src = __ldg(order + kept_pos[i]);
      const float4 b = __ldg(props + src);   // un-normalised original box
      r[0] = (float)img; r[1] = b.x; r[2] = b.y; r[3] = b.z; r[4] = b.w;
      roi_scores[i] = __ldg(scores + src);
      keep[i] = src;
    } else {
      r[0] = r[1] = r[2] = r[3] = r[4] = 0.f;
      roi_scores[i] = 0.f;
      keep[i] = -1;
    }
  }
  if (threadIdx.x == 0) *num = nk;
}

// 'top' mode (no NMS) with more outputs than the shared-memory kept set: plain gather of the first max_out
__global__ void gather_top_kernel(const float4* __restrict__ props, const float* __restrict__ scores, const int* __restrict__ order,
                                  int n_seg, int m, int max_out, float* __restrict__ rois, float* __restrict__ roi_scores,
                                  int* __restrict__ keep, int* __restrict__ num) {
  const int img = blockIdx.y;
  props += (size_t)img * n_seg; scores += (size_t)img * n_seg; order += (size_t)img * n_seg;
  rois += (size_t)img * max_out * 5; roi_scores += (size_t)img * max_out; keep += (size_t)img * max_out; num += img;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) *num = min(m, max_out);
  if (i >= max_out) return;
  float* r = rois + (size_t)i * 5;
  if (i < m) {
    const int src = __ldg(order + i);
    const float4 b = __ldg(props + src);
    r[0] = (float)img; r[1] = b.x; r[2] = b.y; r[3] = b.z; r[4] = b.w;
    roi_scores[i] = __ldg(scores + src);
    keep[i] = src;
  } else {
    r[0] = r[1] = r[2] = r[3] = r[4] = 0.f;
    roi_scores[i] = 0.f;
    keep[i] = -1;
  }
}

// ---- generic sorted-input NMS with the kept set in global memory (the `_nms` compatible path) -----------
__global__ void __launch_bounds__(NMS_THREADS, 1)
nms_sorted_kernel(const float* __restrict__ boxes, int stride, int m, float thr, unsigned flags, int max_out,
                  float4* __restrict__ kept, float* __restrict__ kept_area, int* __restrict__ keep, int* __restrict__ num) {
  __shared__ GreedyShared sh;
  block_greedy_nms([&](int i) { const float* b = boxes + (size_t)i * stride; return make_float4(b[0], b[1], b[2], b[3]); }, m, thr,
                   flags, max_out, kept, kept_area, keep, sh);
  if (threadIdx.x == 0) *num = sh.nkept;
}

// ---- final per-class NMS + cap -----------------------------------------------------------------------------
constexpr int DET_CAP = 1024;       // RoIs per image with the candidate list AND the kept set in shared memory (300 / 1000 proposals)
constexpr int DET_CAP_BIG = 8192;   // TEST.MODE 'top' (RPN_TOP_N = 5000, lib/model/config.py:208): candidates in shared, kept set in global memory

// one CTA per (foreground class, image).  CAP = power of two >= r.  Dynamic shared memory: skey[CAP] | sidx[CAP] and, when
// !GLOBAL_KEPT, kept[CAP] (float4) | kept_area[CAP] | kept_pos[CAP]; with GLOBAL_KEPT those three live in `gws`
// ([batch][C][r] slices, see frcnn_detect_post_workspace_bytes).
template <int CAP, bool GLOBAL_KEPT>
__global__ void __launch_bounds__(NMS_THREADS, 1)
class_nms_kernel(const float* __restrict__ probs, const float4* __restrict__ pred, const int* __restrict__ num_rois, int r, int C,
                 float score_thresh, float nms_thresh, unsigned flags, int* __restrict__ keep, int* __restrict__ keep_cnt,
                 float* __restrict__ keep_score, uint8_t* __restrict__ gws) {
  __shared__ GreedyShared sh;
  __shared__ int s_m;
  extern __shared__ __align__(16) uint8_t cls_dyn[];
  float4* kept; float* kept_area; int* kept_pos; float* skey; int* sidx;
  const int cls = blockIdx.x + 1, img = blockIdx.y;
  if (GLOBAL_KEPT) {
    skey = reinterpret_cast<float*>(cls_dyn); sidx = reinterpret_cast<int*>(skey + CAP);
    const size_t rr = (size_t)((r + 3) & ~3);          // slices stay 16-byte aligned
    uint8_t* slice = gws + ((size_t)img * C + cls) * rr * 24;
    kept = reinterpret_cast<float4*>(slice); kept_area = reinterpret_cast<float*>(slice + rr * 16);
    kept_pos = reinterpret_cast<int*>(slice + rr * 20);
  } else {
    kept = reinterpret_cast<float4*>(cls_dyn); kept_area = reinterpret_cast<float*>(kept + CAP);
    kept_pos = reinterpret_cast<int*>(kept_area + CAP); skey = reinterpret_cast<float*>(kept_pos + CAP); sidx = reinterpret_cast<int*>(skey + CAP);
  }
  probs += (size_t)img * r * C; pred += (size_t)img * r * C;
  keep += (size_t)img * C * r; keep_score += (size_t)img * C * r; keep_cnt += (size_t)img * C;
  const int tid = threadIdx.x;
  const int nr = min(__ldg(num_rois + img), r);
  // candidates: score > thresh (test.py:163); sort key (score desc, index asc); invalid -> -inf at the tail
  if (tid == 0) s_m = 0;
  __syncthreads();
  int mine = 0;
  for (int e = tid; e < CAP; e += NMS_THREADS) {
    float key = __int_as_float(0xff800000);
    if (e < nr) {
      const float s = __ldg(probs + (size_t)e * C + cls);
      if (s > score_thresh) { key = s; ++mine; }
    }
    skey[e] = key; sidx[e] = e;
  }
  if (mine) atomicAdd(&s_m, mine);
  __syncthreads();
  // bitonic sort of CAP (key desc, idx asc)
  for (int k = 2; k <= CAP; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int e = tid; e < CAP; e += NMS_THREADS) {
        const int ixj = e ^ j;
        if (ixj > e) {
          const float a = skey[e], b = skey[ixj];
          const int ia = sidx[e], ib = sidx[ixj];
          const bool a_first = (a > b) || (a == b && ia < ib);   // a precedes b in the final order
          const bool up = (e & k) == 0;
          if (up ? !a_first : a_first) { skey[e] = b; skey[ixj] = a; sidx[e] = ib; sidx[ixj] = ia; }
        }
      }
      __syncthreads();
    }
  }
  const int m = s_m;
  block_greedy_nms([&](int i) { return __ldg(pred + (size_t)sidx[i] * C + cls); }, m, nms_thresh, flags, m, kept, kept_area, kept_pos, sh);
  const int nk = sh.nkept;
  for (int i = tid; i < r; i += blockDim.x) {
    if (i < nk) { const int pos = kept_pos[i]; keep[(size_t)cls * r + i] = sidx[pos]; keep_score[(size_t)cls * r + i] = skey[pos]; }
    else { keep[(size_t)cls * r + i] = -1; keep_score[(size_t)cls * r + i] = 0.f; }
  }
  if (tid == 0) keep_cnt[cls] = nk;
  if (blockIdx.x == 0) {
    for (int i = tid; i < r; i += blockDim.x) { keep[i] = -1; keep_score[i] = 0.f; }
    if (tid == 0) keep_cnt[0] = 0;
  }
}

// single CTA: max_per_image cap + record emission (test.py:173-180).  Every class list is sorted by descending score, so
// (1) count_c(t) = #scores >= t is a binary search per class, (2) the k-th largest kept score overall is found by a bitwise
// search on the fp32 pattern (scores > 0 => unsigned order == float order; 32 rounds of 80 parallel binary searches + a block
// reduction), (3) "keep score >= image_thresh" just truncates each list to count_c(thresh) (ties kept, as the reference).
__device__ __forceinline__ int count_ge(const float* __restrict__ sorted_desc, int n, unsigned tbits) {
  int lo = 0, hi = n;                       // first index whose score < t
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (__float_as_uint(sorted_desc[mid]) >= tbits) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// VOTED: the record box of keep entry (c, j) is vote_box[img][c][j] (box voting) instead of pred[keep[c][j]].
// Thread t holds the classes t, t + 1024, ... (CLS_PER_THREAD of them: C <= MAX_CLASSES); at C <= 1024 that is one class each.
constexpr int MAX_CLASSES = 4096;
constexpr int CLS_PER_THREAD = MAX_CLASSES / NMS_THREADS;

template <bool VOTED>
__global__ void __launch_bounds__(NMS_THREADS, 1)
cap_emit_kernel(const float4* __restrict__ pred, int r, int C, int max_per_image, int max_det, int* __restrict__ keep,
                int* __restrict__ keep_cnt, const float* __restrict__ keep_score, float* __restrict__ det, int* __restrict__ ndet,
                int det_stride, int ndet_stride, const float4* __restrict__ vote_box) {
  __shared__ int s_warp[NMS_THREADS / 32];
  __shared__ int s_total;
  __shared__ int s_off[MAX_CLASSES + 1];
  const int img = blockIdx.x;                       // one CTA per image of the batch
  pred += (size_t)img * r * C; keep += (size_t)img * C * r; keep_cnt += (size_t)img * C; keep_score += (size_t)img * C * r;
  det += (size_t)img * det_stride; ndet += (size_t)img * ndet_stride;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  int my_cnt[CLS_PER_THREAD], new_cnt[CLS_PER_THREAD];
#pragma unroll
  for (int q = 0; q < CLS_PER_THREAD; ++q) {
    const int c = tid + q * NMS_THREADS;
    my_cnt[q] = (c >= 1 && c < C) ? keep_cnt[c] : 0;
    new_cnt[q] = my_cnt[q];
  }
  auto count_mine = [&](unsigned tbits) -> int {
    int n = 0;
#pragma unroll
    for (int q = 0; q < CLS_PER_THREAD; ++q)
      if (my_cnt[q]) n += count_ge(keep_score + (size_t)(tid + q * NMS_THREADS) * r, my_cnt[q], tbits);
    return n;
  };
  auto block_sum = [&](int v) -> int {
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if (lane == 0) s_warp[warp] = v;
    __syncthreads();
    if (tid == 0) { int t = 0; for (int w = 0; w < NMS_THREADS / 32; ++w) t += s_warp[w]; s_total = t; }
    __syncthreads();
    return s_total;
  };
  int mine = 0;
#pragma unroll
  for (int q = 0; q < CLS_PER_THREAD; ++q) mine += my_cnt[q];
  const int total = block_sum(mine);
  if (max_per_image > 0 && total > max_per_image) {
    unsigned t = 0u;                                   // largest pattern with count(score >= t) >= max_per_image
    for (int bit = 31; bit >= 0; --bit) {
      const unsigned cand = t | (1u << bit);
      const int cnt = block_sum(count_mine(cand));
      if (cnt >= max_per_image) t = cand;
    }
#pragma unroll
    for (int q = 0; q < CLS_PER_THREAD; ++q)
      if (my_cnt[q]) new_cnt[q] = count_ge(keep_score + (size_t)(tid + q * NMS_THREADS) * r, my_cnt[q], t);
  }
#pragma unroll
  for (int q = 0; q < CLS_PER_THREAD; ++q) {
    const int c = tid + q * NMS_THREADS;
    if (c >= 1 && c < C) {
      for (int j = new_cnt[q]; j < my_cnt[q]; ++j) keep[(size_t)c * r + j] = -1;
      keep_cnt[c] = new_cnt[q];
    }
  }
  // exclusive prefix of the per-class counts in passes of 1024 classes (warp scan + warp totals), carried across passes
  int carry = 0;
  for (int base = 0; base < C; base += NMS_THREADS) {
    const int c = base + tid, q = base / NMS_THREADS;
    int v = 0;
#pragma unroll
    for (int k = 0; k < CLS_PER_THREAD; ++k) if (k == q && c >= 1 && c < C) v = new_cnt[k];
    int incl = v;
    for (int o = 1; o < 32; o <<= 1) { const int n = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += n; }
    __syncthreads();
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    int before = carry, pass = 0;
    for (int w = 0; w < NMS_THREADS / 32; ++w) { const int s = s_warp[w]; before += w < warp ? s : 0; pass += s; }
    if (c < C) s_off[c] = before + incl - v;
    carry += pass;
  }
  if (tid == 0) { s_off[C] = carry; *ndet = carry; }   // the TRUE count: the host rejects a record set that did not fit (> max_det)
  __syncthreads();
  // records driven by slot: the class of a slot is the last c with s_off[c] <= slot
  const int n = min(carry, max_det);
  for (int slot = tid; slot < n; slot += blockDim.x) {
    int lo = 1, hi = C;
    while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (s_off[mid] <= slot) lo = mid; else hi = mid; }
    const int c = lo, j = slot - s_off[c];
    float4 b;
    if (VOTED) b = __ldg(vote_box + ((size_t)img * C + c) * r + j);
    else b = __ldg(pred + (size_t)keep[(size_t)c * r + j] * C + c);
    float* d = det + (size_t)slot * 6;
    d[0] = b.x; d[1] = b.y; d[2] = b.z; d[3] = b.w;
    d[4] = keep_score[(size_t)c * r + j]; d[5] = (float)c;
  }
}

// ---- Soft-NMS (Bodla et al., ICCV 2017) for the final per-class stage -----------------------------------------------
// Sequential definition (include/frcnn_b200.h, frcnn_soft_nms_host): select the lowest position holding the maximal score,
// swap it to the front, decay every later candidate by it, and replace each overlapped candidate that fell below the prune
// threshold by the last one (the replacement is examined in turn).  The decays of one selection are independent of each other,
// so one iteration is data parallel: decay everything, count the pruned positions, and fill the holes in closed form.  With
// L = i+1, D = #pruned in [L, N) and B = N - D (the new count): survivors below B stay; the k-th pruned position below B
// (ascending) receives the k-th survivor at or above B in DESCENDING position order -- exactly where the swap-with-last loop
// puts it.  A survivor at p >= B knows its rank from the exclusive pruned count E(p): j = (N-1-p) - (D - E(p)).
// Candidates live in shared memory as separate arrays (x1, y1, x2, y2, score, RoI index) plus the hole table; thread t owns
// positions k*T + t.  Barriers per selection: the count, the hole table (only when something was pruned), the argmax.
constexpr int SOFT_THREADS = 256, SOFT_PER = 4;            // r <= DET_CAP
constexpr int SOFT_THREADS_BIG = 1024, SOFT_PER_BIG = 8;   // r <= DET_CAP_BIG
static_assert(SOFT_THREADS * SOFT_PER == DET_CAP && SOFT_THREADS_BIG * SOFT_PER_BIG == DET_CAP_BIG, "soft-NMS capacities");

struct SoftParams { int method; float sigma, nt, thresh; };

constexpr size_t soft_smem_bytes(int cap) { return (size_t)cap * 24 + (size_t)(cap / 2) * 4; }   // at most cap/2 holes

__device__ __forceinline__ float area_plus1(float x1, float y1, float x2, float y2) {
  return __fmul_rn(__fadd_rn(__fsub_rn(x2, x1), 1.f), __fadd_rn(__fsub_rn(y2, y1), 1.f));
}

// Decays s by the selected box t (area ta).  Returns false (s untouched) when the boxes do not overlap.
__device__ __forceinline__ bool soft_decay(float tx1, float ty1, float tx2, float ty2, float ta, float x1, float y1, float x2,
                                           float y2, float& s, const SoftParams& p) {
  const float iw = __fadd_rn(__fsub_rn(fminf(tx2, x2), fmaxf(tx1, x1)), 1.f);
  if (!(iw > 0.f)) return false;
  const float ih = __fadd_rn(__fsub_rn(fminf(ty2, y2), fmaxf(ty1, y1)), 1.f);
  if (!(ih > 0.f)) return false;
  const float inter = __fmul_rn(iw, ih);
  const float ov = __fdiv_rn(inter, __fsub_rn(__fadd_rn(ta, area_plus1(x1, y1, x2, y2)), inter));
  float w;
  if (p.method == FRCNN_SOFT_NMS_GAUSSIAN) w = (float)exp(-(double)__fdiv_rn(__fmul_rn(ov, ov), p.sigma));   // exp_cr
  else if (p.method == FRCNN_SOFT_NMS_LINEAR) w = ov > p.nt ? __fsub_rn(1.f, ov) : 1.f;
  else w = ov > p.nt ? 0.f : 1.f;
  s = __fmul_rn(w, s);
  return true;
}

// Exclusive count of flag[k] over the positions k*T + tid of rows k < rows (rows is block uniform) into ex[k]; returns the
// total.  One barrier; s_cnt [PER * T/32] is read after it, so the caller needs another barrier before the next call.
template <int T, int PER>
__device__ __forceinline__ int block_count_rows(const bool (&flag)[PER], int (&ex)[PER], int rows, int* s_cnt) {
  constexpr int NW = T / 32;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < PER; ++k) {
    if (k < rows) {
      const unsigned bal = __ballot_sync(0xffffffffu, flag[k]);
      ex[k] = __popc(bal & ((1u << lane) - 1u));
      if (lane == 0) s_cnt[k * NW + warp] = __popc(bal);
    }
  }
  __syncthreads();
  int run = 0;
#pragma unroll
  for (int k = 0; k < PER; ++k) {
    if (k < rows) {
      const int v = lane < NW ? s_cnt[k * NW + lane] : 0;
      int inc = v;
#pragma unroll
      for (int o = 1; o < NW; o <<= 1) { const int u = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += u; }
      ex[k] += run + __shfl_sync(0xffffffffu, inc - v, warp);
      run += __shfl_sync(0xffffffffu, inc, NW - 1);
    }
  }
  return run;
}

__device__ __forceinline__ void better_of(float& s, int& pos, float s2, int p2) {
  if (s2 > s || (s2 == s && p2 < pos)) { s = s2; pos = p2; }
}

// The argmax key of score s at position p when `head` is the next selection's first position.  The definition's scan
// (m = head; m = p where s[m] < s[p]) keeps a NaN head and never moves onto a NaN from a number: so a NaN at the head competes
// as +inf (ties go to the lowest position, the head), and any other NaN never wins (better_of's comparisons are false).
__device__ __forceinline__ float scan_key(float s, int p, int head) {
  return (p == head && isnan(s)) ? __int_as_float(0x7f800000) : s;
}

// Position of the block's best (score, position): larger score first, then lower position.  One barrier; every thread gets
// the result.  Threads without a candidate pass (-inf, 0x7fffffff).
template <int T>
__device__ __forceinline__ int block_argmax(float s, int pos, float* s_as, int* s_ap) {
  constexpr int NW = T / 32;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o; o >>= 1) better_of(s, pos, __shfl_xor_sync(0xffffffffu, s, o), __shfl_xor_sync(0xffffffffu, pos, o));
  if (lane == 0) { s_as[warp] = s; s_ap[warp] = pos; }
  __syncthreads();
  s = lane < NW ? s_as[lane] : __int_as_float(0xff800000);
  pos = lane < NW ? s_ap[lane] : 0x7fffffff;
#pragma unroll
  for (int o = 16; o; o >>= 1) better_of(s, pos, __shfl_xor_sync(0xffffffffu, s, o), __shfl_xor_sync(0xffffffffu, pos, o));
  return pos;
}

// CTA-cooperative Soft-NMS over the inputs e < n for which is_cand(e) holds, taken in ascending e (blockDim.x == T).
// box(e) / score(e) read an input; emit(i, e, box, score) is called by thread 0 for the i-th selection.  sm: dynamic shared
// memory of soft_smem_bytes(T * PER).  Returns the number selected (block uniform).
template <int T, int PER, typename CandFn, typename BoxFn, typename ScoreFn, typename EmitFn>
__device__ int block_soft_nms(int n, CandFn is_cand, BoxFn box, ScoreFn score, const SoftParams prm, EmitFn emit, float* sm) {
  constexpr int CAP = T * PER;
  __shared__ int s_cnt[PER * (T / 32)];
  __shared__ float s_as[T / 32];
  __shared__ int s_ap[T / 32];
  float* x1 = sm; float* y1 = sm + CAP; float* x2 = sm + 2 * CAP; float* y2 = sm + 3 * CAP; float* sc = sm + 4 * CAP;
  int* id = reinterpret_cast<int*>(sm + 5 * CAP);
  int* hole = id + CAP;
  const int tid = threadIdx.x;
  const float NEG_INF = __int_as_float(0xff800000);
  bool f[PER];
  int ex[PER];
  // compaction of the candidates, ascending input index
  int rows = (n + T - 1) / T;
#pragma unroll
  for (int k = 0; k < PER; ++k) { const int e = k * T + tid; f[k] = k < rows && e < n && is_cand(e); }
  int N = block_count_rows<T, PER>(f, ex, rows, s_cnt);
  float bs = NEG_INF;
  int bp = 0x7fffffff;
#pragma unroll
  for (int k = 0; k < PER; ++k) {
    if (f[k]) {
      const int e = k * T + tid, p = ex[k];
      const float4 b = box(e);
      const float s = score(e);
      x1[p] = b.x; y1[p] = b.y; x2[p] = b.z; y2[p] = b.w; sc[p] = s; id[p] = e;
      better_of(bs, bp, scan_key(s, p, 0), p);
    }
  }
  int m = block_argmax<T>(bs, bp, s_as, s_ap);
  for (int i = 0; i < N; ++i) {
    // the selection sits at m; position m holds the former a[i] (the swap is applied lazily: its owner reads from i).  A NaN
    // at position i entered the argmax as +inf (scan_key), so the argmax is never empty while i < N; the guard is defensive.
    if (m >= N) m = i;
    const float tx1 = x1[m], ty1 = y1[m], tx2 = x2[m], ty2 = y2[m];
    if (tid == 0) emit(i, id[m], make_float4(tx1, ty1, tx2, ty2), sc[m]);
    const float ta = area_plus1(tx1, ty1, tx2, ty2);
    const int L = i + 1;
    rows = (N + T - 1) / T;
    float ns[PER];
#pragma unroll
    for (int k = 0; k < PER; ++k) {
      const int p = k * T + tid;
      f[k] = false; ns[k] = 0.f;
      if (k < rows && p >= L && p < N) {
        const int src = p == m ? i : p;
        float s = sc[src];
        const bool ov = soft_decay(tx1, ty1, tx2, ty2, ta, x1[src], y1[src], x2[src], y2[src], s, prm);
        ns[k] = s;
        f[k] = ov && s < prm.thresh;
      }
    }
    const int D = block_count_rows<T, PER>(f, ex, rows, s_cnt);
    const int B = N - D;
    bs = NEG_INF; bp = 0x7fffffff;
#pragma unroll
    for (int k = 0; k < PER; ++k) {
      const int p = k * T + tid;
      if (k < rows && p >= L && p < B) {
        if (f[k]) {
          hole[ex[k]] = p;
        } else {                                    // survivor that keeps its position
          sc[p] = ns[k];
          if (p == m && m != i) { x1[p] = x1[i]; y1[p] = y1[i]; x2[p] = x2[i]; y2[p] = y2[i]; id[p] = id[i]; }
          better_of(bs, bp, scan_key(ns[k], p, L), p);
        }
      }
    }
    if (D) {
      __syncthreads();                              // hole table complete
#pragma unroll
      for (int k = 0; k < PER; ++k) {
        const int p = k * T + tid;
        if (k < rows && p >= B && p < N && !f[k]) {  // survivor above the new end: fills a hole
          const int dst = hole[(N - 1 - p) - (D - ex[k])];
          const int src = p == m ? i : p;
          x1[dst] = x1[src]; y1[dst] = y1[src]; x2[dst] = x2[src]; y2[dst] = y2[src]; id[dst] = id[src]; sc[dst] = ns[k];
          better_of(bs, bp, scan_key(ns[k], dst, L), dst);
        }
      }
    }
    N = B;
    m = block_argmax<T>(bs, bp, s_as, s_ap);
  }
  return N;
}

// one CTA per (foreground class, image); the keep / keep_cnt / keep_score conventions of class_nms_kernel
template <int T, int PER>
__global__ void __launch_bounds__(T)
class_soft_nms_kernel(const float* __restrict__ probs, const float4* __restrict__ pred, const int* __restrict__ num_rois, int r, int C,
                      float score_thresh, SoftParams prm, int* __restrict__ keep, int* __restrict__ keep_cnt,
                      float* __restrict__ keep_score) {
  extern __shared__ __align__(16) float soft_dyn[];
  const int cls = blockIdx.x + 1, img = blockIdx.y, tid = threadIdx.x;
  probs += (size_t)img * r * C; pred += (size_t)img * r * C;
  keep += (size_t)img * C * r; keep_score += (size_t)img * C * r; keep_cnt += (size_t)img * C;
  const int nr = min(__ldg(num_rois + img), r);
  int* ck = keep + (size_t)cls * r;
  float* cs = keep_score + (size_t)cls * r;
  const int nk = block_soft_nms<T, PER>(
      nr, [&](int e) { return __ldg(probs + (size_t)e * C + cls) > score_thresh; },
      [&](int e) { return __ldg(pred + (size_t)e * C + cls); }, [&](int e) { return __ldg(probs + (size_t)e * C + cls); }, prm,
      [&](int i, int e, float4, float s) { ck[i] = e; cs[i] = s; }, soft_dyn);
  for (int i = nk + tid; i < r; i += T) { ck[i] = -1; cs[i] = 0.f; }
  if (tid == 0) keep_cnt[cls] = nk;
  if (blockIdx.x == 0) {
    for (int i = tid; i < r; i += T) { keep[i] = -1; keep_score[i] = 0.f; }
    if (tid == 0) keep_cnt[0] = 0;
  }
}

// one CTA: the whole input set (rows of `dim` floats: x1, y1, x2, y2, score, ...) is the candidate list
template <int T, int PER>
__global__ void __launch_bounds__(T)
soft_nms_set_kernel(const float* __restrict__ dets, int n, int dim, SoftParams prm, float* __restrict__ dets_out,
                    int* __restrict__ keep_out, int* __restrict__ num) {
  extern __shared__ __align__(16) float soft_dyn[];
  const int nk = block_soft_nms<T, PER>(
      n, [](int) { return true; },
      [&](int e) { const float* d = dets + (size_t)e * dim; return make_float4(d[0], d[1], d[2], d[3]); },
      [&](int e) { return dets[(size_t)e * dim + 4]; }, prm,
      [&](int i, int e, float4 b, float s) {
        float* o = dets_out + (size_t)i * 5;
        o[0] = b.x; o[1] = b.y; o[2] = b.z; o[3] = b.w; o[4] = s;
        keep_out[i] = e;
      },
      soft_dyn);
  if (threadIdx.x == 0) *num = nk;
}

// ---- box voting (Detectron's TEST.BBOX_VOTE) between the per-class stage and the cap ---------------------------------------
// Definition and operation order: include/frcnn_b200.h (frcnn_box_vote_host).  The candidates are compacted into shared memory
// in ascending input order (x1, y1, x2, y2, score arrays, compacted position p).  One warp votes one top box: lane l visits the
// positions l, l+32, l+64, ... in ascending order and accumulates fp64 partials, then the xor butterfly 16, 8, 4, 2, 1 adds them
// (IEEE addition commutes, so every lane ends with lane 0's bits), and lane 0 forms the outputs.  The fp32 products s*x, ov*s
// and beta*s are exact in fp64, so an FMA contraction of an accumulation gives the same bits as a separate multiply and add.
struct VoteParams { float thresh; int method; float beta; };

constexpr size_t vote_smem_bytes(int cap) { return (size_t)cap * 24; }   // 5 candidate floats; the re-sort: float4 box | score | roi

struct VoteAcc { double s, x1, y1, x2, y2, m0, m1; int n; };

__device__ __forceinline__ void vote_add(VoteAcc& a, float4 t, float ta, float x1, float y1, float x2, float y2, float sc,
                                         const VoteParams& p) {
  const float iw = __fadd_rn(__fsub_rn(fminf(t.z, x2), fmaxf(t.x, x1)), 1.f);
  if (!(iw > 0.f)) return;
  const float ih = __fadd_rn(__fsub_rn(fminf(t.w, y2), fmaxf(t.y, y1)), 1.f);
  if (!(ih > 0.f)) return;
  const float inter = __fmul_rn(iw, ih);
  const float ov = __fdiv_rn(inter, __fsub_rn(__fadd_rn(ta, area_plus1(x1, y1, x2, y2)), inter));
  if (!(ov >= p.thresh)) return;
  const double s = (double)sc;
  a.s += s; a.x1 += s * (double)x1; a.y1 += s * (double)y1; a.x2 += s * (double)x2; a.y2 += s * (double)y2;
  a.n += 1;
  if (p.method == FRCNN_BOX_VOTE_IOU_AVG) {
    a.m0 += (double)ov * s; a.m1 += (double)ov;
  } else if (p.method == FRCNN_BOX_VOTE_GENERALIZED_AVG) {
    a.m0 += exp((double)p.beta * s);
  } else if (p.method == FRCNN_BOX_VOTE_TEMP_AVG) {
    const double q = 1.0 - s, m = fmax(s, q), b = (double)p.beta;
    const double e0 = exp(log(s / m) / b), e1 = exp(log(q / m) / b);
    a.m0 += e0 / (e0 + e1);
  }
}

__device__ __forceinline__ double xor_sum(double v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// n^beta of QUASI_SUM: exact for beta 1 and 2 (n <= 8192), the correctly rounded sqrt for 0.5, else pow
__device__ __forceinline__ double vote_pow(double n, double b) {
  return b == 1.0 ? n : b == 2.0 ? n * n : b == 0.5 ? sqrt(n) : pow(n, b);
}

// The voted box and score of top box t (score ts) from the reduced sums; an empty vote set keeps both, a zero weight sum the box.
__device__ __forceinline__ void vote_finish(const VoteAcc& a, const VoteParams& p, float4& t, float& ts) {
  if (a.n == 0) return;
  if (a.s != 0.0) t = make_float4((float)(a.x1 / a.s), (float)(a.y1 / a.s), (float)(a.x2 / a.s), (float)(a.y2 / a.s));
  const double n = (double)a.n, b = (double)p.beta;
  switch (p.method) {
    case FRCNN_BOX_VOTE_AVG: ts = (float)(a.s / n); break;
    case FRCNN_BOX_VOTE_IOU_AVG: ts = (float)(a.m0 / a.m1); break;
    case FRCNN_BOX_VOTE_GENERALIZED_AVG: ts = (float)(log(a.m0 / n) / b); break;
    case FRCNN_BOX_VOTE_QUASI_SUM: ts = (float)(a.s / vote_pow(n, b)); break;
    case FRCNN_BOX_VOTE_TEMP_AVG: ts = (float)(a.m0 / n); break;
    default: break;                                                   // ID: the NMS / Soft-NMS score
  }
}

// CTA-cooperative voting (blockDim.x == T): candidates are the inputs e < n (n <= T*PER) with is_cand(e), box(e) / score(e);
// top(i, box, score) reads top box i < n_top; out(i, box, score) is called by one lane per top box.  sm: vote_smem_bytes(T*PER).
template <int T, int PER, typename CandFn, typename BoxFn, typename ScoreFn, typename TopFn, typename OutFn>
__device__ void block_vote(int n, CandFn is_cand, BoxFn box, ScoreFn score, int n_top, TopFn top, const VoteParams prm, OutFn out,
                           float* sm) {
  constexpr int CAP = T * PER;
  __shared__ int s_cnt[PER * (T / 32)];
  float* x1 = sm; float* y1 = sm + CAP; float* x2 = sm + 2 * CAP; float* y2 = sm + 3 * CAP; float* sc = sm + 4 * CAP;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  bool f[PER];
  int ex[PER];
  const int rows = (n + T - 1) / T;
#pragma unroll
  for (int k = 0; k < PER; ++k) { const int e = k * T + tid; f[k] = k < rows && e < n && is_cand(e); }
  const int N = block_count_rows<T, PER>(f, ex, rows, s_cnt);
#pragma unroll
  for (int k = 0; k < PER; ++k) {
    if (f[k]) {
      const int e = k * T + tid, p = ex[k];
      const float4 b = box(e);
      x1[p] = b.x; y1[p] = b.y; x2[p] = b.z; y2[p] = b.w; sc[p] = score(e);
    }
  }
  __syncthreads();
  for (int i = warp; i < n_top; i += T / 32) {
    float4 t; float ts;
    top(i, t, ts);
    const float ta = area_plus1(t.x, t.y, t.z, t.w);
    VoteAcc a{0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0};
    for (int p = lane; p < N; p += 32) vote_add(a, t, ta, x1[p], y1[p], x2[p], y2[p], sc[p], prm);
    a.s = xor_sum(a.s); a.x1 = xor_sum(a.x1); a.y1 = xor_sum(a.y1); a.x2 = xor_sum(a.x2); a.y2 = xor_sum(a.y2);
    if (prm.method == FRCNN_BOX_VOTE_IOU_AVG || prm.method == FRCNN_BOX_VOTE_GENERALIZED_AVG || prm.method == FRCNN_BOX_VOTE_TEMP_AVG)
      a.m0 = xor_sum(a.m0);
    if (prm.method == FRCNN_BOX_VOTE_IOU_AVG) a.m1 = xor_sum(a.m1);
#pragma unroll
    for (int o = 16; o; o >>= 1) a.n += __shfl_xor_sync(0xffffffffu, a.n, o);
    if (lane == 0) {
      vote_finish(a, prm, t, ts);
      out(i, t, ts);
    }
  }
}

// one CTA per (foreground class, image), after the per-class stage: votes the class's kept list keep / keep_score [0, keep_cnt)
// against the stage's candidates (score > score_thresh, ascending RoI order, original scores), writes vote_box, and for a
// score-changing method overwrites keep_score and re-sorts keep / keep_score / vote_box stably by descending voted score.
template <int T, int PER>
__global__ void __launch_bounds__(T)
class_vote_kernel(const float* __restrict__ probs, const float4* __restrict__ pred, const int* __restrict__ num_rois, int r, int C,
                  float score_thresh, VoteParams prm, int* __restrict__ keep, const int* __restrict__ keep_cnt,
                  float* __restrict__ keep_score, float4* __restrict__ vote_box) {
  constexpr int CAP = T * PER;
  extern __shared__ __align__(16) float vote_dyn[];
  const int cls = blockIdx.x + 1, img = blockIdx.y, tid = threadIdx.x;
  probs += (size_t)img * r * C; pred += (size_t)img * r * C;
  const size_t row = ((size_t)img * C + cls) * r;
  int* ck = keep + row;
  float* cs = keep_score + row;
  float4* vb = vote_box + row;
  const int nr = min(__ldg(num_rois + img), r);
  const int nk = __ldg(keep_cnt + (size_t)img * C + cls);
  const bool rescore = prm.method != FRCNN_BOX_VOTE_ID;
  block_vote<T, PER>(
      nr, [&](int e) { return __ldg(probs + (size_t)e * C + cls) > score_thresh; },
      [&](int e) { return __ldg(pred + (size_t)e * C + cls); }, [&](int e) { return __ldg(probs + (size_t)e * C + cls); }, nk,
      [&](int i, float4& b, float& s) { b = __ldg(pred + (size_t)ck[i] * C + cls); s = cs[i]; }, prm,
      [&](int i, float4 b, float s) { vb[i] = b; if (rescore) cs[i] = s; }, vote_dyn);
  if (!rescore) return;
  // stable re-sort by descending voted score: rank = #(higher) + #(equal and earlier).  Voted scores are >= +0, so the order
  // of their bit patterns is the float order, and a strict total order: the ranks are a permutation whatever the values.
  __syncthreads();                                             // votes written; the candidate arrays are free
  float4* sbox = reinterpret_cast<float4*>(vote_dyn);
  unsigned* sbits = reinterpret_cast<unsigned*>(vote_dyn + 4 * CAP);
  int* sroi = reinterpret_cast<int*>(vote_dyn + 5 * CAP);
  for (int i = tid; i < nk; i += T) { sbox[i] = vb[i]; sbits[i] = __float_as_uint(cs[i]); sroi[i] = ck[i]; }
  __syncthreads();
  for (int i = tid; i < nk; i += T) {
    const unsigned u = sbits[i];
    int rank = 0;
    for (int j = 0; j < nk; ++j) { const unsigned v = sbits[j]; rank += (v > u) | ((v == u) & (j < i)); }
    vb[rank] = sbox[i]; cs[rank] = __uint_as_float(u); ck[rank] = sroi[i];
  }
}

// one CTA: top rows [n_top, top_dim >= 5] voted against all rows [n_all, all_dim >= 5]; out [n_top, 5] in top's row order
template <int T, int PER>
__global__ void __launch_bounds__(T)
box_vote_set_kernel(const float* __restrict__ top, int n_top, int top_dim, const float* __restrict__ all, int n_all, int all_dim,
                    VoteParams prm, float* __restrict__ out) {
  extern __shared__ __align__(16) float vote_dyn[];
  block_vote<T, PER>(
      n_all, [](int) { return true; },
      [&](int e) { const float* d = all + (size_t)e * all_dim; return make_float4(d[0], d[1], d[2], d[3]); },
      [&](int e) { return all[(size_t)e * all_dim + 4]; }, n_top,
      [&](int i, float4& b, float& s) { const float* d = top + (size_t)i * top_dim; b = make_float4(d[0], d[1], d[2], d[3]); s = d[4]; },
      prm,
      [&](int i, float4 b, float s) { float* o = out + (size_t)i * 5; o[0] = b.x; o[1] = b.y; o[2] = b.z; o[3] = b.w; o[4] = s; },
      vote_dyn);
}

// ---- per-detection head features ---------------------------------------------------------------------------
// Runs after cap_emit_kernel and rebuilds its slot order from the truncated keep lists (classes ascending, slot =
// prefix(keep_cnt)[c] + j), so slot k of the features is record row k.  One CTA per (block of FEAT_SLOTS slots, image):
// each thread scans 4 consecutive class counts per pass of 1024 classes (C <= MAX_CLASSES), then the CTA copies its slots' fc7 rows,
// float4 wide.
constexpr int FEAT_THREADS = 256;
constexpr int FEAT_SLOTS = 8;

__global__ void __launch_bounds__(FEAT_THREADS)
detect_features_kernel(const int* __restrict__ keep, const int* __restrict__ keep_cnt, const float4* __restrict__ fc7, int r, int C,
                       int f4, int max_det, float4* __restrict__ feat_out, int* __restrict__ roi_out) {
  __shared__ int s_off[MAX_CLASSES + 1];
  __shared__ int s_warp[FEAT_THREADS / 32];
  __shared__ int s_roi[FEAT_SLOTS];
  const int img = blockIdx.y, slot0 = blockIdx.x * FEAT_SLOTS;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  keep += (size_t)img * C * r; keep_cnt += (size_t)img * C;
  int carry = 0;                                                // passes of 4 * FEAT_THREADS classes, carried
  for (int base = 0; base < C; base += 4 * FEAT_THREADS) {
    int cnt[4], v = 0;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int c = base + 4 * tid + q;
      cnt[q] = (c >= 1 && c < C) ? __ldg(keep_cnt + c) : 0;   // class 0 (background) never emits
      v += cnt[q];
    }
    int incl = v;
    for (int o = 1; o < 32; o <<= 1) { const int n = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += n; }
    if (base) __syncthreads();                                  // the previous pass has read s_warp
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    int run = carry + incl - v;
    for (int w = 0; w < warp; ++w) run += s_warp[w];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int c = base + 4 * tid + q;
      if (c < C) s_off[c] = run;
      run += cnt[q];
    }
    for (int w = 0; w < FEAT_THREADS / 32; ++w) carry += s_warp[w];
  }
  if (tid == 0) s_off[C] = carry;                               // detections of the image (the record's ndet)
  __syncthreads();
  if (tid < FEAT_SLOTS) {
    const int slot = slot0 + tid;
    int roi = -1;
    if (slot < max_det && slot < s_off[C]) {
      int lo = 1, hi = C;                                       // last class c with s_off[c] <= slot
      while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (s_off[mid] <= slot) lo = mid; else hi = mid; }
      roi = __ldg(keep + (size_t)lo * r + (slot - s_off[lo]));
    }
    s_roi[tid] = roi;
    if (slot < max_det) roi_out[(size_t)img * max_det + slot] = roi;
  }
  __syncthreads();
  const float4* src = fc7 + (size_t)img * r * f4;
  for (int i = tid; i < FEAT_SLOTS * f4; i += FEAT_THREADS) {
    const int s = i / f4, k = i - s * f4, slot = slot0 + s;
    if (slot >= max_det) break;
    const int roi = s_roi[s];
    feat_out[((size_t)img * max_det + slot) * f4 + k] = roi >= 0 ? __ldg(src + (size_t)roi * f4 + k) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

// ---- bottom-up regions (frcnn_detect_regions; the definition is in include/frcnn_b200.h) -------------------------------------
// class_nms_kernel runs unchanged over the RoI boxes: roi_box [batch*r, C] holds box_i in every class column, so it reads the RoI
// box where the post stage reads pred_boxes.  The per-RoI result of all classes is one 64-bit key: the score bits of a kept entry
// in the high word (scores >= +0, so unsigned order is float order) and ~class in the low word, merged with atomicMax -- the
// largest score wins and, among equal scores, the lowest class; the result does not depend on the order of the atomics.
constexpr int REGION_THREADS = 1024;
constexpr int REGION_CAP = DET_CAP_BIG;   // RoIs per image; the selection sorts up to this many 64-bit keys in shared memory

// thread per (row, class): box_i = rois[row, 1:5] / scale of the row's image, one __fdiv_rn per coordinate (bbox_decode's
// division); the key of the row is cleared once
__global__ void regions_boxes_kernel(const float* __restrict__ rois, const float* __restrict__ im_meta, int r, int C, int rows,
                                     float4* __restrict__ roi_box, unsigned long long* __restrict__ key) {
  const size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (size_t)rows * C) return;
  const int row = (int)(e / C);
  const float s = __ldg(im_meta + (size_t)(row / r) * 3);
  const float* q = rois + (size_t)row * 5;
  roi_box[e] = make_float4(__fdiv_rn(__ldg(q + 1), s), __fdiv_rn(__ldg(q + 2), s), __fdiv_rn(__ldg(q + 3), s), __fdiv_rn(__ldg(q + 4), s));
  if (e == (size_t)row * C) key[row] = 0ull;
}

// one CTA per (foreground class, image): folds the class's kept list into the per-RoI keys
__global__ void regions_fold_kernel(const int* __restrict__ keep, const int* __restrict__ keep_cnt, const float* __restrict__ keep_score,
                                    int r, int C, unsigned long long* __restrict__ key) {
  const int cls = blockIdx.x + 1, img = blockIdx.y;
  const size_t row = ((size_t)img * C + cls) * r;
  const int nk = __ldg(keep_cnt + (size_t)img * C + cls);
  for (int j = threadIdx.x; j < nk; j += blockDim.x) {
    const unsigned long long k = ((unsigned long long)__float_as_uint(__ldg(keep_score + row + j)) << 32) | (unsigned)~cls;
    atomicMax(key + (size_t)img * r + __ldg(keep + row + j), k);
  }
}

// one CTA per image: count conf >= thresh, then either the ascending compaction (min_boxes <= count <= max_boxes) or a bitonic sort
// of the cap (conf, ~index) keys, descending (conf descending, ties to the lower index); then the outputs of rows [0, max_out).
// Dynamic shared memory: cap (power of two >= r) 64-bit words.  box_stride: float4 boxes per RoI row of roi_box (C or 1).
__global__ void __launch_bounds__(REGION_THREADS, 1)
regions_select_kernel(const unsigned long long* __restrict__ key, const float4* __restrict__ roi_box, const int* __restrict__ num_rois,
                      int r, int box_stride, int cap, float conf_thresh, int min_boxes, int max_boxes, int max_out, float* __restrict__ boxes_out,
                      float* __restrict__ conf_out, int* __restrict__ class_out, int* __restrict__ index_out, int* __restrict__ count_out) {
  extern __shared__ __align__(16) unsigned long long sel[];
  __shared__ int s_warp[REGION_THREADS / 32];
  constexpr int NW = REGION_THREADS / 32;
  const int img = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  key += (size_t)img * r;
  const int nr = max(0, min(__ldg(num_rois + img), r));
  auto conf_of = [&](int e) { return __uint_as_float((unsigned)(key[e] >> 32)); };
  int mine = 0;
  for (int e = tid; e < nr; e += REGION_THREADS) mine += conf_of(e) >= conf_thresh;
  for (int o = 16; o; o >>= 1) mine += __shfl_xor_sync(0xffffffffu, mine, o);
  if (lane == 0) s_warp[warp] = mine;
  __syncthreads();
  int count = 0;
  for (int w = 0; w < NW; ++w) count += s_warp[w];
  __syncthreads();
  const bool in_range = count >= min_boxes && count <= max_boxes;
  const int n = in_range ? count : min(min(max(count, min_boxes), max_boxes), nr);
  if (in_range) {
    // ordered compaction in windows of REGION_THREADS rows; sel[k] holds ~index in its low word
    int done = 0;
    for (int base = 0; base < nr; base += REGION_THREADS) {
      const int e = base + tid;
      const bool f = e < nr && conf_of(e) >= conf_thresh;
      const unsigned bal = __ballot_sync(0xffffffffu, f);
      if (lane == 0) s_warp[warp] = __popc(bal);
      __syncthreads();
      int before = 0, tot = 0;
      for (int w = 0; w < NW; ++w) { const int v = s_warp[w]; before += w < warp ? v : 0; tot += v; }
      if (f) sel[done + before + __popc(bal & ((1u << lane) - 1u))] = (unsigned)~e;
      done += tot;
      __syncthreads();
    }
  } else {
    for (int e = tid; e < cap; e += REGION_THREADS)
      sel[e] = e < nr ? (key[e] & 0xffffffff00000000ull) | (unsigned)~e : 0ull;   // the keys are distinct except the padding
    __syncthreads();
    for (int k = 2; k <= cap; k <<= 1) {
      for (int j = k >> 1; j > 0; j >>= 1) {
        for (int e = tid; e < cap; e += REGION_THREADS) {
          const int ixj = e ^ j;
          if (ixj > e) {
            const unsigned long long a = sel[e], b = sel[ixj];
            if (((e & k) == 0) ? (a < b) : (a > b)) { sel[e] = b; sel[ixj] = a; }
          }
        }
        __syncthreads();
      }
    }
  }
  __syncthreads();
  for (int k = tid; k < max_out; k += REGION_THREADS) {
    float4 b = make_float4(0.f, 0.f, 0.f, 0.f);
    float cf = 0.f;
    int cl = 0, i = -1;
    if (k < n) {
      i = (int)~(unsigned)sel[k];
      const unsigned long long kk = key[i];
      const unsigned cb = (unsigned)(kk >> 32);
      cf = __uint_as_float(cb);
      cl = cb ? (int)~(unsigned)kk : 0;
      b = roi_box[((size_t)img * r + i) * box_stride];
    }
    const size_t o = (size_t)img * max_out + k;
    reinterpret_cast<float4*>(boxes_out)[o] = b;
    conf_out[o] = cf; class_out[o] = cl; index_out[o] = i;
  }
  if (tid == 0) count_out[img] = n;
}

// ---- bottom-up regions above REGIONS_CLASS_NMS_MAX classes: one overlap mask per image, one greedy walk per (class, image) ----------
// Every class runs greedy NMS over the same unregressed boxes, so the overlaps are computed once per image: mask[img][i][w] bit b =
// suppresses(box_i, box_{32w+b}) with the canonical boxes and areas class_nms_kernel uses (suppresses is symmetric in its two
// boxes), rows and columns >= nr empty.  A class then only needs its score order and a walk over the mask: the next row in order that
// no kept row has removed is kept, and removes its mask row.  That is block_greedy_nms's result, row for row.
constexpr int REGIONS_CLASS_NMS_MAX = 1024;   // frcnn_detect_regions: per-class NMS + fold up to this C, the mask walk above
constexpr int WALK_WARPS = 8;                 // r <= DET_CAP: one warp per class, 8 classes per CTA sharing the image's mask

__host__ __device__ constexpr int mask_words(int r) { return (r + 31) / 32; }

// thread per mask word (row i, word w) of image blockIdx.y; box [batch*r] float4 (regions_boxes_kernel with C = 1)
__global__ void regions_mask_kernel(const float4* __restrict__ box, const int* __restrict__ num_rois, int r, float thr, unsigned flags,
                                    unsigned* __restrict__ mask) {
  const int img = blockIdx.y, W = mask_words(r);
  const int e = blockIdx.x * blockDim.x + threadIdx.x;         // r * W <= 8192 * 256
  if (e >= r * W) return;
  const int i = e / W, w = e - i * W;
  const int nr = min(__ldg(num_rois + img), r);
  box += (size_t)img * r;
  unsigned bits = 0u;
  if (i < nr && thr >= 0.f) {                                   // thr < 0: block_greedy_nms suppresses nothing
    const float4 a = canon(__ldg(box + i), flags);
    const float aa = box_area(a, flags);
    const int nb = min(32, nr - w * 32);
    for (int b = 0; b < nb; ++b) {
      const float4 o = canon(__ldg(box + w * 32 + b), flags);
      if (suppresses(a, aa, o, box_area(o, flags), thr, flags)) bits |= 1u << b;
    }
  }
  mask[((size_t)img * r + i) * W + w] = bits;
}

// One unit per (foreground class, image).  BIG = false (r <= DET_CAP): a warp per unit, WALK_WARPS units per CTA; the CTA copies the
// image's mask rows into shared memory, each warp sorts its class in its own cap slots.  BIG = true (r <= DET_CAP_BIG): a CTA of
// NMS_THREADS per unit sorts, warp 0 walks with the mask rows read from global memory.  The sort is class_nms_kernel's (candidates
// score > -1, i.e. every valid row; key desc, row asc; the rest -inf at the tail).  The removed set is one register word per lane
// (!BIG) or mask_words(r) words of shared memory (BIG).  Each kept row is folded into the per-RoI key as regions_fold_kernel does.
// Dynamic shared memory: BIG: cap floats | cap ints | mask_words(r) words;  !BIG: mask_words(r) * r words (rounded to 4) | WALK_WARPS x (cap floats | cap ints).
template <bool BIG>
__global__ void __launch_bounds__(BIG ? NMS_THREADS : WALK_WARPS * 32)
regions_walk_kernel(const float* __restrict__ probs, const unsigned* __restrict__ mask, const int* __restrict__ num_rois, int r, int C,
                    int cap, unsigned long long* __restrict__ key) {
  extern __shared__ __align__(16) unsigned walk_dyn[];
  const int img = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, W = mask_words(r);
  const int nr = min(__ldg(num_rois + img), r);
  mask += (size_t)img * r * W;
  const unsigned* rows = mask;
  float* skey;
  int cls, g, G;                                                // this thread is g of the G sorting the class
  if (BIG) {
    skey = reinterpret_cast<float*>(walk_dyn);
    cls = blockIdx.x + 1; g = tid; G = NMS_THREADS;
  } else {
    for (int k = tid; k < nr * W; k += blockDim.x) walk_dyn[k] = __ldg(mask + k);
    rows = walk_dyn;
    skey = reinterpret_cast<float*>(walk_dyn + ((r * W + 3) & ~3)) + (size_t)warp * 2 * cap;
    cls = blockIdx.x * WALK_WARPS + warp + 1; g = lane; G = 32;
    __syncthreads();
    if (cls >= C) return;
  }
  int* sidx = reinterpret_cast<int*>(skey + cap);
  auto sync = [&] { if (BIG) __syncthreads(); else __syncwarp(); };
  probs += (size_t)img * r * C;
  for (int e = g; e < cap; e += G) {
    float k = __int_as_float(0xff800000);
    if (e < nr) {
      const float s = __ldg(probs + (size_t)e * C + cls);
      if (s > -1.f) k = s;
    }
    skey[e] = k; sidx[e] = e;
  }
  for (int k = 2; k <= cap; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      sync();
      for (int e = g; e < cap; e += G) {
        const int ixj = e ^ j;
        if (ixj > e) {
          const float a = skey[e], b = skey[ixj];
          const int ia = sidx[e], ib = sidx[ixj];
          const bool a_first = (a > b) || (a == b && ia < ib);
          const bool up = (e & k) == 0;
          if (up ? !a_first : a_first) { skey[e] = b; skey[ixj] = a; sidx[e] = ib; sidx[ixj] = ia; }
        }
      }
    }
  }
  sync();
  if (BIG && warp != 0) return;
  unsigned rem = 0u;                                            // !BIG: word `lane` of the removed set
  unsigned* srem = reinterpret_cast<unsigned*>(sidx + cap);     // BIG: the removed set in shared memory
  if (BIG) {
    for (int k = lane; k < W; k += 32) srem[k] = 0u;
    __syncwarp();
  }
  const unsigned long long low = (unsigned)~cls;
  unsigned long long* krow = key + (size_t)img * r;
  for (int p = 0; p < cap; ++p) {
    const float s = skey[p];
    if (!(s > -1.f)) break;                                     // the -inf tail: no candidates left
    const int row = sidx[p];
    const unsigned wv = BIG ? srem[row >> 5] : __shfl_sync(0xffffffffu, rem, row >> 5);
    if ((wv >> (row & 31)) & 1u) continue;                      // removed by a kept row
    if (lane == 0) atomicMax(krow + row, ((unsigned long long)__float_as_uint(s) << 32) | low);
    const unsigned* m = rows + (size_t)row * W;
    if (BIG) {
      __syncwarp();                                             // every lane has read srem
      for (int k = lane; k < W; k += 32) srem[k] |= __ldg(m + k);
      __syncwarp();
    } else if (lane < W) {
      rem |= m[lane];
    }
  }
}

// one CTA per (block of FEAT_SLOTS output rows, image): fc7 row of each selected RoI, zeros past the count
__global__ void __launch_bounds__(FEAT_THREADS)
regions_features_kernel(const int* __restrict__ index_out, const float4* __restrict__ fc7, int r, int f4, int max_out,
                        float4* __restrict__ feat_out) {
  const int img = blockIdx.y, k0 = blockIdx.x * FEAT_SLOTS;
  const float4* src = fc7 + (size_t)img * r * f4;
  for (int t = threadIdx.x; t < FEAT_SLOTS * f4; t += FEAT_THREADS) {
    const int s = t / f4, q = t - s * f4, k = k0 + s;
    if (k >= max_out) break;
    const int i = __ldg(index_out + (size_t)img * max_out + k);
    feat_out[((size_t)img * max_out + k) * f4 + q] = i >= 0 ? __ldg(src + (size_t)i * f4 + q) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

}  // namespace frcnn

using namespace frcnn;

extern "C" int frcnn_proposals(const float* props, const float* scores, const int* order, int n, int batch, int pre_nms_top_n,
                               int post_nms_top_n, float thresh, unsigned flags, float* rois, float* roi_scores, int* keep,
                               int* num, void* stream) {
  FRCNN_REQUIRE(props && scores && order && rois && roi_scores && keep && num && n > 0 && batch > 0 && post_nms_top_n > 0, "proposals: bad argument");
  const int m = (pre_nms_top_n > 0 && pre_nms_top_n < n) ? pre_nms_top_n : n;
  cudaStream_t st = (cudaStream_t)stream;
  if (thresh < 0.f) {
    gather_top_kernel<<<dim3((unsigned)cdiv(post_nms_top_n, 256), (unsigned)batch), 256, 0, st>>>(
        reinterpret_cast<const float4*>(props), scores, order, n, m, post_nms_top_n, rois, roi_scores, keep, num);
  } else {
    if (post_nms_top_n > PROPOSAL_CAP) { set_error("proposals: post_nms_top_n %d > capacity %d", post_nms_top_n, PROPOSAL_CAP); return ERR_CAPACITY; }
    proposals_kernel<<<(unsigned)batch, NMS_THREADS, 0, st>>>(reinterpret_cast<const float4*>(props), scores, order, n, m, post_nms_top_n,
                                                             thresh, flags, rois, roi_scores, keep, num);
  }
  FRCNN_LAUNCH_CHECK();
  return OK;
}

// Kept-set workspace of the `_nms`-compatible path: one slot PER DEVICE (ADVICE r01: a process-wide buffer was reused on
// whatever device a later call named), grown on demand; single stream use per device.
constexpr int MAX_DEVICES = 64;
static float4* g_kept[MAX_DEVICES]; static float* g_kept_area[MAX_DEVICES]; static int g_kept_cap[MAX_DEVICES];
static int ensure_kept(int dev, int n) {
  FRCNN_REQUIRE(dev >= 0 && dev < MAX_DEVICES, "device index %d out of range", dev);
  if (n <= g_kept_cap[dev]) return OK;
  if (g_kept[dev]) { cudaFree(g_kept[dev]); cudaFree(g_kept_area[dev]); g_kept[dev] = nullptr; g_kept_area[dev] = nullptr; g_kept_cap[dev] = 0; }
  FRCNN_CUDA(cudaMalloc(&g_kept[dev], (size_t)n * sizeof(float4)));
  FRCNN_CUDA(cudaMalloc(&g_kept_area[dev], (size_t)n * sizeof(float)));
  g_kept_cap[dev] = n;
  return OK;
}

extern "C" int frcnn_nms_sorted_dev(const float* boxes, int n, float thresh, unsigned flags, int max_out, int* keep, int* num, void* stream) {
  FRCNN_REQUIRE(boxes && keep && num && n > 0 && max_out > 0, "nms_sorted_dev: bad argument");
  int dev = 0;
  FRCNN_CUDA(cudaGetDevice(&dev));
  int rc = ensure_kept(dev, max_out < n ? max_out : n);
  if (rc) return rc;
  nms_sorted_kernel<<<1, NMS_THREADS, 0, (cudaStream_t)stream>>>(boxes, 4, n, thresh, flags, max_out, g_kept[dev], g_kept_area[dev], keep, num);
  FRCNN_LAUNCH_CHECK();
  return OK;
}

// device_id < 0: the calling thread's current device.  The caller's current device is restored before returning.
extern "C" int frcnn_nms_host(int* keep_out, int* num_out, const float* boxes_host, int boxes_num, int boxes_dim, float thresh,
                              int device_id, unsigned flags) {
  FRCNN_REQUIRE(keep_out && num_out, "nms_host: null output");
  *num_out = 0;
  if (boxes_num <= 0) return OK;
  FRCNN_REQUIRE(boxes_host && boxes_dim >= 4, "nms_host: bad input");
  int cur = -1;
  FRCNN_CUDA(cudaGetDevice(&cur));
  const int dev = device_id < 0 ? cur : device_id;
  if (cur != dev) FRCNN_CUDA(cudaSetDevice(dev));
  float* dboxes = nullptr; int* dkeep = nullptr; int* dnum = nullptr;
  int rc = ensure_kept(dev, boxes_num);
  cudaError_t e = cudaSuccess;
  if (!rc) {
    e = cudaMalloc(&dboxes, (size_t)boxes_num * boxes_dim * sizeof(float));
    if (e == cudaSuccess) e = cudaMalloc(&dkeep, (size_t)(boxes_num + 1) * sizeof(int));
    if (e == cudaSuccess) {
      dnum = dkeep + boxes_num;
      e = cudaMemcpy(dboxes, boxes_host, (size_t)boxes_num * boxes_dim * sizeof(float), cudaMemcpyHostToDevice);
    }
    if (e == cudaSuccess) {
      nms_sorted_kernel<<<1, NMS_THREADS>>>(dboxes, boxes_dim, boxes_num, thresh, flags, boxes_num, g_kept[dev], g_kept_area[dev], dkeep, dnum);
      e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpy(num_out, dnum, sizeof(int), cudaMemcpyDeviceToHost);
    if (e == cudaSuccess && *num_out > 0) e = cudaMemcpy(keep_out, dkeep, (size_t)(*num_out) * sizeof(int), cudaMemcpyDeviceToHost);
    cudaFree(dboxes); cudaFree(dkeep);
  }
  if (cur != dev) cudaSetDevice(cur);                    // leave the caller's (torch's) current device untouched
  if (rc) return rc;
  if (e != cudaSuccess) return cuda_fail(e, "frcnn_nms_host", __FILE__, __LINE__);
  return OK;
}

extern "C" size_t frcnn_detect_post_workspace_bytes(int r, int num_classes, int batch) {
  if (r <= DET_CAP) return 256;
  return (size_t)batch * num_classes * (size_t)((r + 3) & ~3) * 24 + 256;
}

extern "C" int frcnn_detect_regions_workspace_bytes(int r, int num_classes, int batch, size_t* bytes) {
  FRCNN_REQUIRE(bytes && r > 0 && batch > 0 && num_classes >= 2 && num_classes <= MAX_CLASSES,
                "detect_regions_workspace_bytes: bytes != NULL, r>0, batch>0, 2<=C<=%d required", MAX_CLASSES);
  *bytes = num_classes <= REGIONS_CLASS_NMS_MAX ? frcnn_detect_post_workspace_bytes(r, num_classes, batch)
                                                : (size_t)batch * r * mask_words(r) * 4 + 256;
  return OK;
}

static int soft_params(int method, float sigma, float nt, float score_thresh, SoftParams* p, const char* who) {
  FRCNN_REQUIRE(method == FRCNN_SOFT_NMS_LINEAR || method == FRCNN_SOFT_NMS_GAUSSIAN || method == FRCNN_SOFT_NMS_HARD,
                "%s: method %d is not FRCNN_SOFT_NMS_LINEAR / _GAUSSIAN / _HARD", who, method);
  FRCNN_REQUIRE(sigma > 0.f, "%s: sigma must be > 0", who);
  FRCNN_REQUIRE(score_thresh > 0.f, "%s: the prune threshold must be > 0", who);
  FRCNN_REQUIRE(nt == nt, "%s: the overlap threshold is NaN", who);
  *p = SoftParams{method, sigma, nt, score_thresh};
  return OK;
}

// the big variants need more than the default 48 KB of dynamic shared memory; set once per device
template <typename K>
static int smem_attr_once(K kernel, size_t bytes, bool (&done)[MAX_DEVICES]) {
  int dev = 0;
  FRCNN_CUDA(cudaGetDevice(&dev));
  FRCNN_REQUIRE(dev >= 0 && dev < MAX_DEVICES, "device index %d out of range", dev);
  if (!done[dev]) {
    FRCNN_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    done[dev] = true;
  }
  return OK;
}

static int vote_params(float thresh, int method, float beta, VoteParams* p, const char* who) {
  FRCNN_REQUIRE(method >= FRCNN_BOX_VOTE_ID && method <= FRCNN_BOX_VOTE_TEMP_AVG,
                "%s: method %d is not one of FRCNN_BOX_VOTE_ID ... FRCNN_BOX_VOTE_TEMP_AVG", who, method);
  FRCNN_REQUIRE(thresh > 0.f && thresh <= 1.f, "%s: the vote threshold must lie in (0, 1]", who);
  FRCNN_REQUIRE(beta > 0.f && beta <= FLT_MAX, "%s: beta must be finite and > 0", who);
  *p = VoteParams{thresh, method, beta};
  return OK;
}

// Both post entries: the shared checks, then class_stage(grid, st, pred) (its own checks, then the per-class launch), with `vote`
// the box-voting stage into vote_box, then the cap and the records: image b's count at ndet[b*s], its rows at det + b*s,
// s = record_stride (0: det [batch, max_det, 6], ndet [batch]).
template <typename ClassStage>
static int detect_post_run(const char* who, const float* cls_prob, const float* pred_boxes, const int* num_rois, int r, int batch,
                           int num_classes, float score_thresh, int max_per_image, int max_det, float* det, int* ndet, int record_stride,
                           int* keep, int* keep_cnt, float* keep_score, const VoteParams* vote, float* vote_box, void* stream,
                           ClassStage class_stage) {
  FRCNN_REQUIRE(cls_prob && pred_boxes && num_rois && det && ndet && keep && keep_cnt && keep_score, "%s: null pointer", who);
  FRCNN_REQUIRE(r > 0 && batch > 0 && num_classes >= 2 && num_classes <= MAX_CLASSES, "%s: r>0, batch>0, 2<=C<=%d required", who,
                MAX_CLASSES);
  if (r > DET_CAP_BIG) { set_error("%s: %d RoIs per image > capacity %d", who, r, DET_CAP_BIG); return ERR_CAPACITY; }
  FRCNN_REQUIRE(record_stride == 0 || record_stride >= (long long)max_det * 6, "%s: record_stride %d < max_det*6", who, record_stride);
  FRCNN_REQUIRE(!vote || (vote_box && ((uintptr_t)vote_box & 15) == 0), "%s: vote_box must be a 16-byte aligned device buffer", who);
  cudaStream_t st = (cudaStream_t)stream;
  const float4* pred = reinterpret_cast<const float4*>(pred_boxes);
  const dim3 grid((unsigned)(num_classes - 1), (unsigned)batch);
  if (int rc = class_stage(grid, st, pred)) return rc;
  FRCNN_LAUNCH_CHECK();
  const int rs = record_stride ? record_stride : max_det * 6, ns = record_stride ? record_stride : 1;
  if (!vote) {
    cap_emit_kernel<false><<<(unsigned)batch, NMS_THREADS, 0, st>>>(pred, r, num_classes, max_per_image, max_det, keep, keep_cnt,
                                                                   keep_score, det, ndet, rs, ns, nullptr);
    FRCNN_LAUNCH_CHECK();
    return OK;
  }
  float4* vb = reinterpret_cast<float4*>(vote_box);
  if (r <= DET_CAP) {
    class_vote_kernel<SOFT_THREADS, SOFT_PER><<<grid, SOFT_THREADS, vote_smem_bytes(DET_CAP), st>>>(
        cls_prob, pred, num_rois, r, num_classes, score_thresh, *vote, keep, keep_cnt, keep_score, vb);
  } else {
    static bool attr_done[MAX_DEVICES];
    if (int rc = smem_attr_once(class_vote_kernel<SOFT_THREADS_BIG, SOFT_PER_BIG>, vote_smem_bytes(DET_CAP_BIG), attr_done)) return rc;
    class_vote_kernel<SOFT_THREADS_BIG, SOFT_PER_BIG><<<grid, SOFT_THREADS_BIG, vote_smem_bytes(DET_CAP_BIG), st>>>(
        cls_prob, pred, num_rois, r, num_classes, score_thresh, *vote, keep, keep_cnt, keep_score, vb);
  }
  FRCNN_LAUNCH_CHECK();
  cap_emit_kernel<true><<<(unsigned)batch, NMS_THREADS, 0, st>>>(pred, r, num_classes, max_per_image, max_det, keep, keep_cnt, keep_score,
                                                                det, ndet, rs, ns, vb);
  FRCNN_LAUNCH_CHECK();
  return OK;
}

// the greedy per-class NMS launch of the post entries and frcnn_detect_regions: the kept sets in shared memory up to DET_CAP RoIs,
// else in `workspace`
static int class_nms_launch(dim3 grid, cudaStream_t st, const float* cls_prob, const float4* pred, const int* num_rois, int r, int batch,
                            int num_classes, float score_thresh, float nms_thresh, unsigned flags, int* keep, int* keep_cnt,
                            float* keep_score, void* workspace, size_t workspace_bytes) {
  if (r <= DET_CAP) {
    class_nms_kernel<DET_CAP, false><<<grid, NMS_THREADS, DET_CAP * 32, st>>>(cls_prob, pred, num_rois, r, num_classes, score_thresh,
                                                                              nms_thresh, flags, keep, keep_cnt, keep_score, nullptr);
    return OK;
  }
  FRCNN_REQUIRE(workspace && workspace_bytes >= frcnn_detect_post_workspace_bytes(r, num_classes, batch), "detect_post: workspace too small");
  static bool attr_done[MAX_DEVICES];
  if (int rc = smem_attr_once(class_nms_kernel<DET_CAP_BIG, true>, DET_CAP_BIG * 8, attr_done)) return rc;
  class_nms_kernel<DET_CAP_BIG, true><<<grid, NMS_THREADS, DET_CAP_BIG * 8, st>>>(cls_prob, pred, num_rois, r, num_classes, score_thresh,
                                                                                  nms_thresh, flags, keep, keep_cnt, keep_score,
                                                                                  reinterpret_cast<uint8_t*>(workspace));
  return OK;
}

// the greedy post (frcnn_detect_post / _vote); vote == nullptr: no voting stage
static int greedy_post(const char* who, const float* cls_prob, const float* pred_boxes, const int* num_rois, int r, int batch,
                       int num_classes, float score_thresh, float nms_thresh, unsigned flags, int max_per_image, int max_det, float* det,
                       int* ndet, int record_stride, int* keep, int* keep_cnt, float* keep_score, void* workspace, size_t workspace_bytes,
                       const VoteParams* vote, float* vote_box, void* stream) {
  return detect_post_run(who, cls_prob, pred_boxes, num_rois, r, batch, num_classes, score_thresh, max_per_image, max_det, det,
                         ndet, record_stride, keep, keep_cnt, keep_score, vote, vote_box, stream,
                         [&](dim3 grid, cudaStream_t st, const float4* pred) -> int {
    return class_nms_launch(grid, st, cls_prob, pred, num_rois, r, batch, num_classes, score_thresh, nms_thresh, flags, keep, keep_cnt,
                            keep_score, workspace, workspace_bytes);
  });
}

// the Soft-NMS post (frcnn_detect_post_soft / _soft_vote); vote == nullptr: no voting stage
static int soft_post(const char* who, const float* cls_prob, const float* pred_boxes, const int* num_rois, int r, int batch, int num_classes,
                     float score_thresh, int method, float sigma, float nt, float prune_thresh, int max_per_image, int max_det, float* det,
                     int* ndet, int record_stride, int* keep, int* keep_cnt, float* keep_score, const VoteParams* vote, float* vote_box,
                     void* stream) {
  return detect_post_run(who, cls_prob, pred_boxes, num_rois, r, batch, num_classes, score_thresh, max_per_image, max_det, det, ndet,
                         record_stride, keep, keep_cnt, keep_score, vote, vote_box, stream,
                         [&](dim3 grid, cudaStream_t st, const float4* pred) -> int {
    SoftParams prm;
    if (int rc = soft_params(method, sigma, nt, prune_thresh, &prm, who)) return rc;
    if (r <= DET_CAP) {
      class_soft_nms_kernel<SOFT_THREADS, SOFT_PER><<<grid, SOFT_THREADS, soft_smem_bytes(DET_CAP), st>>>(
          cls_prob, pred, num_rois, r, num_classes, score_thresh, prm, keep, keep_cnt, keep_score);
      return OK;
    }
    static bool attr_done[MAX_DEVICES];
    if (int rc = smem_attr_once(class_soft_nms_kernel<SOFT_THREADS_BIG, SOFT_PER_BIG>, soft_smem_bytes(DET_CAP_BIG), attr_done)) return rc;
    class_soft_nms_kernel<SOFT_THREADS_BIG, SOFT_PER_BIG><<<grid, SOFT_THREADS_BIG, soft_smem_bytes(DET_CAP_BIG), st>>>(
        cls_prob, pred, num_rois, r, num_classes, score_thresh, prm, keep, keep_cnt, keep_score);
    return OK;
  });
}

extern "C" int frcnn_detect_post(const float* cls_prob, const float* pred_boxes, const int* num_rois, int r, int batch, int num_classes,
                                 float score_thresh, float nms_thresh, unsigned flags, int max_per_image, int max_det,
                                 float* det, int* ndet, int record_stride, int* keep, int* keep_cnt, float* keep_score, void* workspace,
                                 size_t workspace_bytes, void* stream) {
  return greedy_post("detect_post", cls_prob, pred_boxes, num_rois, r, batch, num_classes, score_thresh, nms_thresh, flags, max_per_image,
                     max_det, det, ndet, record_stride, keep, keep_cnt, keep_score, workspace, workspace_bytes, nullptr, nullptr, stream);
}

extern "C" int frcnn_detect_post_vote(const float* cls_prob, const float* pred_boxes, const int* num_rois, int r, int batch,
                                      int num_classes, float score_thresh, float nms_thresh, unsigned flags, int max_per_image, int max_det,
                                      float* det, int* ndet, int record_stride, int* keep, int* keep_cnt, float* keep_score,
                                      void* workspace, size_t workspace_bytes, float vote_thresh, int vote_method, float vote_beta,
                                      float* vote_box, void* stream) {
  VoteParams vp;
  if (int rc = vote_params(vote_thresh, vote_method, vote_beta, &vp, "detect_post_vote")) return rc;
  return greedy_post("detect_post_vote", cls_prob, pred_boxes, num_rois, r, batch, num_classes, score_thresh, nms_thresh, flags,
                     max_per_image, max_det, det, ndet, record_stride, keep, keep_cnt, keep_score, workspace, workspace_bytes, &vp,
                     vote_box, stream);
}

extern "C" int frcnn_detect_post_soft(const float* cls_prob, const float* pred_boxes, const int* num_rois, int r, int batch,
                                      int num_classes, float score_thresh, int method, float sigma, float nt, float prune_thresh,
                                      int max_per_image, int max_det, float* det, int* ndet, int record_stride, int* keep,
                                      int* keep_cnt, float* keep_score, void* workspace, size_t workspace_bytes, void* stream) {
  (void)workspace; (void)workspace_bytes;
  return soft_post("detect_post_soft", cls_prob, pred_boxes, num_rois, r, batch, num_classes, score_thresh, method, sigma, nt, prune_thresh,
                   max_per_image, max_det, det, ndet, record_stride, keep, keep_cnt, keep_score, nullptr, nullptr, stream);
}

extern "C" int frcnn_detect_post_soft_vote(const float* cls_prob, const float* pred_boxes, const int* num_rois, int r, int batch,
                                           int num_classes, float score_thresh, int method, float sigma, float nt, float prune_thresh,
                                           int max_per_image, int max_det, float* det, int* ndet, int record_stride, int* keep,
                                           int* keep_cnt, float* keep_score, void* workspace, size_t workspace_bytes, float vote_thresh,
                                           int vote_method, float vote_beta, float* vote_box, void* stream) {
  (void)workspace; (void)workspace_bytes;
  VoteParams vp;
  if (int rc = vote_params(vote_thresh, vote_method, vote_beta, &vp, "detect_post_soft_vote")) return rc;
  return soft_post("detect_post_soft_vote", cls_prob, pred_boxes, num_rois, r, batch, num_classes, score_thresh, method, sigma, nt,
                   prune_thresh, max_per_image, max_det, det, ndet, record_stride, keep, keep_cnt, keep_score, &vp, vote_box, stream);
}

extern "C" int frcnn_box_vote_host(float* dets_out, const float* top_host, int n_top, int top_dim, const float* all_host, int n_all,
                                   int all_dim, float thresh, int method, float beta, int device_id) {
  FRCNN_REQUIRE(dets_out, "box_vote_host: null output");
  VoteParams prm;
  int rc = vote_params(thresh, method, beta, &prm, "box_vote_host");
  if (rc) return rc;
  if (n_top <= 0) return OK;
  FRCNN_REQUIRE(top_host && top_dim >= 5, "box_vote_host: bad top rows (rows of >= 5 floats: x1, y1, x2, y2, score)");
  if (n_all < 0) n_all = 0;
  FRCNN_REQUIRE(n_all == 0 || (all_host && all_dim >= 5), "box_vote_host: bad candidate rows (rows of >= 5 floats: x1, y1, x2, y2, score)");
  if (n_all > DET_CAP_BIG) { set_error("box_vote_host: %d candidates > capacity %d", n_all, DET_CAP_BIG); return ERR_CAPACITY; }
  int cur = -1;
  FRCNN_CUDA(cudaGetDevice(&cur));
  const int dev = device_id < 0 ? cur : device_id;
  if (cur != dev) FRCNN_CUDA(cudaSetDevice(dev));
  static bool attr_done[MAX_DEVICES];
  if (n_all > DET_CAP) rc = smem_attr_once(box_vote_set_kernel<SOFT_THREADS_BIG, SOFT_PER_BIG>, vote_smem_bytes(DET_CAP_BIG), attr_done);
  float* dtop = nullptr; float* dall = nullptr; float* dout = nullptr;
  cudaError_t e = cudaSuccess;
  if (!rc) {
    e = cudaMalloc(&dtop, (size_t)n_top * top_dim * sizeof(float));
    if (e == cudaSuccess) e = cudaMalloc(&dout, (size_t)n_top * 5 * sizeof(float));
    if (e == cudaSuccess && n_all > 0) e = cudaMalloc(&dall, (size_t)n_all * all_dim * sizeof(float));
    if (e == cudaSuccess) e = cudaMemcpy(dtop, top_host, (size_t)n_top * top_dim * sizeof(float), cudaMemcpyHostToDevice);
    if (e == cudaSuccess && n_all > 0) e = cudaMemcpy(dall, all_host, (size_t)n_all * all_dim * sizeof(float), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) {
      if (n_all <= DET_CAP)
        box_vote_set_kernel<SOFT_THREADS, SOFT_PER><<<1, SOFT_THREADS, vote_smem_bytes(DET_CAP)>>>(dtop, n_top, top_dim, dall, n_all,
                                                                                                  all_dim, prm, dout);
      else
        box_vote_set_kernel<SOFT_THREADS_BIG, SOFT_PER_BIG><<<1, SOFT_THREADS_BIG, vote_smem_bytes(DET_CAP_BIG)>>>(
            dtop, n_top, top_dim, dall, n_all, all_dim, prm, dout);
      e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpy(dets_out, dout, (size_t)n_top * 5 * sizeof(float), cudaMemcpyDeviceToHost);
    cudaFree(dtop); cudaFree(dall); cudaFree(dout);
  }
  if (cur != dev) cudaSetDevice(cur);                    // leave the caller's (torch's) current device untouched
  if (rc) return rc;
  if (e != cudaSuccess) return cuda_fail(e, "frcnn_box_vote_host", __FILE__, __LINE__);
  return OK;
}

extern "C" int frcnn_soft_nms_host(float* dets_out, int* keep_out, int* num_out, const float* dets_host, int n, int dim, int method,
                                   float sigma, float nt, float score_thresh, int device_id) {
  FRCNN_REQUIRE(dets_out && keep_out && num_out, "soft_nms_host: null output");
  *num_out = 0;
  SoftParams prm;
  int rc = soft_params(method, sigma, nt, score_thresh, &prm, "soft_nms_host");
  if (rc) return rc;
  if (n <= 0) return OK;
  FRCNN_REQUIRE(dets_host && dim >= 5, "soft_nms_host: bad input (rows of >= 5 floats: x1, y1, x2, y2, score)");
  if (n > DET_CAP_BIG) { set_error("soft_nms_host: %d boxes > capacity %d", n, DET_CAP_BIG); return ERR_CAPACITY; }
  int cur = -1;
  FRCNN_CUDA(cudaGetDevice(&cur));
  const int dev = device_id < 0 ? cur : device_id;
  if (cur != dev) FRCNN_CUDA(cudaSetDevice(dev));
  static bool attr_done[MAX_DEVICES];
  if (n > DET_CAP) rc = smem_attr_once(soft_nms_set_kernel<SOFT_THREADS_BIG, SOFT_PER_BIG>, soft_smem_bytes(DET_CAP_BIG), attr_done);
  float* din = nullptr; float* dout = nullptr; int* dkeep = nullptr;
  cudaError_t e = cudaSuccess;
  if (!rc) {
    e = cudaMalloc(&din, (size_t)n * dim * sizeof(float));
    if (e == cudaSuccess) e = cudaMalloc(&dout, (size_t)n * 5 * sizeof(float));
    if (e == cudaSuccess) e = cudaMalloc(&dkeep, (size_t)(n + 1) * sizeof(int));
    if (e == cudaSuccess) e = cudaMemcpy(din, dets_host, (size_t)n * dim * sizeof(float), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) {
      if (n <= DET_CAP)
        soft_nms_set_kernel<SOFT_THREADS, SOFT_PER><<<1, SOFT_THREADS, soft_smem_bytes(DET_CAP)>>>(din, n, dim, prm, dout, dkeep, dkeep + n);
      else
        soft_nms_set_kernel<SOFT_THREADS_BIG, SOFT_PER_BIG><<<1, SOFT_THREADS_BIG, soft_smem_bytes(DET_CAP_BIG)>>>(din, n, dim, prm, dout,
                                                                                                                 dkeep, dkeep + n);
      e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaMemcpy(num_out, dkeep + n, sizeof(int), cudaMemcpyDeviceToHost);
    if (e == cudaSuccess && *num_out > 0) e = cudaMemcpy(keep_out, dkeep, (size_t)(*num_out) * sizeof(int), cudaMemcpyDeviceToHost);
    if (e == cudaSuccess && *num_out > 0) e = cudaMemcpy(dets_out, dout, (size_t)(*num_out) * 5 * sizeof(float), cudaMemcpyDeviceToHost);
    cudaFree(din); cudaFree(dout); cudaFree(dkeep);
  }
  if (cur != dev) cudaSetDevice(cur);                    // leave the caller's (torch's) current device untouched
  if (rc) return rc;
  if (e != cudaSuccess) { *num_out = 0; return cuda_fail(e, "frcnn_soft_nms_host", __FILE__, __LINE__); }
  return OK;
}

extern "C" int frcnn_detect_features(const int* keep, const int* keep_cnt, const float* fc7, int r, int batch, int num_classes,
                                     int feat_dim, int max_det, float* feat_out, int* roi_out, void* stream) {
  FRCNN_REQUIRE(keep && keep_cnt && fc7 && feat_out && roi_out, "detect_features: null pointer");
  FRCNN_REQUIRE(r > 0 && batch > 0 && num_classes >= 2 && num_classes <= MAX_CLASSES && max_det > 0,
                "detect_features: r>0, batch>0, 2<=C<=%d, max_det>0 required", MAX_CLASSES);
  FRCNN_REQUIRE((long long)r * num_classes <= INT_MAX, "detect_features: r*C = %lld does not fit in int", (long long)r * num_classes);
  FRCNN_REQUIRE(feat_dim > 0 && feat_dim % 4 == 0 && ((uintptr_t)fc7 & 15) == 0 && ((uintptr_t)feat_out & 15) == 0,
                "detect_features: feat_dim %d must be a positive multiple of 4 and fc7 / feat_out 16-byte aligned", feat_dim);
  const dim3 grid((unsigned)cdiv(max_det, FEAT_SLOTS), (unsigned)batch);
  detect_features_kernel<<<grid, FEAT_THREADS, 0, (cudaStream_t)stream>>>(keep, keep_cnt, reinterpret_cast<const float4*>(fc7), r,
                                                                         num_classes, feat_dim / 4, max_det,
                                                                         reinterpret_cast<float4*>(feat_out), roi_out);
  FRCNN_LAUNCH_CHECK();
  return OK;
}

extern "C" int frcnn_detect_regions(const float* cls_prob, const float* rois, const int* num_rois, const float* im_meta, const float* fc7,
                                    int r, int batch, int num_classes, int feat_dim, float nms_thresh, unsigned flags, float conf_thresh,
                                    int min_boxes, int max_boxes, int* keep, int* keep_cnt, float* keep_score, void* workspace,
                                    size_t workspace_bytes, float* roi_box, unsigned long long* key, float* boxes_out, float* conf_out,
                                    int* class_out, int* index_out, float* feat_out, int* count_out, void* stream) {
  const bool walk = num_classes > REGIONS_CLASS_NMS_MAX;        // the overlap-mask path: keep / keep_cnt / keep_score are not used
  FRCNN_REQUIRE(cls_prob && rois && num_rois && im_meta && fc7 && (walk || (keep && keep_cnt && keep_score)) && roi_box && key &&
                boxes_out && conf_out && class_out && index_out && feat_out && count_out, "detect_regions: null pointer");
  FRCNN_REQUIRE(r > 0 && batch > 0 && num_classes >= 2 && num_classes <= MAX_CLASSES, "detect_regions: r>0, batch>0, 2<=C<=%d required",
                MAX_CLASSES);
  if (r > REGION_CAP) { set_error("detect_regions: %d RoIs per image > capacity %d", r, REGION_CAP); return ERR_CAPACITY; }
  FRCNN_REQUIRE((long long)r * batch <= INT_MAX, "detect_regions: r*batch = %lld does not fit in int", (long long)r * batch);
  FRCNN_REQUIRE(feat_dim > 0 && feat_dim % 4 == 0 && ((uintptr_t)fc7 & 15) == 0 && ((uintptr_t)feat_out & 15) == 0,
                "detect_regions: feat_dim %d must be a positive multiple of 4 and fc7 / feat_out 16-byte aligned", feat_dim);
  FRCNN_REQUIRE(((uintptr_t)roi_box & 15) == 0 && ((uintptr_t)boxes_out & 15) == 0 && ((uintptr_t)key & 7) == 0,
                "detect_regions: roi_box / boxes_out must be 16-byte and key 8-byte aligned");
  FRCNN_REQUIRE(conf_thresh >= 0.f && conf_thresh <= 1.f, "detect_regions: conf_thresh must lie in [0, 1]");
  FRCNN_REQUIRE(min_boxes >= 0 && max_boxes >= 1 && min_boxes <= max_boxes, "detect_regions: 0 <= min_boxes <= max_boxes, max_boxes >= 1 required");
  size_t need = 0;
  if (walk)
    FRCNN_REQUIRE(workspace && ((uintptr_t)workspace & 3) == 0 && frcnn_detect_regions_workspace_bytes(r, num_classes, batch, &need) == OK &&
                  workspace_bytes >= need, "detect_regions: workspace too small");
  else
    FRCNN_REQUIRE(r <= DET_CAP || (workspace && workspace_bytes >= frcnn_detect_post_workspace_bytes(r, num_classes, batch)),
                  "detect_regions: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  float4* rb = reinterpret_cast<float4*>(roi_box);
  const int rows = r * batch;
  const int box_stride = walk ? 1 : num_classes;
  int cap = 1;                                                  // sort capacity: power of two >= r
  while (cap < r) cap <<= 1;
  regions_boxes_kernel<<<(unsigned)(((size_t)rows * box_stride + 255) / 256), 256, 0, st>>>(rois, im_meta, r, box_stride, rows, rb, key);
  FRCNN_LAUNCH_CHECK();
  if (walk) {
    unsigned* mask = reinterpret_cast<unsigned*>(workspace);
    const int W = mask_words(r);
    regions_mask_kernel<<<dim3((unsigned)cdiv(r * W, 256), (unsigned)batch), 256, 0, st>>>(rb, num_rois, r, nms_thresh, flags, mask);
    FRCNN_LAUNCH_CHECK();
    if (r <= DET_CAP) {
      static bool attr_done[MAX_DEVICES];
      const size_t smem_max = (size_t)DET_CAP * mask_words(DET_CAP) * 4 + (size_t)WALK_WARPS * DET_CAP * 8;
      if (int rc = smem_attr_once(regions_walk_kernel<false>, smem_max, attr_done)) return rc;
      const size_t smem = (size_t)((r * W + 3) & ~3) * 4 + (size_t)WALK_WARPS * cap * 8;
      regions_walk_kernel<false><<<dim3((unsigned)cdiv(num_classes - 1, WALK_WARPS), (unsigned)batch), WALK_WARPS * 32, smem, st>>>(
          cls_prob, mask, num_rois, r, num_classes, cap, key);
    } else {
      static bool attr_done[MAX_DEVICES];
      const size_t smem_max = (size_t)DET_CAP_BIG * 8 + (size_t)mask_words(DET_CAP_BIG) * 4;
      if (int rc = smem_attr_once(regions_walk_kernel<true>, smem_max, attr_done)) return rc;
      regions_walk_kernel<true><<<dim3((unsigned)(num_classes - 1), (unsigned)batch), NMS_THREADS, (size_t)cap * 8 + (size_t)W * 4, st>>>(
          cls_prob, mask, num_rois, r, num_classes, cap, key);
    }
    FRCNN_LAUNCH_CHECK();
  } else {
    // every valid row is a candidate of every class: score_thresh -1 < any score >= +0
    if (int rc = class_nms_launch(dim3((unsigned)(num_classes - 1), (unsigned)batch), st, cls_prob, rb, num_rois, r, batch, num_classes, -1.f,
                                  nms_thresh, flags, keep, keep_cnt, keep_score, workspace, workspace_bytes)) return rc;
    FRCNN_LAUNCH_CHECK();
    regions_fold_kernel<<<dim3((unsigned)(num_classes - 1), (unsigned)batch), 256, 0, st>>>(keep, keep_cnt, keep_score, r, num_classes, key);
    FRCNN_LAUNCH_CHECK();
  }
  static bool attr_done[MAX_DEVICES];
  if (int rc = smem_attr_once(regions_select_kernel, (size_t)REGION_CAP * 8, attr_done)) return rc;
  const int max_out = max_boxes < r ? max_boxes : r;
  regions_select_kernel<<<(unsigned)batch, REGION_THREADS, (size_t)cap * 8, st>>>(key, rb, num_rois, r, box_stride, cap, conf_thresh,
                                                                                  min_boxes, max_boxes, max_out, boxes_out, conf_out,
                                                                                  class_out, index_out, count_out);
  FRCNN_LAUNCH_CHECK();
  regions_features_kernel<<<dim3((unsigned)cdiv(max_out, FEAT_SLOTS), (unsigned)batch), FEAT_THREADS, 0, st>>>(
      index_out, reinterpret_cast<const float4*>(fc7), r, feat_dim / 4, max_out, reinterpret_cast<float4*>(feat_out));
  FRCNN_LAUNCH_CHECK();
  return OK;
}
