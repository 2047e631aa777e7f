/* frcnn_b200 -- C ABI of the H100 (sm_90a) Faster R-CNN inference path.
 *
 * Drop-in boundary for endernewton/tf-faster-rcnn's `Network.test_image()` / `im_detect()` / `nms()`
 * hot path.  The reference's only native interface on this path is
 *     void _nms(int* keep_out, int* num_out, const float* boxes_host, int boxes_num,
 *               int boxes_dim, float nms_overlap_thresh, int device_id);      (lib/nms/gpu_nms.hpp:1-2)
 * reached through lib/nms/gpu_nms.pyx:16-31 and lib/model/nms_wrapper.py:15-23; everything else on the
 * path is TensorFlow graph ops called from Python (lib/nets/network.py).  This header therefore exports
 *   (1) frcnn_nms_host      -- argument-compatible superset of `_nms` (same order + `flags`),
 *   (2) one entry point per device stage of the TEST-mode graph, so the Python host code that mirrors
 *       lib/nets/{vgg16,resnet_v1,mobilenet_v1}.py can enqueue the graph on a CUDA stream (and capture it into a CUDA graph).
 *
 * Conventions
 *   - plain C types only; every function returns 0 on success or a negative frcnn_status; the message of
 *     the last failure on the calling thread is read with frcnn_last_error().  Nothing is printed
 *     (the reference's CUDA_CHECK prints and continues, lib/nms/nms_kernel.cu:12-19).
 *   - pointers named *_dev are device pointers owned by the caller (PyTorch tensors' data_ptr());
 *     `stream` is a cudaStream_t passed as void*; all device entry points are asynchronous on it.
 *   - activations: NHWC fp32, dense.  conv weights: packed by frcnn_pack_conv_weights.
 *   - a handle/plan is single-stream and not re-entrant; one per GPU/rank.
 */
#ifndef FRCNN_B200_H_
#define FRCNN_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
  FRCNN_OK = 0,
  FRCNN_ERR_CUDA = -1,         /* a CUDA runtime/driver call failed (text in frcnn_last_error) */
  FRCNN_ERR_ARG = -2,          /* invalid argument */
  FRCNN_ERR_NO_DEVICE = -3,    /* no usable sm_90 device */
  FRCNN_ERR_DRIVER_ENTRY = -4, /* cuTensorMapEncodeTiled not obtainable from the driver */
  FRCNN_ERR_CAPACITY = -5      /* problem larger than the compiled-in capacity */
} frcnn_status;

/* NMS predicate flags (SURVEY.md 8(a) row N). */
#define FRCNN_NMS_PLUS_ONE 1u        /* '+1' pixel areas (cpu_nms.pyx / nms_kernel.cu); else continuous (TF) */
#define FRCNN_NMS_INCLUSIVE 2u       /* suppress when ovr >= thr (cpu_nms.pyx:65); else ovr > thr */
#define FRCNN_NMS_SKIP_DEGENERATE 4u /* IoU := 0 when either area <= 0 (tf.image.non_max_suppression) */
#define FRCNN_NMS_MODE_CPU_NMS (FRCNN_NMS_PLUS_ONE | FRCNN_NMS_INCLUSIVE)
#define FRCNN_NMS_MODE_GPU_NMS (FRCNN_NMS_PLUS_ONE)
#define FRCNN_NMS_MODE_TF (FRCNN_NMS_SKIP_DEGENERATE)

/* activation applied by conv/depthwise epilogues */
#define FRCNN_ACT_NONE 0
#define FRCNN_ACT_RELU 1
#define FRCNN_ACT_RELU6 2

int frcnn_version(void);
/* copies the calling thread's last error text into buf (NUL terminated); returns its length */
int frcnn_last_error(char* buf, size_t buflen);
/* 0 when device `device_id` exists and is compute capability 10.x */
int frcnn_check_device(int device_id);
/* cudaMemsetAsync(dev_ptr, 0, bytes) on `stream`: lets a host layer clear buffers (detection records) without a framework fill kernel */
int frcnn_zero_async(void* dev_ptr, size_t bytes, void* stream);

/* CUDA-graph capture of a sequence of the stage calls below (one image or batch = one replay): begin on a NON-default stream,
 * enqueue the stages on that stream, end -> an executable graph; launch it on any stream.  No allocation or synchronisation
 * happens inside the stages, so the whole TEST-mode path is capturable. */
typedef struct frcnn_graph frcnn_graph;
int frcnn_graph_begin(void* stream);
int frcnn_graph_end(void* stream, frcnn_graph** out);
int frcnn_graph_launch(const frcnn_graph* g, void* stream);
void frcnn_graph_destroy(frcnn_graph* g);

/* ---- (1) NMS, host buffers: replaces `_nms` (lib/nms/gpu_nms.hpp:1-2, nms_kernel.cu:91-144) ----------
 * boxes_host: [boxes_num, boxes_dim>=4] rows (x1,y1,x2,y2,...), ALREADY sorted by descending score, as the
 * reference's Cython wrapper guarantees (gpu_nms.pyx:25-28).  keep_out: capacity boxes_num; receives
 * indices into the sorted input in ascending order.  Synchronous.  device_id < 0 selects the calling thread's current
 * device; the caller's current device is restored before returning (the reference's _nms leaves it switched). */
int frcnn_nms_host(int* keep_out, int* num_out, const float* boxes_host, int boxes_num, int boxes_dim,
                   float nms_overlap_thresh, int device_id, unsigned flags);

/* Same greedy NMS, device buffers, no sort: boxes_dev [n,4] in priority order.  keep_dev: capacity
 * max_out (int32 indices into boxes_dev), num_dev: int32 count.  Early exit at max_out kept. */
int frcnn_nms_sorted_dev(const float* boxes_dev, int n, float thresh, unsigned flags, int max_out,
                         int* keep_dev, int* num_dev, void* stream);

/* ---- (2) dense stages: conv / FC as implicit GEMM on wgmma (FP16x3 operand split, fp32 accumulate in registers) -
 * Replaces slim.conv2d / slim.fully_connected (+ folded bias or BatchNorm scale/shift, ReLU/ReLU6,
 * residual add) as used by lib/nets/{vgg16,resnet_v1,mobilenet_v1}.py and network.py:323-378.
 *   out[n,ho,wo,co] = act( (sum_{r,s,ci} in[n, ho*stride+r-pad_t, wo*stride+s-pad_l, ci] * w[co,r,s,ci])
 *                          * scale[co] + shift[co] (+ residual[n,ho,wo,co]) )
 * Requirements: cin % 32 == 0.  w_hi/w_lo from frcnn_pack_conv_weights.  scale may be NULL (=1). */
typedef struct frcnn_conv_plan frcnn_conv_plan;
#define FRCNN_CONV_F16X3 0   /* fp16 hi/lo split of both operands, 3 x wgmma f16, fp32 accumulate.  Operands carried to 2^-22
                              * relative for activations 2^-14 <= |x| < 65520 and weights down to 2^-27 below the layer's largest;
                              * smaller activations lose precision (2^-20 at 2^-16, 2^-12 at 2^-24).  |x| >= 65520, +-Inf and NaN
                              * make every output whose receptive field holds them non-finite. */
#define FRCNN_CONV_TF32X3 1  /* tf32 hi/lo split, 3 x wgmma tf32 (same 22-bit products, twice the tensor time); 2^-22 relative from
                              * 2^-115 up to the tf32 overflow, non-finite inputs give non-finite outputs */
#define FRCNN_CONV_F16X1 2   /* THROUGHPUT mode, not fp32-grade: plain fp16 operands (the hi planes only, 2^-12 relative), 1 MMA per
                              * product, fp32 accumulate; ~3e-4 of the output range per layer instead of ~4e-7.  Same packed
                              * weights and the same activation range as F16X3. */

typedef struct {
  const float* in_dev;       /* [n, h, w, cin] */
  const void* w_hi_dev;      /* [cout, kh*kw*cin] hi plane from frcnn_pack_conv_weights (fp16) / _tf32 (fp32) */
  const void* w_lo_dev;      /* [cout, kh*kw*cin] lo plane (residual of the hi rounding) */
  const float* scale_dev;    /* [cout] or NULL */
  const float* shift_dev;    /* [cout] or NULL */
  const float* residual_dev; /* [n, ho, wo, cout] or NULL */
  float* out_dev;            /* [n, ho, wo, cout] */
  int n, h, w, cin;
  int cout, kh, kw, stride;
  int pad_t, pad_l;          /* zero padding before the first row / column */
  int ho, wo;
  int act;                   /* FRCNN_ACT_* */
  int block_n;               /* 0 = choose; else 64/128 */
  int kb_per_chunk;          /* validated and reported (frcnn_conv_plan_geometry); the sm_90a kernel promotes every k-block */
  int split_k;               /* 0 = choose; 1 = never; n = split the K loop over n CTAs + deterministic reduce pass */
  int impl;                  /* FRCNN_CONV_F16X3 (0, default) | FRCNN_CONV_TF32X3 (kept for A/B measurements) | FRCNN_CONV_F16X1 */
  float out_mult;            /* F16X3: 2^-wexp of frcnn_pack_conv_weights (0 is read as 1) */
  /* Second A source (pointwise layers only: 1x1, stride 1, no padding): K = cin + cin2, the packed weights are
   * [cout][cin + cin2] and the input channels cin .. cin + cin2 - 1 are read from in2_dev [n, h, w, cin2].  A ResNet
   * projection shortcut rides in the closing 1x1 conv's K loop this way.  NULL / 0 = one source. */
  const float* in2_dev;
  int cin2;                  /* 0, or a positive multiple of 32 */
  /* Mean epilogue (pointwise layers only), on when mean_hw > 0: instead of out_dev, write mean_dev[p / mean_hw, cout] = the
   * mean of the activated outputs of the mean_hw consecutive pixels p of each group (n*h*w % mean_hw == 0); out_dev is not
   * written and may be NULL.  Summed in a fixed order (no atomics), divided once by mean_hw.  Never split along K. */
  float* mean_dev;
  int mean_hw;               /* 0 = off */
} frcnn_conv_desc;

int frcnn_conv_plan_create(frcnn_conv_plan** out, const frcnn_conv_desc* d);
int frcnn_conv_plan_run(const frcnn_conv_plan* p, void* stream);
/* Host-only (no CUDA call): the work decomposition frcnn_conv_plan_create would choose on a GPU with sm_count SMs.  Device
 * pointers in *d are ignored.  out16 = {block_n, tile_n, tile_h, tile_w, m_tiles, n_tiles, tiles, split_tiles, splits,
 * k_blocks_per_split, work_units, grid, k_blocks, k_blocks_per_chunk, tiles_h, tiles_w}. */
int frcnn_conv_plan_geometry(const frcnn_conv_desc* d, int sm_count, int* out16);
int frcnn_conv_plan_info(const frcnn_conv_plan* p, int* block_n, int* tile_n, int* tile_h, int* tile_w,
                         int* grid_m, int* grid_n, int* splits, int* smem_bytes);
/* debug aid (watchdog build only): trace_dev (int64[64*8], device) receives clock64() stamps of the pipeline hand-offs of
 * CTA 0 for its first 64 k-blocks: [kb][0]=producer issued the loads, [1]=consumer thread 0 saw the operands,
 * [2]=consumer thread 0 released the stage. NULL disables. */
int frcnn_conv_plan_set_trace(frcnn_conv_plan* p, long long* trace_dev);
void frcnn_conv_plan_destroy(frcnn_conv_plan* p);
/* development aid: in the watchdog build (libfrcnn_b200_wd.so, -DFRCNN_WATCHDOG) a barrier wait of the dense kernel that
 * lasts > ~0.2 s aborts the kernel instead of hanging the GPU; out16 = {aborted, waits_timed_out, block, thread, wait_tag,
 * parity, aux, ...}.  In the normal build out16[15] = 0xffffffff and the rest is zero. */
int frcnn_debug_watchdog(unsigned int* out16, int reset);

/* HWIO [kh,kw,cin,cout] (TF layout) -> K-major [cout][kh][kw][cin] fp16 planes:
 *   hi = RN_f16(w * 2^wexp), lo = RN_f16((w * 2^wexp - hi) * 2^11).  The caller picks wexp so that max|w| * 2^wexp lies in
 * [2^13, 2^14) and passes out_mult = 2^-wexp in the conv descriptor. */
int frcnn_pack_conv_weights(const float* w_hwio_dev, void* w_hi_dev, void* w_lo_dev, int kh, int kw,
                            int cin, int cout, int wexp, void* stream);
/* same layout, fp32 planes of tf32-rounded values (hi = RN_tf32(w), lo = RN_tf32(w - hi)) for FRCNN_CONV_TF32X3 */
int frcnn_pack_conv_weights_tf32(const float* w_hwio_dev, float* w_hi_dev, float* w_lo_dev, int kh, int kw,
                                 int cin, int cout, void* stream);

/* ---- (3) bandwidth stages (SIMT, fp32, no FMA contraction where the oracle has separate roundings) ---- */
/* first-layer convolution for cin==3 (vgg conv1_1, resnet conv1 7x7/2, mobilenet Conv2d_0 3x3/2):
 * direct fp32 FFMA conv, w HWIO [k,k,3,cout], y = act(conv*scale + shift) */
int frcnn_conv_first(const float* in_dev, const float* w_hwio_dev, const float* scale_dev,
                     const float* shift_dev, float* out_dev, int n, int h, int w, int cout, int k,
                     int stride, int pad_t, int pad_l, int ho, int wo, int act, void* stream);
/* depthwise 3x3 (slim.separable_conv2d with num_outputs=None, mobilenet_v1.py:21-49):
 * w [3,3,c] ; y = act(dw*scale + shift) */
int frcnn_depthwise3x3(const float* in_dev, const float* w_dev, const float* scale_dev,
                       const float* shift_dev, float* out_dev, int n, int h, int w, int c, int stride,
                       int pad_t, int pad_l, int ho, int wo, int act, void* stream);
/* max pool k x k / stride; padded cells are skipped when pad_is_neg_inf != 0 (TF 'SAME'),
 * or count as zeros (tf.pad + 'VALID', resnet_v1.py:83-84) */
int frcnn_max_pool(const float* in_dev, float* out_dev, int n, int h, int w, int c, int k, int stride,
                   int pad_t, int pad_l, int ho, int wo, int pad_is_neg_inf, void* stream);
/* mean over the spatial positions: [r, hw, c] -> [r, c]  (tf.reduce_mean axis=[1,2]) */
int frcnn_spatial_mean(const float* in_dev, float* out_dev, int r, int hw, int c, void* stream);

/* image -> network blob on the device (lib/model/test.py:26-58 for one scale): blob[y,x,c] = bilinear resize, with OpenCV's
 * INTER_LINEAR float arithmetic, of (float32(img) - means) ; img_dev uint8 BGR [h0,w0,3]; blob_dev fp32 [H,W,3] with
 * H = cvRound(h0*fy), W = cvRound(w0*fx) computed by the caller.  means3 is a HOST pointer. */
int frcnn_preprocess(const unsigned char* img_dev, int h0, int w0, const double* means3, double fx, double fy,
                     float* blob_dev, int H, int W, void* stream);
/* the same blob of the mirrored image img[:, ::-1] (the flipped view of test-time augmentation): mirror first, then resize, so
 * that un-flipping a box is exact in original pixels.  Bit for bit frcnn_preprocess of a host-mirrored image. */
int frcnn_preprocess_hflip(const unsigned char* img_dev, int h0, int w0, const double* means3, double fx, double fy,
                           float* blob_dev, int H, int W, void* stream);

/* ---- (4) proposal / detection stages.  Every stage takes `batch` images of one blob shape (the reference is batch 1,
 * lib/nets/network.py:388; batch > 1 is the throughput extension of SURVEY.md 8(f) rank 4): per-image arrays are
 * concatenated image-major, RoI rows carry their image index in column 0 exactly like crop_and_resize's box_ind. ---- */

/* RPN: 2-way softmax (fg prob), anchor generation, bbox_transform_inv, clip -- proposal_layer.py:62-69.
 * rpn_out_dev: [batch*hw, ld] rows with the 2A class logits at column 0 and the 4A deltas at column delta_col
 * (delta_col % 4 == 0, ld % 4 == 0: the fused 1x1 RPN head writes both).
 * base_anchors_dev [A,4].  scores_dev [batch*hw*A], props_dev [batch*hw*A,4] in (image,h,w,a) order. */
int frcnn_rpn_decode(const float* rpn_out_dev, int ld, int delta_col, const float* base_anchors_dev, int num_anchors,
                     int batch, int fh, int fw, int feat_stride, float im_h, float im_w, float* scores_dev,
                     float* props_dev, void* stream);
/* stable descending sort of `batch` segments of n fp32 keys each (ties: lower index first) -> order_dev int32[batch*n],
 * indices LOCAL to the segment; one thread-block cluster per segment, n <= 90 112.  The workspace arguments are kept
 * from the r01 (CUB based) signature and may be NULL / 0. */
size_t frcnn_sort_workspace_bytes(int n);
int frcnn_sort_desc(const float* keys_dev, int n, int batch, int* order_dev, float* sorted_keys_dev, void* workspace_dev,
                    size_t workspace_bytes, void* stream);
/* proposal selection (proposal_layer_tf / proposal_layer / proposal_top_layer), per image: walk `order`, greedy NMS
 * with `flags` over the first `pre_nms_top_n` (<=0: all) candidates, stop at post_nms_top_n.  thresh < 0
 * means no NMS (TEST.MODE='top').  props/scores/order: [batch][n].  rois_dev [batch*post_nms_top_n,5] =
 * (image,x1,y1,x2,y2), zero padded per image; roi_scores_dev [batch*post_nms_top_n]; keep_dev int32 segment-local
 * indices into props; num_dev int32[batch] counts. */
int frcnn_proposals(const float* props_dev, const float* scores_dev, const int* order_dev, int n, int batch,
                    int pre_nms_top_n, int post_nms_top_n, float thresh, unsigned flags, float* rois_dev,
                    float* roi_scores_dev, int* keep_dev, int* num_dev, void* stream);
/* tf.image.crop_and_resize on the stride-16 feature map + optional 2x2 max pool (network.py:141-157,
 * resnet_v1.py:55-76).  feat_dev [batch,fh,fw,c]; rois_dev [r,5] = (image index, blob-scale pixels).  pooled = 7;
 * pre_pool 0: direct 7x7, 1: 14x14 then 2x2/2 max.  out [r,7,7,c] */
int frcnn_crop_pool(const float* feat_dev, int batch, int fh, int fw, int c, const float* rois_dev, int r, int pooled,
                    int pre_pool, float* out_dev, void* stream);
/* POOLING_MODE 'align' (extension): torchvision.ops.roi_align(spatial_scale, sampling_ratio, aligned) on NHWC, each fp32
 * operation rounded once (no contraction); a sample outside [-1, dim] is not read.  feat_dev [batch,fh,fw,c], c % 4 == 0;
 * rois_dev [r,5] = (image index clamped to [0, batch-1], x1, y1, x2, y2 in blob pixels); 1 <= pooled <= 16;
 * 0 <= sampling_ratio <= FRCNN_ROI_ALIGN_MAX_SAMPLING (0 = adaptive, ceil(roi size / pooled) per axis: the launch walks every
 * sample, so the caller keeps boxes bounded -- RPN RoIs lie inside the blob, caller boxes within [-W,2W] x [-H,2H]).
 * out_dev [r,pooled,pooled,c]. */
#define FRCNN_ROI_ALIGN_MAX_SAMPLING 16
int frcnn_roi_align(const float* feat_dev, int batch, int fh, int fw, int c, const float* rois_dev, int r, int pooled,
                    float spatial_scale, int sampling_ratio, int aligned, float* out_dev, void* stream);
/* POOLING_MODE 'pool' (extension): torchvision.ops.roi_pool -- corners round(x*spatial_scale) half away from zero, bins of
 * max(size+1,1)/pooled cells, max by '>' from -FLT_MAX (empty bin: 0).  Arguments as frcnn_roi_align. */
int frcnn_roi_pool(const float* feat_dev, int batch, int fh, int fw, int c, const float* rois_dev, int r, int pooled,
                   float spatial_scale, float* out_dev, void* stream);
/* split the fused [r, ld] head GEMM output (cls logits at col 0, 4C deltas at col C):
 * cls_score [r,C], cls_prob = softmax, bbox_pred = delta*stds + means (network.py:361-378,428-432) */
int frcnn_cls_finish(const float* head_out_dev, int ld, int r, int num_classes, const float* stds4,
                     const float* means4, float* cls_score_dev, float* cls_prob_dev, float* bbox_pred_dev,
                     void* stream);
/* im_detect tail: boxes = rois[:,1:5]/scale; bbox_transform_inv; one-sided clip to the ORIGINAL image
 * (lib/model/test.py:95-102,67-77).  r * num_classes must fit in int (else FRCNN_ERR_ARG).  im_meta_dev [batch,3] fp32 = (im_scale, orig_h, orig_w) per image, read on the
 * device (the launch is CUDA-graph capturable: the host only rewrites the 12 bytes).  pred_boxes_dev [r,4C] */
int frcnn_bbox_decode(const float* rois_dev, const float* bbox_pred_dev, int r, int num_classes, int batch,
                      const float* im_meta_dev, float* pred_boxes_dev, void* stream);
/* test_net tail (lib/model/test.py:162-180), per image: per class j>=1: score > thresh, NMS(flags, nms_thresh), then the
 * max_per_image cap over all classes.  2 <= C <= 4096 classes (background included).  r = RoI rows per image (<= 8192; above 1024 -- TEST.MODE='top' with
 * RPN_TOP_N=5000 -- the kept sets live in `workspace_dev`, frcnn_detect_post_workspace_bytes(r, C, batch) bytes, else the
 * workspace may be NULL).  num_rois_dev: int32[batch] valid-row counts.  det_dev [batch,max_det,6] =
 * (x1,y1,x2,y2,score,class) sorted by (class, descending score); ndet_dev int32[batch] = the number of detections of
 * the image, which EXCEEDS max_det when the records did not fit (the caller must treat that as an error).
 * record_stride (4-byte words; 0 = dense): distance between consecutive images in BOTH det_dev and ndet_dev, so that a
 * caller can interleave count and rows into one fixed-size record per image (the multi-GPU all-gather payload).
 * keep_dev [batch,C,r] int32 roi indices per class (after the cap), keep_cnt_dev [batch,C]; keep_score_dev [batch,C,r]. */
size_t frcnn_detect_post_workspace_bytes(int r, int num_classes, int batch);
int frcnn_detect_post(const float* cls_prob_dev, const float* pred_boxes_dev, const int* num_rois_dev, int r, int batch,
                      int num_classes, float score_thresh, float nms_thresh, unsigned flags,
                      int max_per_image, int max_det, float* det_dev, int* ndet_dev, int record_stride, int* keep_dev,
                      int* keep_cnt_dev, float* keep_score_dev, void* workspace_dev, size_t workspace_bytes, void* stream);
/* Soft-NMS (Bodla et al., ICCV 2017) in place of the greedy per-class NMS: an overlapping box has its score lowered instead of
 * being dropped.  An extension beyond the reference (Detectron's TEST.SOFT_NMS).  Per candidate list a[0..N) (each row
 * x1,y1,x2,y2,s):
 *   for i = 0, 1, ... while i < N:
 *     m = i; for q = i+1 .. N-1: if a[m].s < a[q].s: m = q   (the lowest position of the maximal score; a NaN score at i is
 *         selected at once, and otherwise NaN scores wait until only NaN scores are left)
 *     swap a[i], a[m]; p = i + 1
 *     while p < N: decay a[p] by a[i]; if a[p] overlapped a[i] and its new score < score_thresh: a[p] = a[N-1], N -= 1
 *                  (position p is examined again) else p += 1
 *   result: a[0..N) in this order with the decayed scores.
 * Decay of b by t, every step a separate fp32 round-to-nearest operation, '+1' pixel areas:
 *   iw = (min(t.x2,b.x2) - max(t.x1,b.x1)) + 1; if iw > 0: ih = (min(t.y2,b.y2) - max(t.y1,b.y1)) + 1; if ih > 0 they overlap:
 *   ov = (iw*ih) / ((area(t) + area(b)) - iw*ih), area(u) = ((u.x2-u.x1)+1) * ((u.y2-u.y1)+1), and b.s = weight * b.s with
 *   LINEAR: ov > nt ? 1 - ov : 1;  GAUSSIAN: RN_f32(exp_f64(-((ov*ov) / sigma)));  HARD: ov > nt ? 0 : 1.
 * A box that does not overlap is neither decayed nor pruned.  Output scores never increase from row to row and, with
 * score_thresh > 0, are > 0.  sigma > 0 and score_thresh > 0 are required (else FRCNN_ERR_ARG); capacity 8192 boxes. */
#define FRCNN_SOFT_NMS_LINEAR 0
#define FRCNN_SOFT_NMS_GAUSSIAN 1
#define FRCNN_SOFT_NMS_HARD 2
/* host buffers, synchronous, one set: the candidates are the n rows of dets_host [n, dim >= 5] in input order.  dets_out
 * [n, 5] receives the kept rows in selection order with decayed scores, keep_out [n] their row indices in dets_host, num_out
 * their count.  device_id < 0: the calling thread's current device; the caller's current device is left unchanged. */
int frcnn_soft_nms_host(float* dets_out, int* keep_out, int* num_out, const float* dets_host, int n, int dim, int method,
                        float sigma, float nt, float score_thresh, int device_id);
/* frcnn_detect_post with Soft-NMS as the per-class stage: per class j >= 1 the candidates are the rows with score > score_thresh
 * in ascending RoI order; keep / keep_cnt / keep_score hold the selection order and the decayed scores, and the max_per_image
 * cap and records follow as in frcnn_detect_post.  prune_thresh is Soft-NMS's score_thresh above, nt the overlap threshold.
 * workspace_dev is not used (the candidates fit in shared memory) and may be NULL. */
int frcnn_detect_post_soft(const float* cls_prob_dev, const float* pred_boxes_dev, const int* num_rois_dev, int r, int batch,
                           int num_classes, float score_thresh, int method, float sigma, float nt, float prune_thresh,
                           int max_per_image, int max_det, float* det_dev, int* ndet_dev, int record_stride, int* keep_dev,
                           int* keep_cnt_dev, float* keep_score_dev, void* workspace_dev, size_t workspace_bytes, void* stream);
/* Box voting (Detectron's TEST.BBOX_VOTE, box_voting) between the per-class NMS / Soft-NMS and the max_per_image cap: each kept
 * box is replaced by the score-weighted average of the candidates of its class that overlap it, and optionally so is its score.
 * An extension beyond the reference.  For one set, the top boxes t (the NMS / Soft-NMS output, with its scores) and the candidates
 * a[0..n) (the rows NMS started from, with their ORIGINAL scores s_a), every fp32 step a separate round-to-nearest operation:
 *   ov(t, a): iw = (min(t.x2,a.x2) - max(t.x1,a.x1)) + 1; if iw > 0: ih = (min(t.y2,a.y2) - max(t.y1,a.y1)) + 1; if ih > 0:
 *             ov = (iw*ih) / ((area(t) + area(a)) - iw*ih), area(u) = ((u.x2-u.x1)+1) * ((u.y2-u.y1)+1)  (Soft-NMS's overlap);
 *             otherwise ov = 0.
 *   V(t) = { a : ov(t, a) >= thresh }, n = |V(t)|, thresh in (0, 1].
 *   Sums over V(t) in fp64 (each fp32 product below is exact in fp64), in this order: candidate k goes to partial k mod 32, each
 *   partial adds its candidates in ascending k starting from +0, then the 32 partials P are combined by the butterfly
 *   P[l] = P[l] + P[l ^ o] for o = 16, 8, 4, 2, 1 (every l at once), and the result is P[0]:
 *     S = sum s_a;  X1 = sum s_a*a.x1 (and Y1, X2, Y2);
 *     IOU_AVG: M0 = sum ov*s_a, M1 = sum ov;  GENERALIZED_AVG: M0 = sum exp(beta*s_a);
 *     TEMP_AVG: M0 = sum e0/(e0+e1), q = 1-s_a, m = max(s_a, q), e0 = exp(log(s_a/m)/beta), e1 = exp(log(q/m)/beta).
 *   Box: (X1/S, Y1/S, X2/S, Y2/S), each an fp64 division rounded once to fp32.
 *   Score, computed in fp64 and rounded once to fp32:  ID: unchanged (the NMS / Soft-NMS score);  AVG: S/n;  IOU_AVG: M0/M1;
 *     GENERALIZED_AVG: log(M0/n)/beta;  QUASI_SUM: S/n^beta;  TEMP_AVG: M0/n  (beta finite and > 0).  n^beta is n for beta 1,
 *     n*n for beta 2 and sqrt(n) for beta 0.5 (all exact or correctly rounded), else pow(n, beta).  exp, log and pow are the fp64
 *     library functions, within an ulp or two of the exact value, so an output may differ from another libm's in its last bit.
 *   Choices of this implementation: n = 0 (possible through frcnn_box_vote_host only: on the post path every top box is a
 *   candidate and overlaps itself with ov = 1) keeps the box and the score, where Detectron divides by zero; S = 0 (zero scores)
 *   keeps the box.  Detectron accumulates in float32; these fp64 sums are at least as accurate.
 * In the post entries the candidates are the stage's own (score > score_thresh, ascending RoI order) and the top boxes the kept
 * list keep / keep_score [0, keep_cnt) of each class.  For every method except ID each class list is then re-sorted stably by
 * descending voted score (ties keep the NMS order), so that it is again sorted by descending score, which the cap needs: the cap
 * counts scores >= t by binary search and finds the max_per_image-th score by a bitwise search on the fp32 pattern, valid when
 * every score is >= +0.  Voted scores are: AVG, QUASI_SUM > 0 (positive scores); IOU_AVG > 0 (ov >= thresh > 0); GENERALIZED_AVG
 * = log(mean(exp(beta*s)))/beta >= log(1)/beta = +0; TEMP_AVG a mean of e0/(e0+e1) in [+0, 1] -- never -0 and never NaN for
 * scores in [0, 1] and beta > 0.  The record set after the cap equals Detectron's (vote, then cap); only the row order within a
 * class is the voted-score order instead of Detectron's NMS order. */
#define FRCNN_BOX_VOTE_ID 0
#define FRCNN_BOX_VOTE_AVG 1
#define FRCNN_BOX_VOTE_IOU_AVG 2
#define FRCNN_BOX_VOTE_GENERALIZED_AVG 3
#define FRCNN_BOX_VOTE_QUASI_SUM 4
#define FRCNN_BOX_VOTE_TEMP_AVG 5
/* host buffers, synchronous, one set: top_host [n_top, top_dim >= 5] and all_host [n_all, all_dim >= 5] rows (x1, y1, x2, y2,
 * score, ...).  dets_out [n_top, 5] = the voted rows in top_host's row order (no re-sort).  n_all <= 8192 (else
 * FRCNN_ERR_CAPACITY).  An unknown method, thresh outside (0, 1] or beta not finite and > 0 give FRCNN_ERR_ARG.  device_id < 0:
 * the calling thread's current device; the caller's current device is left unchanged. */
int frcnn_box_vote_host(float* dets_out, const float* top_host, int n_top, int top_dim, const float* all_host, int n_all,
                        int all_dim, float thresh, int method, float beta, int device_id);
/* frcnn_detect_post / frcnn_detect_post_soft with box voting between the per-class stage and the cap.  vote_box_dev [batch, C, r]
 * float4 (16-byte aligned): entry (b, c, j) = the voted box of keep_dev[b, c, j] for j < the class's count before the cap; the
 * records take their boxes from it.  keep_score_dev holds the voted scores and keep_dev the re-sorted order (methods other than
 * ID), so frcnn_detect_features stays consistent with the record rows. */
int frcnn_detect_post_vote(const float* cls_prob_dev, const float* pred_boxes_dev, const int* num_rois_dev, int r, int batch,
                           int num_classes, float score_thresh, float nms_thresh, unsigned flags, int max_per_image, int max_det,
                           float* det_dev, int* ndet_dev, int record_stride, int* keep_dev, int* keep_cnt_dev, float* keep_score_dev,
                           void* workspace_dev, size_t workspace_bytes, float vote_thresh, int vote_method, float vote_beta,
                           float* vote_box_dev, void* stream);
int frcnn_detect_post_soft_vote(const float* cls_prob_dev, const float* pred_boxes_dev, const int* num_rois_dev, int r, int batch,
                                int num_classes, float score_thresh, int method, float sigma, float nt, float prune_thresh,
                                int max_per_image, int max_det, float* det_dev, int* ndet_dev, int record_stride, int* keep_dev,
                                int* keep_cnt_dev, float* keep_score_dev, void* workspace_dev, size_t workspace_bytes,
                                float vote_thresh, int vote_method, float vote_beta, float* vote_box_dev, void* stream);
/* per-detection head features, run after frcnn_detect_post on the same keep_dev / keep_cnt_dev: slot k of image b is record
 * row k of that image (classes ascending, slot = prefix(keep_cnt)[c] + j, slot < max_det).  fc7_dev [batch*r, feat_dim] is the
 * head output the class / box FC read (feat_dim % 4 == 0, 16-byte aligned).  roi_out_dev int32 [batch, max_det] = RoI index
 * within the image, -1 past the image's detection count; feat_out_dev [batch, max_det, feat_dim] = fc7 row of that RoI, zeros
 * past the count.  2 <= C <= 4096 and r * C must fit in int (else FRCNN_ERR_ARG). */
int frcnn_detect_features(const int* keep_dev, const int* keep_cnt_dev, const float* fc7_dev, int r, int batch, int num_classes,
                          int feat_dim, int max_det, float* feat_out_dev, int* roi_out_dev, void* stream);
/* Bottom-up regions (Anderson et al. 2018, the protocol of bottom-up-attention's generate_tsv.py), an extension beyond the
 * reference: per image a set of DISTINCT RoIs, each ranked by its best class confidence after per-class NMS, with its unregressed
 * box and its head feature.  Per image b, over the valid rows i < nr = min(num_rois[b], r):
 *   1. box_i = rois[i, 1:5] / scale_b, one fp32 round-to-nearest division per coordinate (scale_b = im_meta[b, 0]; the division of
 *      frcnn_bbox_decode, no regression, no clipping).
 *   2. For each class c = 1..C-1: greedy NMS over ALL nr rows (no score threshold) with boxes box_i and scores cls_prob[i, c],
 *      threshold nms_thresh and predicate `flags` as in frcnn_detect_post; order: score descending, ties to the lower row.
 *   3. conf_i = max of cls_prob[i, c] over the classes c whose NMS kept i, 0 if none kept it; class_i = the lowest such c reaching
 *      conf_i, and 0 when conf_i is 0.
 *   4. count = #{i : conf_i >= conf_thresh}, an fp32 comparison (a caller holding a float64 threshold passes the smallest fp32 not
 *      below it, which gives the float64 comparison's result for every fp32 conf_i).  If min_boxes <= count <= max_boxes the
 *      regions are those rows in ascending row order; otherwise the first min(max(count, min_boxes), max_boxes, nr) rows in
 *      descending conf_i, ties to the lower row.
 *   5. Region k of image b: boxes_out[b, k] = box_i, conf_out[b, k] = conf_i, class_out[b, k] = class_i, index_out[b, k] = i,
 *      feat_out[b, k] = fc7 row i; count_out[b] = the number of regions.  Rows k >= count_out[b] are zeros with index -1.
 * cls_prob entries must be >= +0 (softmax outputs).  Requirements: 2 <= C <= 4096, r <= 8192, r * batch fits in int,
 * conf_thresh in [0, 1], 0 <= min_boxes <= max_boxes, max_boxes >= 1, feat_dim % 4 == 0.
 * Two implementations of step 2, chosen by C; both give the definition's result bit for bit:
 *   C <= 1024: per-class NMS kernels (the post stage's) over the boxes broadcast to every class, then a fold of the kept lists;
 *   C >  1024: one overlap bitmask per image (bit j of row i: does box_i suppress box_j; r * ceil(r/32) 32-bit words), then one greedy
 *              walk of that mask per (class, image) in the class's score order.
 * Buffers (M = min(max_boxes, r)):
 *   inputs  cls_prob_dev [batch*r, C], rois_dev [batch*r, 5], num_rois_dev int32 [batch], im_meta_dev [batch, 3] (as for
 *           frcnn_bbox_decode), fc7_dev [batch*r, feat_dim] (16-byte aligned);
 *   scratch C <= 1024: keep_dev / keep_cnt_dev / keep_score_dev and workspace_dev as for frcnn_detect_post (they receive the
 *             per-class NMS of step 2, uncapped); roi_box_dev [batch*r, C, 4] fp32;
 *           C > 1024: keep_dev / keep_cnt_dev / keep_score_dev are not used and may be NULL; workspace_dev (4-byte aligned) holds the
 *             masks, batch * r * ceil(r/32) * 4 bytes; roi_box_dev [batch*r, 4] fp32;
 *           both: workspace_bytes >= the frcnn_detect_regions_workspace_bytes of (r, C, batch) (at C <= 1024 that is
 *             frcnn_detect_post_workspace_bytes, and the workspace may be NULL when r <= 1024); roi_box_dev 16-byte aligned;
 *             key_dev uint64 [batch*r] (8-byte aligned);
 *   outputs boxes_out_dev [batch, M, 4] (16-byte aligned), conf_out_dev [batch, M], class_out_dev int32 [batch, M], index_out_dev
 *           int32 [batch, M], feat_out_dev [batch, M, feat_dim] (16-byte aligned), count_out_dev int32 [batch].
 * No allocation or synchronisation: capturable into a CUDA graph. */
/* *bytes = the workspace frcnn_detect_regions needs for (r, C, batch); FRCNN_ERR_ARG outside its requirements */
int frcnn_detect_regions_workspace_bytes(int r, int num_classes, int batch, size_t* bytes);
int frcnn_detect_regions(const float* cls_prob_dev, const float* rois_dev, const int* num_rois_dev, const float* im_meta_dev,
                         const float* fc7_dev, int r, int batch, int num_classes, int feat_dim, float nms_thresh, unsigned flags,
                         float conf_thresh, int min_boxes, int max_boxes, int* keep_dev, int* keep_cnt_dev, float* keep_score_dev,
                         void* workspace_dev, size_t workspace_bytes, float* roi_box_dev, unsigned long long* key_dev,
                         float* boxes_out_dev, float* conf_out_dev, int* class_out_dev, int* index_out_dev, float* feat_out_dev,
                         int* count_out_dev, void* stream);
/* Attribute head of the bottom-up regions (the Visual Genome model of Anderson et al. 2018: C = 1601 object classes, A = 401
 * attribute classes with 0 = "no attribute"), an extension beyond the reference.  Per RoI, with F the fc7 width, E the embedding
 * width and H the hidden width:
 *   1. c = argmax of the RoI's class logits cls_score[i, 0..C) (background included), numpy's rule: the first NaN column if the
 *      row holds one, else the first column holding the maximum;
 *   2. e = cls_embedding[c] (a [C, E] table);
 *   3. h = relu([fc7_i ; e] . W_fc_attr + b_fc_attr), fc7 first, W_fc_attr [F + E, H];
 *   4. s = h . W_attr_score + b_attr_score (A logits), attr_prob = softmax(s);
 *   5. attributes = 1 + argmax(attr_prob[1..A)) (the same argmax rule), attr_conf = attr_prob[attributes].
 * It is computed on the M = min(max_boxes, r) region rows per image of frcnn_detect_regions (its index_out_dev / count_out_dev).
 * Rows k >= count[b] are padding: emb zeros, attr_prob 0, attributes -1, attr_conf 0.  Steps 3 and 4 are two frcnn_conv_plan
 * FCs (step 3 with the embedding as the second A source, in2_dev); the two entries below are steps 1-2 and the softmax plus
 * step 5.  Both check their arguments before any CUDA call (FRCNN_ERR_ARG), allocate nothing and are capturable into a CUDA
 * graph.
 *
 * Steps 1-2: cls_score_dev [batch*r, C] (frcnn_cls_finish's logits); index_dev / count_dev int32 [batch, M] / [batch] (region k
 * of image b is RoI index[b, k] of that image; a row k < count whose index lies outside [0, r) is written as zeros);
 * embedding_dev [C, embed_dim] -> emb_out_dev [batch*M, embed_dim], row b*M + k = embedding row c of that RoI.  Requirements:
 * 2 <= C <= 4096, 1 <= M <= r, batch >= 1, embed_dim a positive multiple of 4, embedding_dev and emb_out_dev 16-byte aligned. */
int frcnn_regions_attr_embed(const float* cls_score_dev, int r, int batch, int num_classes, const int* index_dev, const int* count_dev,
                             int max_regions, const float* embedding_dev, int embed_dim, float* emb_out_dev, void* stream);
/* Steps 4 (softmax) and 5: score_dev [batch*M, ld] attribute logits (columns A .. ld-1 are not read); per row, with
 * frcnn_cls_finish's arithmetic: m = max of the A logits (fmaxf), e_j = expf(fl(s_j - m)), S = their sum (lane j mod 32 adds its
 * columns in ascending order from +0, then 5 xor-shuffle adds), attr_prob_j = fl(e_j / S).  attributes_dev int32 [batch*M] and
 * attr_conf_dev [batch*M] by step 5 on these fp32 probabilities; attr_prob_dev [batch*M, A].  Requirements: 2 <= A <= 4096,
 * ld >= A, batch >= 1, M >= 1, every buffer 4-byte aligned. */
int frcnn_attr_finish(const float* score_dev, int ld, int batch, int max_regions, int num_attributes, const int* count_dev,
                      float* attr_prob_dev, int* attributes_dev, float* attr_conf_dev, void* stream);
/* caller boxes -> RoI rows (the Fast R-CNN mode: TEST.HAS_RPN = False).  boxes_dev [batch, cap, 4] fp32 (x1,y1,x2,y2) in
 * ORIGINAL-image pixels; counts_dev int32 [batch]; im_meta_dev [batch, 3] as for frcnn_bbox_decode.  rois_dev [batch*cap, 5] =
 * (b, x1*s, y1*s, x2*s, y2*s), one fp32 multiply by im_meta's scale per coordinate, zeros past the count; num_rois_dev int32
 * [batch] = min(count, cap).  No clipping: crop_and_resize samples outside the feature map as 0. */
int frcnn_boxes_to_rois(const float* boxes_dev, const int* counts_dev, const float* im_meta_dev, int batch, int cap,
                        float* rois_dev, int* num_rois_dev, void* stream);

/* ---- test-time augmentation (Detectron's TEST.BBOX_AUG, union mode) -- an extension beyond the reference ----
 * A view is a pair (scale, flip): the base view (TEST.SCALES[0], TEST.MAX_SIZE), one view per TEST.BBOX_AUG.SCALES entry
 * (capped by TEST.BBOX_AUG.MAX_SIZE, the resize rule of _get_image_blob), and with H_FLIP the mirrored twin of each.  A mirrored
 * view is the blob of img[:, ::-1] (frcnn_preprocess_hflip).  Each view runs the unchanged network and im_detect tail
 * (frcnn_bbox_decode, one-sided clip); frcnn_aug_union then merges the views, and the unchanged frcnn_detect_post /
 * frcnn_detect_post_soft run on the union (r = R_union = sum of the views' rows, <= 8192).
 * Union of image b, in view order (the caller's order; the Python layer uses Detectron's: flipped base, then each extra scale
 * followed by its flip, the base view last), the valid rows [0, n_v) of view v with n_v = clamp(num_rois_v[b], 0, R_v):
 *   union row off_v + i = view row i (i < n_v), off_v = n_0 + ... + n_{v-1}; rows past the total are zero;
 *   cls_prob copied; pred_boxes copied, and for a mirrored view un-flipped with W = orig_w of im_meta_dev[b] (fp32, two
 *   roundings each): x1 = (W - x2') - 1, x2 = (W - x1') - 1, y unchanged;  num_rois_dev[b] = sum of n_v.
 * Host arrays of num_views (<= FRCNN_AUG_MAX_VIEWS) entries: the views' device pointers cls_prob [batch, R_v, C], pred_boxes
 * [batch, R_v, 4C] (16-byte aligned), num_rois int32 [batch]; rois_per_view R_v > 0; flip_views 0 / 1.  im_meta_dev [batch, 3] as
 * for frcnn_bbox_decode.  Outputs: cls_prob_dev [batch, R_union, C], pred_boxes_dev [batch, R_union, 4C], num_rois_dev int32
 * [batch].  The pointers are copied into the kernel's parameters, so the launch is CUDA-graph capturable. */
#define FRCNN_AUG_MAX_VIEWS 16
int frcnn_aug_union(const float* const* cls_prob_views, const float* const* pred_boxes_views, const int* const* num_rois_views,
                    const int* rois_per_view, const int* flip_views, int num_views, int batch, int num_classes,
                    const float* im_meta_dev, float* cls_prob_dev, float* pred_boxes_dev, int* num_rois_dev, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* FRCNN_B200_H_ */
