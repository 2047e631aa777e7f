"""Stage-level Python entry points over the C ABI.  torch is used ONLY for device memory
(`torch.empty(..., device='cuda')`, `.data_ptr()`) and the current CUDA stream; every op below
launches hand-written sm_90a kernels from libfrcnn_b200.so.  No CPU fallbacks.
"""
import ctypes as C
import os

import numpy as np
import torch

from . import _native as N


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _f32(t):
    assert t.dtype == torch.float32 and t.is_cuda and t.is_contiguous(), "expected contiguous cuda fp32"
    return t


def zeros(shape, dtype=torch.float32):
    """Device buffer cleared with cudaMemsetAsync on the current stream (no framework fill kernel on the path)."""
    t = torch.empty(shape, dtype=dtype, device="cuda")
    N.check(N.lib().frcnn_zero_async(_p(t), t.numel() * t.element_size(), _stream()), "zero_async")
    return t


def same_pads(n, k, s):
    """TF 'SAME' padding (before, after) for one dimension."""
    out = -(-n // s)
    total = max((out - 1) * s + k - n, 0)
    return total // 2, total - total // 2


def conv_impl():
    """Dense-kernel arithmetic (FRCNN_CONV_IMPL): 'f16' = FP16x3, fp32-grade (default); 'tf32' = the TF32x3 mode (A/B
    measurements); 'f16x1' = THROUGHPUT mode, plain fp16 operands with fp32 accumulation (NOT fp32-grade: ~3e-4 per layer)."""
    return {"tf32": N.CONV_TF32X3, "f16x1": N.CONV_F16X1}.get(os.environ.get("FRCNN_CONV_IMPL", "f16"), N.CONV_F16X3)


def weight_exponent(w):
    """wexp with max|w| * 2^wexp in [2^13, 2^14): the fp16 hi plane then spans 27 binades below the layer's largest
    weight before going subnormal (and even those keep 2^-35 * max|w| through the lo plane)."""
    m = float(np.max(np.abs(w))) if w.size else 0.0
    if not np.isfinite(m) or m <= 0.0:
        return 0
    return int(13 - np.floor(np.log2(m)))


class PackedConv:
    """Device-resident K-major hi/lo weight planes + epilogue vectors of one conv / FC layer."""

    def __init__(self, w_hwio, scale=None, shift=None, impl=None):
        wnp = np.ascontiguousarray(w_hwio, dtype=np.float32)
        w = torch.from_numpy(wnp).cuda()
        if w.dim() == 2:                     # FC [in,out] == 1x1 conv
            w = w.view(1, 1, w.shape[0], w.shape[1])
        self.kh, self.kw, self.cin, self.cout = (int(v) for v in w.shape)
        ktot = self.kh * self.kw * self.cin
        self.impl = conv_impl() if impl is None else impl
        if self.impl in (N.CONV_F16X3, N.CONV_F16X1):
            self.wexp = weight_exponent(wnp)
            self.out_mult = float(np.ldexp(1.0, -self.wexp))
            self.w_hi = torch.empty((self.cout, ktot), dtype=torch.float16, device="cuda")
            self.w_lo = torch.empty_like(self.w_hi)
            N.check(N.lib().frcnn_pack_conv_weights(_p(w), _p(self.w_hi), _p(self.w_lo), self.kh, self.kw, self.cin,
                                                    self.cout, self.wexp, _stream()), "pack_conv_weights")
        else:
            self.wexp, self.out_mult = 0, 1.0
            self.w_hi = torch.empty((self.cout, ktot), dtype=torch.float32, device="cuda")
            self.w_lo = torch.empty_like(self.w_hi)
            N.check(N.lib().frcnn_pack_conv_weights_tf32(_p(w), _p(self.w_hi), _p(self.w_lo), self.kh, self.kw, self.cin,
                                                         self.cout, _stream()), "pack_conv_weights_tf32")
        torch.cuda.current_stream().synchronize()
        self.scale = None if scale is None else torch.as_tensor(np.ascontiguousarray(scale), dtype=torch.float32).cuda()
        self.shift = None if shift is None else torch.as_tensor(np.ascontiguousarray(shift), dtype=torch.float32).cuda()


def concat_scaled_weights(ws, scales):
    """[W_1 diag(s_1) ; W_2 diag(s_2) ; ...] for 1x1 layers summed into one output: HWIO [1, 1, cin_i, cout] weights, each
    times its per-output-channel scale (None = 1) in fp32, stacked along cin -> HWIO [1, 1, sum cin_i, cout] fp32."""
    parts = []
    for w, s in zip(ws, scales):
        w = np.asarray(w, dtype=np.float32)
        assert w.ndim == 4 and w.shape[:2] == (1, 1), w.shape
        parts.append(w if s is None else (w * np.asarray(s, dtype=np.float32)).astype(np.float32))
    return np.ascontiguousarray(np.concatenate(parts, axis=2))


def column_scales(w):
    """Per output channel (last axis) the power of two sigma_c with max_k |w[..., c]| / sigma_c in [1, 2); 1 for a column
    that is all zero or holds a non-finite value.  Dividing a column by its sigma_c and multiplying the epilogue scale by it
    are both exact, and every column then spans the same binades of the f16 split as the layer's largest weight."""
    m = np.max(np.abs(np.asarray(w, np.float32)).reshape(-1, w.shape[-1]), axis=0) if w.size else np.zeros(w.shape[-1], np.float32)
    ok = np.isfinite(m) & (m > 0)
    _, e = np.frexp(np.where(ok, m, 1.0).astype(np.float32))        # m = f * 2^e, f in [0.5, 1)
    return np.where(ok, np.ldexp(np.float32(1.0), e - 1), 1.0).astype(np.float32)


class ConvPlan:
    """frcnn_conv_plan bound to fixed input/output/residual buffers (TMA descriptors hold raw pointers).

    x2: second A source of a pointwise layer (pc packs [cin + cin2] input channels; x2 holds the last cin2).
    mean: out is [n, cout], the mean over each image's h*w activated outputs (pointwise layers), computed in the epilogue."""

    def __init__(self, x, pc, out, stride=1, pad_t=0, pad_l=0, act=N.ACT_NONE, residual=None, block_n=0, kb_per_chunk=0, split_k=0,
                 x2=None, mean=False):
        _f32(x); _f32(out)
        n, h, w, cin = x.shape
        cin2 = 0
        if x2 is not None:
            _f32(x2)
            assert x2.shape[:3] == x.shape[:3], (x2.shape, x.shape)
            cin2 = int(x2.shape[3])
        assert cin + cin2 == pc.cin, (cin, cin2, pc.cin)
        if mean:
            ho, wo = h, w
            assert tuple(out.shape) == (n, pc.cout), (out.shape, n, pc.cout)
        else:
            no, ho, wo, co = out.shape
            assert no == n and co == pc.cout
        d = N.ConvDesc(_p(x), _p(pc.w_hi), _p(pc.w_lo), _p(pc.scale), _p(pc.shift), _p(residual), _p(None if mean else out),
                       n, h, w, cin, pc.cout, pc.kh, pc.kw, stride, pad_t, pad_l, ho, wo, act, block_n, kb_per_chunk, split_k,
                       pc.impl, pc.out_mult, _p(x2), cin2, _p(out if mean else None), h * w if mean else 0)
        self._h = C.c_void_p()
        N.check(N.lib().frcnn_conv_plan_create(C.byref(self._h), C.byref(d)), "conv_plan_create")
        self._keep = (x, pc, out, residual, x2)
        self.flops = 2.0 * n * ho * wo * pc.cout * pc.kh * pc.kw * pc.cin

    def run(self):
        N.check(N.lib().frcnn_conv_plan_run(self._h, _stream()), "conv_plan_run")

    def info(self):
        v = [C.c_int() for _ in range(8)]
        N.check(N.lib().frcnn_conv_plan_info(self._h, *[C.byref(a) for a in v]), "conv_plan_info")
        return dict(zip(["block_n", "tile_n", "tile_h", "tile_w", "grid_m", "grid_n", "splits", "smem"], [a.value for a in v]))

    def __del__(self):
        try:
            if self._h:
                N.lib().frcnn_conv_plan_destroy(self._h)
                self._h = C.c_void_p()
        except Exception:
            pass


def conv_out_hw(h, w, k, stride, mode):
    """mode 'SAME' (TF) or 'EXPLICIT' (slim conv2d_same: pad (k-1)//2 before, rest after, then VALID)."""
    if mode == "SAME":
        pt, _ = same_pads(h, k, stride)
        pl, _ = same_pads(w, k, stride)
        return -(-h // stride), -(-w // stride), pt, pl
    pb = (k - 1) // 2
    return (h + k - 1 - k) // stride + 1, (w + k - 1 - k) // stride + 1, pb, pb


def conv_first(x, w_hwio_dev, scale, shift, out, k, stride, pad_t, pad_l, act):
    n, h, w, _ = x.shape
    _, ho, wo, co = out.shape
    N.check(N.lib().frcnn_conv_first(_p(_f32(x)), _p(w_hwio_dev), _p(scale), _p(shift), _p(_f32(out)), n, h, w, co, k, stride,
                                     pad_t, pad_l, ho, wo, act, _stream()), "conv_first")


def depthwise3x3(x, w_dev, scale, shift, out, stride, pad_t, pad_l, act):
    n, h, w, c = x.shape
    _, ho, wo, _ = out.shape
    N.check(N.lib().frcnn_depthwise3x3(_p(_f32(x)), _p(w_dev), _p(scale), _p(shift), _p(_f32(out)), n, h, w, c, stride, pad_t,
                                       pad_l, ho, wo, act, _stream()), "depthwise3x3")


def max_pool(x, out, k, stride, pad_t, pad_l, pad_is_neg_inf):
    n, h, w, c = x.shape
    _, ho, wo, _ = out.shape
    N.check(N.lib().frcnn_max_pool(_p(_f32(x)), _p(_f32(out)), n, h, w, c, k, stride, pad_t, pad_l, ho, wo,
                                   int(pad_is_neg_inf), _stream()), "max_pool")


def spatial_mean(x, out):
    r, hw, c = x.shape[0], x.shape[1] * x.shape[2], x.shape[3]
    N.check(N.lib().frcnn_spatial_mean(_p(_f32(x)), _p(_f32(out)), r, hw, c, _stream()), "spatial_mean")


def preprocess(img_u8_dev, means3, fx, fy, blob, hflip=False):
    """uint8 BGR [h0,w0,3] (device) -> mean-subtracted, bilinearly resized fp32 blob [1,H,W,3] (device).  hflip: the blob of the
    mirrored image img[:, ::-1] (test-time augmentation's flipped view)."""
    h0, w0, _ = img_u8_dev.shape
    _, H, W, _ = blob.shape
    assert blob.is_contiguous()
    m = (C.c_double * 3)(*[float(v) for v in means3])
    fn = N.lib().frcnn_preprocess_hflip if hflip else N.lib().frcnn_preprocess
    N.check(fn(C.c_void_p(img_u8_dev.data_ptr()), h0, w0, m, float(fx), float(fy), _p(blob), H, W, _stream()),
            "preprocess_hflip" if hflip else "preprocess")


def rpn_decode(rpn_out, delta_col, base_anchors, num_anchors, fh, fw, im_h, im_w, scores, props, feat_stride=16, batch=1):
    """rpn_out: [batch*fh*fw, ld] rows of the fused RPN head."""
    ld = rpn_out.shape[-1]
    N.check(N.lib().frcnn_rpn_decode(_p(_f32(rpn_out)), ld, delta_col, _p(base_anchors), num_anchors, batch, fh, fw, feat_stride,
                                     float(im_h), float(im_w), _p(scores), _p(props), _stream()), "rpn_decode")


def sort_workspace(n):
    return torch.empty(int(N.lib().frcnn_sort_workspace_bytes(n)), dtype=torch.uint8, device="cuda")


def sort_desc(keys, order, sorted_keys, workspace=None, batch=1):
    """`batch` segments of keys.numel() // batch keys each; order = segment-local indices."""
    n = keys.numel() // batch
    N.check(N.lib().frcnn_sort_desc(_p(_f32(keys)), n, batch, _p(order), _p(sorted_keys), _p(workspace),
                                    0 if workspace is None else workspace.numel(), _stream()), "sort_desc")


def proposals(props, scores, order, pre_nms_top_n, post_nms_top_n, thresh, flags, rois, roi_scores, keep, num, batch=1):
    n = scores.numel() // batch
    N.check(N.lib().frcnn_proposals(_p(props), _p(scores), _p(order), n, batch, pre_nms_top_n, post_nms_top_n, float(thresh), flags,
                                    _p(rois), _p(roi_scores), _p(keep), _p(num), _stream()), "proposals")


def crop_pool(feat, rois, pooled, pre_pool, out):
    """rois[:, 0] = index of the image (of feat's batch dimension) the box is cut from."""
    b, fh, fw, c = feat.shape
    r = rois.shape[0]
    N.check(N.lib().frcnn_crop_pool(_p(_f32(feat)), b, fh, fw, c, _p(_f32(rois)), r, pooled, int(pre_pool), _p(_f32(out)), _stream()),
            "crop_pool")


def roi_align(feat, rois, pooled, spatial_scale, sampling_ratio, aligned, out):
    """torchvision.ops.roi_align on NHWC: feat [B,H,W,C], rois [R,5] (image index, x1, y1, x2, y2) -> out [R,pooled,pooled,C]."""
    b, fh, fw, c = feat.shape
    N.check(N.lib().frcnn_roi_align(_p(_f32(feat)), b, fh, fw, c, _p(_f32(rois)), rois.shape[0], pooled, float(spatial_scale),
                                    int(sampling_ratio), int(bool(aligned)), _p(_f32(out)), _stream()), "roi_align")


def roi_pool(feat, rois, pooled, spatial_scale, out):
    """torchvision.ops.roi_pool on NHWC: feat [B,H,W,C], rois [R,5] (image index, x1, y1, x2, y2) -> out [R,pooled,pooled,C]."""
    b, fh, fw, c = feat.shape
    N.check(N.lib().frcnn_roi_pool(_p(_f32(feat)), b, fh, fw, c, _p(_f32(rois)), rois.shape[0], pooled, float(spatial_scale),
                                   _p(_f32(out)), _stream()), "roi_pool")


def cls_finish(head_out, num_classes, stds, means, cls_score, cls_prob, bbox_pred):
    r, ld = head_out.shape
    s4 = (C.c_float * 4)(*[float(v) for v in stds])
    m4 = (C.c_float * 4)(*[float(v) for v in means])
    N.check(N.lib().frcnn_cls_finish(_p(_f32(head_out)), ld, r, num_classes, s4, m4, _p(cls_score), _p(cls_prob), _p(bbox_pred),
                                     _stream()), "cls_finish")


def im_meta_tensor(rows):
    """[(im_scale, orig_h, orig_w), ...] -> device fp32 [batch, 3] (the per-image scalars bbox_decode reads)."""
    return torch.tensor([[float(np.float32(s)), float(h), float(w)] for s, h, w in rows], dtype=torch.float32).cuda()


def bbox_decode(rois, bbox_pred, num_classes, im_meta, pred_boxes):
    """im_meta: device fp32 [batch, 3] (im_scale, orig_h, orig_w); rois[:, 0] selects the row."""
    r = rois.shape[0]
    N.check(N.lib().frcnn_bbox_decode(_p(_f32(rois)), _p(_f32(bbox_pred)), r, num_classes, im_meta.shape[0], _p(_f32(im_meta)),
                                      _p(pred_boxes), _stream()), "bbox_decode")


def detect_post_workspace(r, num_classes, batch=1):
    return torch.empty(int(N.lib().frcnn_detect_post_workspace_bytes(r, num_classes, batch)), dtype=torch.uint8, device="cuda")


def _record_stride(det, ndet):
    """record_stride of the post entries: 0 for a packed det [batch, max_det, 6] beside its own ndet; for det rows inside
    record buffers (image b's record = int32 count ndet[b], then its rows det[b]) the distance between two records, in floats."""
    if det.dim() == 2 or det.stride(0) == det.shape[1] * 6:
        return 0
    assert det.stride()[1:] == (6, 1) and ndet.stride(0) == det.stride(0), "det / ndet are not views of one record buffer"
    return det.stride(0)


def _vote_args(vote, keep):
    """vote = (thresh, method, beta, vote_box): fp32 threshold, FRCNN_BOX_VOTE_* code, fp32 beta (engine.box_vote_args) and the
    [batch, C, r, 4] fp32 buffer of the voted boxes -> the trailing C arguments of the _vote entries."""
    thresh, method, beta, vote_box = vote
    assert vote_box.dtype == torch.float32 and vote_box.is_contiguous() and vote_box.shape == (*keep.shape, 4), "vote_box [batch, C, r, 4]"
    return float(thresh), int(method), float(beta), _p(vote_box)


def detect_post(cls_prob, pred_boxes, num_rois, num_classes, score_thresh, nms_thresh, flags, max_per_image, det, ndet, keep,
                keep_cnt, keep_score, workspace=None, batch=1, vote=None):
    """cls_prob [batch*r, C]; det [batch, max_det, 6] (or [max_det, 6] for batch 1); ndet int32 [batch] = TRUE counts
    (a count above max_det means the records did not fit).  det and ndet may be views of record buffers (_record_stride).
    vote: None, or (thresh, method, beta, vote_box) for box voting ahead of the cap (frcnn_detect_post_vote)."""
    r = cls_prob.shape[0] // batch
    max_det = det.shape[-2]
    args = (_p(cls_prob), _p(pred_boxes), _p(num_rois), r, batch, num_classes, float(score_thresh), float(nms_thresh), flags, max_per_image,
            max_det, _p(det), _p(ndet), _record_stride(det, ndet), _p(keep), _p(keep_cnt), _p(keep_score), _p(workspace),
            0 if workspace is None else workspace.numel())
    if vote is None:
        N.check(N.lib().frcnn_detect_post(*args, _stream()), "detect_post")
    else:
        N.check(N.lib().frcnn_detect_post_vote(*args, *_vote_args(vote, keep), _stream()), "detect_post_vote")


def detect_post_soft(cls_prob, pred_boxes, num_rois, num_classes, score_thresh, method, sigma, nt, prune_thresh, max_per_image, det,
                     ndet, keep, keep_cnt, keep_score, batch=1, vote=None):
    """detect_post with Soft-NMS as the per-class stage; method is an FRCNN_SOFT_NMS_* code (N.SOFT_NMS_METHODS).  vote: as for
    detect_post (frcnn_detect_post_soft_vote)."""
    r = cls_prob.shape[0] // batch
    max_det = det.shape[-2]
    args = (_p(cls_prob), _p(pred_boxes), _p(num_rois), r, batch, num_classes, float(score_thresh), int(method), float(sigma), float(nt),
            float(prune_thresh), max_per_image, max_det, _p(det), _p(ndet), _record_stride(det, ndet), _p(keep), _p(keep_cnt),
            _p(keep_score), None, 0)
    if vote is None:
        N.check(N.lib().frcnn_detect_post_soft(*args, _stream()), "detect_post_soft")
    else:
        N.check(N.lib().frcnn_detect_post_soft_vote(*args, *_vote_args(vote, keep), _stream()), "detect_post_soft_vote")


def detect_features(keep, keep_cnt, fc7, num_classes, feat_out, roi_out):
    """After detect_post: keep [batch, C, r], keep_cnt [batch, C] (the capped lists), fc7 [batch*r, F] ->
    feat_out [batch, max_det, F] = fc7 row of record slot k, roi_out int32 [batch, max_det] (-1 past the count)."""
    batch, max_det, fdim = feat_out.shape
    r = keep.shape[-1]
    N.check(N.lib().frcnn_detect_features(_p(keep), _p(keep_cnt), _p(_f32(fc7)), r, batch, num_classes, fdim, max_det, _p(_f32(feat_out)),
                                          _p(roi_out), _stream()), "detect_features")


# frcnn_detect_regions runs the per-class NMS up to this many classes and the per-image overlap mask above (include/frcnn_b200.h)
REGIONS_CLASS_NMS_MAX = 1024


def regions_box_shape(rows, num_classes):
    """Shape of detect_regions' roi_box scratch: the RoI box broadcast to every class, or one box per row on the mask path."""
    return (rows, num_classes, 4) if num_classes <= REGIONS_CLASS_NMS_MAX else (rows, 4)


def detect_regions_workspace_bytes(r, num_classes, batch=1):
    n = C.c_size_t(0)
    N.check(N.lib().frcnn_detect_regions_workspace_bytes(r, num_classes, batch, C.byref(n)), "detect_regions_workspace_bytes")
    return n.value


def detect_regions_workspace(r, num_classes, batch=1):
    return torch.empty(detect_regions_workspace_bytes(r, num_classes, batch), dtype=torch.uint8, device="cuda")


def detect_regions(cls_prob, rois, num_rois, im_meta, fc7, num_classes, nms_thresh, flags, conf_thresh, min_boxes, max_boxes, keep,
                   keep_cnt, keep_score, workspace, roi_box, key, out, batch=1):
    """Bottom-up regions (frcnn_detect_regions): cls_prob [batch*r, C], rois [batch*r, 5], num_rois int32 [batch], im_meta
    [batch, 3], fc7 [batch*r, F]; workspace of detect_regions_workspace(r, C, batch) bytes or more; keep / keep_cnt / keep_score
    as for detect_post up to REGIONS_CLASS_NMS_MAX classes (unused, may be None, above); roi_box regions_box_shape(batch*r, C) fp32
    and key int64 [batch*r] scratch.  out: dict of boxes [batch, M, 4], conf [batch, M], classes int32 [batch, M], roi_index int32
    [batch, M], features [batch, M, F], count int32 [batch] with M = min(max_boxes, r).  conf_thresh is the fp32 threshold."""
    r = cls_prob.shape[0] // batch
    fdim = fc7.shape[1]
    N.check(N.lib().frcnn_detect_regions(_p(_f32(cls_prob)), _p(_f32(rois)), _p(num_rois), _p(_f32(im_meta)), _p(_f32(fc7)), r, batch,
                                         num_classes, fdim, float(nms_thresh), flags, float(conf_thresh), int(min_boxes), int(max_boxes),
                                         _p(keep), _p(keep_cnt), _p(keep_score), _p(workspace), 0 if workspace is None else workspace.numel(),
                                         _p(_f32(roi_box)), _p(key), _p(_f32(out["boxes"])), _p(_f32(out["conf"])), _p(out["classes"]),
                                         _p(out["roi_index"]), _p(_f32(out["features"])), _p(out["count"]), _stream()), "detect_regions")


def regions_attr_embed(cls_score, num_classes, index, count, embedding, emb_out):
    """Attribute head steps 1-2 (frcnn_regions_attr_embed): cls_score [batch*r, C] logits, index / count int32 [batch, M] / [batch]
    of detect_regions, embedding [C, E] -> emb_out [batch*M, E] = the embedding row of each region's argmax class (zeros past the
    count)."""
    batch, M = index.shape
    r = cls_score.shape[0] // batch
    N.check(N.lib().frcnn_regions_attr_embed(_p(_f32(cls_score)), r, batch, num_classes, _p(index), _p(count), M, _p(_f32(embedding)),
                                             embedding.shape[1], _p(_f32(emb_out)), _stream()), "regions_attr_embed")


def attr_finish(score, num_attributes, count, attr_prob, attributes, attr_conf):
    """Attribute head softmax and step 5 (frcnn_attr_finish): score [batch*M, ld] logits, count int32 [batch] -> attr_prob
    [batch, M, A], attributes int32 [batch, M] (-1 past the count), attr_conf [batch, M]."""
    batch, M, _ = attr_prob.shape
    N.check(N.lib().frcnn_attr_finish(_p(_f32(score)), score.shape[1], batch, M, num_attributes, _p(count), _p(_f32(attr_prob)),
                                      _p(attributes), _p(_f32(attr_conf)), _stream()), "attr_finish")


def boxes_to_rois(boxes, counts, im_meta, rois, num_rois):
    """boxes [batch, cap, 4] original-image pixels, counts int32 [batch], im_meta [batch, 3] -> rois [batch*cap, 5], num_rois."""
    batch, cap, _ = boxes.shape
    N.check(N.lib().frcnn_boxes_to_rois(_p(_f32(boxes)), _p(counts), _p(_f32(im_meta)), batch, cap, _p(_f32(rois)), _p(num_rois),
                                        _stream()), "boxes_to_rois")


def aug_union(views, num_classes, im_meta, cls_prob, pred_boxes, num_rois):
    """Test-time augmentation union.  views: per view (cls_prob, pred_boxes, num_rois, rows, flip) with the three as device
    addresses (ints) of the view's [batch, rows, C] / [batch, rows, 4C] / int32 [batch]; im_meta: device address of [batch, 3]
    (orig_w in column 2).  cls_prob [batch, R_union, C], pred_boxes [batch, R_union, 4C], num_rois int32 [batch] (tensors)."""
    nv = len(views)
    ptrs = [(C.c_void_p * nv)(*[v[k] for v in views]) for k in range(3)]
    rows = (C.c_int * nv)(*[int(v[3]) for v in views])
    flips = (C.c_int * nv)(*[int(bool(v[4])) for v in views])
    batch = num_rois.shape[0]
    N.check(N.lib().frcnn_aug_union(ptrs[0], ptrs[1], ptrs[2], rows, flips, nv, batch, num_classes, C.c_void_p(im_meta), _p(_f32(cls_prob)),
                                    _p(_f32(pred_boxes)), _p(num_rois), _stream()), "aug_union")


def nms_sorted_dev(boxes, thresh, flags, max_out, keep, num):
    N.check(N.lib().frcnn_nms_sorted_dev(_p(_f32(boxes)), boxes.shape[0], float(thresh), flags, max_out, _p(keep), _p(num),
                                         _stream()), "nms_sorted_dev")


def nms_host(sorted_dets, thresh, flags, device_id=-1):
    """`_nms`-compatible call on HOST arrays (already sorted by descending score).  device_id < 0: the current device."""
    d = np.ascontiguousarray(sorted_dets, dtype=np.float32)
    n = d.shape[0]
    keep = np.empty(max(n, 1), dtype=np.int32)
    num = C.c_int(0)
    N.check(N.lib().frcnn_nms_host(keep.ctypes.data_as(N.ip), C.byref(num), d.ctypes.data_as(N.fp), n, d.shape[1] if n else 5,
                                   float(thresh), device_id, flags), "nms_host")
    return keep[:num.value].copy()


def soft_nms_host(dets, method, sigma, nt, score_thresh, device_id=-1):
    """Soft-NMS of one set of HOST rows [n, >=5] (x1, y1, x2, y2, score, ...), candidates in row order; method is an
    FRCNN_SOFT_NMS_* code.  -> (rows [k,5] fp32 in selection order with decayed scores, keep [k] int32 rows of dets)."""
    d = np.ascontiguousarray(dets, dtype=np.float32)
    n = d.shape[0]
    out = np.empty((max(n, 1), 5), dtype=np.float32)
    keep = np.empty(max(n, 1), dtype=np.int32)
    num = C.c_int(0)
    N.check(N.lib().frcnn_soft_nms_host(out.ctypes.data_as(N.fp), keep.ctypes.data_as(N.ip), C.byref(num), d.ctypes.data_as(N.fp), n,
                                        d.shape[1] if n else 5, int(method), float(sigma), float(nt), float(score_thresh), device_id),
            "soft_nms_host")
    return out[:num.value].copy(), keep[:num.value].copy()


def box_vote_host(top_dets, all_dets, thresh, method, beta, device_id=-1):
    """Box voting of one set of HOST rows (x1, y1, x2, y2, score, ...): top_dets [n, >=5] voted against the candidates all_dets
    [m, >=5]; method is an FRCNN_BOX_VOTE_* code.  -> fp32 [n, 5], the voted rows in top_dets' row order."""
    t = np.ascontiguousarray(top_dets, dtype=np.float32)
    a = np.ascontiguousarray(all_dets, dtype=np.float32)
    n, m = t.shape[0], a.shape[0]
    out = np.empty((max(n, 1), 5), dtype=np.float32)
    N.check(N.lib().frcnn_box_vote_host(out.ctypes.data_as(N.fp), t.ctypes.data_as(N.fp), n, t.shape[1] if n else 5, a.ctypes.data_as(N.fp),
                                        m, a.shape[1] if m else 5, float(thresh), int(method), float(beta), device_id), "box_vote_host")
    return out[:n].copy()
