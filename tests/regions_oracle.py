"""Oracle of the bottom-up regions (test infrastructure): a numpy transcription of the definition in include/frcnn_b200.h
(frcnn_detect_regions), built on oracle.nms.nms_plus1_c and the oracle's fp32 RoI division rois / F(scale).

The steps are separate functions so that tests can recombine them (tests/test_regions.py builds plausible mistakes from them)."""
import numpy as np

from oracle import nms as NMS

F = np.float32


def valid_rows(num_rois, r):
    return max(0, min(int(num_rois), int(r)))


def roi_boxes(rois, scale):
    """rois [n, 5] (image, x1, y1, x2, y2 in blob pixels) -> fp32 [n, 4] = rois[:, 1:5] / F(scale), one fp32 division each."""
    return (np.asarray(rois, F)[:, 1:5] / F(scale)).astype(F)


def best_kept_class(boxes, probs, nms_thresh, use_gpu_nms):
    """Per-class greedy NMS over every row (no score threshold), then per row the largest score over the classes whose NMS kept
    it (0 if none) and the lowest class reaching it (0 when the score is 0): the protocol's ascending class loop with '>'."""
    n, C = probs.shape
    conf, cls = np.zeros(n, F), np.zeros(n, np.int32)
    for c in range(1, C):
        dets = np.hstack([boxes, probs[:, c:c + 1]]).astype(F)
        keep = NMS.nms_plus1_c(dets, nms_thresh, inclusive=not use_gpu_nms)
        s = probs[keep, c]
        better = s > conf[keep]
        conf[keep[better]] = s[better]
        cls[keep[better]] = c
    return conf, cls


def select(conf, conf_thresh, min_boxes, max_boxes):
    """Row indices of the regions: np.where(conf >= conf_thresh) (compared in float64) when min_boxes <= count <= max_boxes, else
    the first min(max(count, min_boxes), max_boxes) rows in descending conf, ties to the lower row."""
    sel = np.where(conf.astype(np.float64) >= float(conf_thresh))[0]
    if min_boxes <= sel.shape[0] <= max_boxes:
        return sel
    order = np.lexsort((np.arange(conf.shape[0]), -conf.astype(np.float64)))
    return order[:min(max(sel.shape[0], min_boxes), max_boxes)]


def pack(boxes, conf, cls, idx, fc7=None):
    out = dict(boxes=boxes[idx], conf=conf[idx], classes=cls[idx].astype(np.int32), roi_index=idx.astype(np.int32))
    if fc7 is not None:
        out["features"] = fc7[idx]
    return out


def image_regions(cls_prob, rois, num_rois, scale, nms_thresh, use_gpu_nms, conf_thresh, min_boxes, max_boxes, fc7=None):
    """One image: cls_prob [r, C], rois [r, 5], num_rois, the fp32 scale, TEST.NMS / USE_GPU_NMS and the float64 conf_thresh
    -> dict(boxes [n,4], conf [n], classes [n] int32, roi_index [n] int32 (, features [n,F] when fc7 [r,F] is given))."""
    nr = valid_rows(num_rois, cls_prob.shape[0])
    boxes = roi_boxes(rois[:nr], scale)
    conf, cls = best_kept_class(boxes, np.asarray(cls_prob[:nr], F), nms_thresh, use_gpu_nms)
    idx = select(conf, conf_thresh, min_boxes, max_boxes)
    return pack(boxes, conf, cls, idx, None if fc7 is None else fc7[:nr])


def compare(got, want):
    """Exact equality of every field of one image's regions (AssertionError naming the first field that differs)."""
    for k in want:
        assert k in got, k
        a, b = np.asarray(got[k]), np.asarray(want[k])
        assert a.shape == b.shape, (k, a.shape, b.shape)
        assert a.dtype == b.dtype, (k, a.dtype, b.dtype)
        assert a.tobytes() == b.tobytes(), (k, a, b)
