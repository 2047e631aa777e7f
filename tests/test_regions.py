"""Bottom-up regions without a GPU: the oracle (tests/regions_oracle.py) against an independent restatement, the comparator
against plausible mistakes, the argument refusals and the TSV writer of tools/extract_features.py."""
import base64
import csv
import ctypes
import io
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
import regions_oracle as RO  # noqa: E402
from tf_faster_rcnn_b200 import engine  # noqa: E402

F = np.float32


def random_case(rng, r, C, nr, spread=600.0, size=(20, 200)):
    """cls_prob [r, C] (softmax rows, every row filled, also past nr), rois [r, 5] (padding rows past nr are zero)."""
    logits = rng.normal(0, 2, (r, C))
    p = np.exp(logits - logits.max(1, keepdims=True))
    probs = (p / p.sum(1, keepdims=True)).astype(F)
    xy = rng.uniform(0, spread, (r, 2))
    wh = rng.uniform(size[0], size[1], (r, 2))
    rois = np.hstack([np.zeros((r, 1)), xy, xy + wh]).astype(F)
    rois[nr:] = 0
    return probs, rois


# ---- an independent restatement: py_cpu_nms-style loop, then plain loops over rows and classes ---------------------------------
def loop_nms(dets, thresh, inclusive):
    x1, y1, x2, y2, s = (dets[:, k] for k in range(5))
    areas = (x2 - x1 + F(1)) * (y2 - y1 + F(1))
    order = list(s.argsort()[::-1])                     # tie-free inputs: the protocol's order
    t = F(thresh)
    if inclusive and float(t) < thresh:
        t = np.nextafter(t, F(np.inf))
    keep = []
    while order:
        i = order.pop(0)
        keep.append(i)
        rest = []
        for j in order:
            w = max(F(0), min(x2[i], x2[j]) - max(x1[i], x1[j]) + F(1))
            h = max(F(0), min(y2[i], y2[j]) - max(y1[i], y1[j]) + F(1))
            inter = F(w * h)
            ovr = F(inter / F(F(areas[i] + areas[j]) - inter))
            if not ((ovr >= t) if inclusive else (ovr > t)):
                rest.append(j)
        order = rest
    return keep


def loop_regions(probs, rois, nr, scale, nms_thresh, use_gpu_nms, conf_thresh, min_boxes, max_boxes):
    boxes = np.array([[F(rois[i, k]) / F(scale) for k in range(1, 5)] for i in range(nr)], F).reshape(nr, 4)
    C = probs.shape[1]
    conf, cls = [0.0] * nr, [0] * nr
    for c in range(1, C):
        kept = set(loop_nms(np.hstack([boxes, probs[:nr, c:c + 1]]).astype(F), nms_thresh, not use_gpu_nms))
        for i in range(nr):
            if i in kept and float(probs[i, c]) > conf[i]:
                conf[i], cls[i] = float(probs[i, c]), c
    sel = [i for i in range(nr) if conf[i] >= conf_thresh]
    if not min_boxes <= len(sel) <= max_boxes:
        sel = sorted(range(nr), key=lambda i: -conf[i])[:min(max(len(sel), min_boxes), max_boxes)]
    idx = np.array(sel, np.int64)
    return dict(boxes=boxes[idx], conf=np.array(conf, F)[idx], classes=np.array(cls, np.int32)[idx], roi_index=idx.astype(np.int32))


@pytest.mark.parametrize("C,r,nr,thr,mn,mx,gpu_pred", [
    (2, 60, 60, 0.2, 10, 100, False), (7, 80, 57, 0.2, 10, 100, True), (5, 70, 70, 0.5, 3, 8, False),
    (4, 40, 31, 0.9, 10, 20, True), (6, 50, 50, 0.0, 5, 12, False)])
def test_oracle_matches_independent_restatement(C, r, nr, thr, mn, mx, gpu_pred):
    rng = np.random.default_rng(C * 100 + r)
    probs, rois = random_case(rng, r, C, nr, spread=200.0, size=(20, 120))
    scale = 1.6
    want = loop_regions(probs, rois, nr, scale, 0.3, gpu_pred, thr, mn, mx)
    got = RO.image_regions(probs, rois, nr, scale, 0.3, gpu_pred, thr, mn, mx)
    RO.compare(got, want)
    assert got["boxes"].shape[0] > 0


# ---- the comparator rejects each plausible mistake ---------------------------------------------------------------------------
def pieces(probs, rois, nr, scale=1.25):
    boxes = RO.roi_boxes(rois[:nr], scale)
    return boxes, probs[:nr]


def test_mistake_regressed_boxes():
    rng = np.random.default_rng(1)
    probs, rois = random_case(rng, 100, 5, 100)
    want = RO.image_regions(probs, rois, 100, 1.25, 0.3, False, 0.2, 10, 100)
    boxes, p = pieces(probs, rois, 100)
    deltas = rng.uniform(-6, 6, (probs.shape[1], 4)).astype(F)      # each class's box regressed by its own offset
    conf, cls = np.zeros(100, F), np.zeros(100, np.int32)
    for c in range(1, probs.shape[1]):
        kb = (boxes + deltas[c]).astype(F)
        keep = RO.NMS.nms_plus1_c(np.hstack([kb, p[:, c:c + 1]]), 0.3, True)
        better = p[keep, c] > conf[keep]
        conf[keep[better]], cls[keep[better]] = p[keep[better], c], c
    idx = RO.select(conf, 0.2, 10, 100)
    reg = (boxes + deltas[cls]).astype(F)
    with pytest.raises(AssertionError):
        RO.compare(RO.pack(reg, conf, cls, idx), want)


def test_mistake_conf_sorted_within_range():
    rng = np.random.default_rng(2)
    probs, rois = random_case(rng, 100, 5, 100)
    boxes, p = pieces(probs, rois, 100)
    conf, cls = RO.best_kept_class(boxes, p, 0.3, False)
    idx = RO.select(conf, 0.2, 1, 100)
    assert 1 <= idx.shape[0] <= 100 and np.array_equal(idx, np.sort(idx))
    wrong = idx[np.argsort(-conf[idx], kind="stable")]
    with pytest.raises(AssertionError):
        RO.compare(RO.pack(boxes, conf, cls, wrong), RO.pack(boxes, conf, cls, idx))


def test_mistake_padded_rows_counted():
    rng = np.random.default_rng(3)
    probs, rois = random_case(rng, 120, 5, 60)
    want = RO.image_regions(probs, rois, 60, 1.25, 0.3, False, 0.2, 10, 100)
    with pytest.raises(AssertionError):
        RO.compare(RO.image_regions(probs, rois, 120, 1.25, 0.3, False, 0.2, 10, 100), want)


def test_mistake_strict_threshold():
    rng = np.random.default_rng(4)
    probs, rois = random_case(rng, 80, 5, 80)
    boxes, p = pieces(probs, rois, 80)
    conf, cls = RO.best_kept_class(boxes, p, 0.3, False)
    t = float(np.sort(conf)[-5])                         # exactly one region's confidence
    want = RO.pack(boxes, conf, cls, RO.select(conf, t, 1, 100))
    wrong = np.where(conf.astype(np.float64) > t)[0]
    with pytest.raises(AssertionError):
        RO.compare(RO.pack(boxes, conf, cls, wrong), want)


def test_mistake_max_without_nms():
    rng = np.random.default_rng(5)
    probs, rois = random_case(rng, 100, 5, 100, spread=150.0)
    boxes, p = pieces(probs, rois, 100)
    want = RO.image_regions(probs, rois, 100, 1.25, 0.3, False, 0.2, 10, 100)
    conf = p[:, 1:].max(1).astype(F)
    cls = (p[:, 1:].argmax(1) + 1).astype(np.int32)
    with pytest.raises(AssertionError):
        RO.compare(RO.pack(boxes, conf, cls, RO.select(conf, 0.2, 10, 100)), want)


def test_mistake_ties_to_higher_index():
    rng = np.random.default_rng(6)
    probs, rois = random_case(rng, 40, 4, 40, spread=2000.0, size=(10, 20))   # isolated boxes: every class keeps every row
    probs[7], probs[23] = probs[31], probs[31]                                 # three rows with the same confidence
    boxes, p = pieces(probs, rois, 40)
    conf, cls = RO.best_kept_class(boxes, p, 0.3, False)
    want = RO.pack(boxes, conf, cls, RO.select(conf, 0.2, 40, 40))
    order = np.lexsort((-np.arange(40), -conf.astype(np.float64)))
    with pytest.raises(AssertionError):
        RO.compare(RO.pack(boxes, conf, cls, order), want)


def test_mistake_threshold_rounded_to_nearest():
    t = 0.7                                              # fp32(0.7) = 0.699999988 < 0.7
    assert float(F(t)) < t and engine.region_args(t, 0, 100)[0] > t
    rng = np.random.default_rng(7)
    probs, rois = random_case(rng, 40, 3, 40, spread=2000.0, size=(10, 20))
    probs[:, 1:] = np.minimum(probs[:, 1:], F(0.5))
    probs[9, 2] = F(t)
    boxes, p = pieces(probs, rois, 40)
    conf, cls = RO.best_kept_class(boxes, p, 0.3, False)
    want = RO.pack(boxes, conf, cls, RO.select(conf, t, 0, 100))
    assert want["roi_index"].shape[0] == 0
    wrong = np.where(conf >= F(t))[0]
    with pytest.raises(AssertionError):
        RO.compare(RO.pack(boxes, conf, cls, wrong), want)
    # the device threshold (smallest fp32 not below t) gives the float64 comparison's selection
    assert np.array_equal(np.where(conf >= F(engine.region_args(t, 0, 100)[0]))[0], want["roi_index"])


# ---- argument refusals --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("args", [(float("nan"), 10, 100), (float("inf"), 10, 100), (-0.01, 10, 100), (1.5, 10, 100), ("x", 10, 100),
                                  (0.2, 10.0, 100), (0.2, 10, "100"), (0.2, True, 100), (0.2, -1, 100), (0.2, 0, 0),
                                  (0.2, 50, 40)])
def test_region_args_refused(args):
    with pytest.raises(ValueError):
        engine.region_args(*args)


def test_region_args_accepted():
    assert engine.region_args(0.2, 10, 100) == (float(F(0.2)), 10, 100)
    assert engine.region_args(0, 0, 1) == (0.0, 0, 1)
    assert engine.region_args(1, np.int64(36), 36) == (1.0, 36, 36)
    t = engine.region_args(0.7, 10, 100)[0]
    assert t >= 0.7 and float(np.nextafter(F(t), F(0))) < 0.7


def test_detect_regions_refuses_before_device_work():
    from model.config import cfg
    from nets.resnet_v1 import resnetv1
    net = resnetv1(num_layers=50)
    net.create_architecture("TEST", 21, tag="default", anchor_scales=(8, 16, 32), anchor_ratios=(0.5, 1, 2))
    blob = np.zeros((1, 64, 64, 3), F)
    for bad in (dict(conf_thresh=-1.0), dict(min_boxes=20, max_boxes=10), dict(max_boxes=0), dict(min_boxes=2.5)):
        with pytest.raises(ValueError):
            net.detect_regions(blob, [1.0], [(64, 64)], **bad)
    old = cfg.TEST.BBOX_AUG.ENABLED
    cfg.TEST.BBOX_AUG.ENABLED = True
    try:
        with pytest.raises(ValueError, match="BBOX_AUG"):
            net.detect_regions(blob, [1.0], [(64, 64)])
    finally:
        cfg.TEST.BBOX_AUG.ENABLED = old


def test_c_entry_validates_before_any_cuda_call():
    """Non-null (never dereferenced) pointers with one bad parameter each: FRCNN_ERR_ARG with a message, no device needed."""
    from tf_faster_rcnn_b200 import _native as N
    fn = N.lib().frcnn_detect_regions
    p = ctypes.c_void_p(4096)
    good = dict(r=300, batch=1, C=21, fdim=64, nms=0.3, conf=0.2, mn=10, mx=100)

    def call(**kw):
        a = dict(good, **kw)
        return fn(p, p, p, p, p, a["r"], a["batch"], a["C"], a["fdim"], a["nms"], 1, a["conf"], a["mn"], a["mx"], p, p, p, None, 0,
                  p, p, p, p, p, p, p, p, None)
    for bad in (dict(conf=1.5), dict(conf=-0.5), dict(conf=float("nan")), dict(mn=-1), dict(mx=0), dict(mn=11, mx=10), dict(fdim=6),
                dict(C=1), dict(r=0), dict(r=2000)):
        assert call(**bad) == -2, bad
        assert N.last_error()
    assert call(r=9000) == -5


# ---- the TSV writer -----------------------------------------------------------------------------------------------------------
def test_tsv_round_trip():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import extract_features as EF
    rng = np.random.default_rng(8)
    rows = [("img_a", 375, 500, rng.normal(0, 100, (12, 4)).astype(F), rng.normal(0, 1, (12, 2048)).astype(F)),
            ("7", 480, 640, np.zeros((0, 4), F), np.zeros((0, 2048), F))]
    buf = io.StringIO()
    w = EF.tsv_writer(buf)
    for r in rows:
        w.writerow(EF.tsv_row(*r))
    buf.seek(0)
    back = list(csv.DictReader(buf, delimiter="\t", fieldnames=EF.TSV_FIELDS))
    assert EF.TSV_FIELDS == ["image_id", "image_w", "image_h", "num_boxes", "boxes", "features"]
    assert len(back) == 2
    for (iid, h, w_, boxes, feats), d in zip(rows, back):
        n = int(d["num_boxes"])
        assert d["image_id"] == iid and int(d["image_h"]) == h and int(d["image_w"]) == w_ and n == boxes.shape[0]
        b = np.frombuffer(base64.b64decode(d["boxes"]), dtype=F).reshape(n, 4)
        f = np.frombuffer(base64.b64decode(d["features"]), dtype=F).reshape(n, 2048)
        assert np.array_equal(b, boxes) and f.shape == feats.shape and np.array_equal(f, feats)
