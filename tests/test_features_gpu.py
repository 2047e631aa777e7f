"""Region features on the GPU: Network.detect_features (the head feature and RoI index of every detection, gathered in the
detect graph), Network.score_boxes / im_detect(boxes=...) (caller boxes as the RoIs: the Fast R-CNN mode) and
tools/extract_features.py.

Bit-exactness claims are made where both sides read the same device buffers: the gathered feature of detection k IS the fc7
row of its RoI, its box / score ARE that RoI's pred_boxes / cls_prob entries, and a batch through the two new kernels equals
the images one at a time.  Across different batch sizes the network itself is equal only up to summation order (the dense
kernel's split-K choice depends on the batch), so whole-network batch-vs-single comparisons use the 1e-4 bounds."""
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import pipeline as P

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import region_oracle as RO  # noqa: E402
from tf_faster_rcnn_b200 import engine, ops, synth

pytestmark = pytest.mark.gpu
F = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build(net_name, num_classes, scales):
    from model.config import cfg
    from nets.vgg16 import vgg16
    from nets.resnet_v1 import resnetv1
    from nets.mobilenet_v1 import mobilenetv1
    cfg.TEST.HAS_RPN = True
    net = vgg16() if net_name == "vgg16" else mobilenetv1() if net_name == "mobile" else resnetv1(num_layers=int(net_name[3:]))
    net.create_architecture("TEST", num_classes, tag="default", anchor_scales=scales, anchor_ratios=(0.5, 1, 2))
    w = synth.make(net_name, num_classes, 3 * len(scales))
    net.load_weights(w)
    return net, w


def fc7_err(a, b, ref):
    return float(np.abs(a - b).max() / np.abs(ref).max()) if a.size else 0.0


def check_gather(net, plan, res):
    """Every detection's feature / box / score is, bit for bit, the fc7 / pred_boxes / cls_prob entry of its RoI; slots past
    the count are -1 / zero."""
    R, C = plan.R, net.num_classes
    fc7, prob = plan.fc7.cpu().numpy(), plan.cls_prob.cpu().numpy()
    pred = plan.pred_boxes.cpu().numpy().reshape(-1, C, 4)
    nroi = plan.num_rois.cpu().numpy()
    feat_out, roi_out = plan.feat_out.cpu().numpy(), plan.roi_out.cpu().numpy()
    for b, (det, feats, roi) in enumerate(res):
        n = det.shape[0]
        assert n > 0 and feats.shape == (n, fc7.shape[1]) and feats.dtype == F and roi.dtype == np.int32
        assert roi.min() >= 0 and roi.max() < nroi[b]
        rows, cls = b * R + roi, det[:, 5].astype(np.int64)
        assert np.array_equal(feats, fc7[rows])
        assert np.array_equal(det[:, :4], pred[rows, cls]) and np.array_equal(det[:, 4], prob[rows, cls])
        assert (roi_out[b, n:] == -1).all() and not feat_out[b, n:].any()


@pytest.mark.parametrize("net_name", ["res50", "vgg16"])
def test_feature_gather_is_exact(cuda, net_name):
    net, w = build(net_name, 21, (8, 16, 32))
    hw = (224, 304)
    blobs = np.concatenate([synth.synthetic_blob(hw[0], hw[1], seed) for seed in (1, 2, 3)], axis=0)
    scales, orig = [1.0, 1.25, 0.8], [(224, 304), (179, 243), (280, 380)]
    res3, plan3 = net.detect_features(blobs, scales, orig)
    check_gather(net, plan3, res3)
    for (det, _, _), want in zip(res3, net.detect_batch(blobs, scales, orig)[0]):
        assert det.shape == want.shape and det.tobytes() == want.tobytes()
    # the gather kernel over the batch == the same kernel over each image's keep lists and fc7 rows alone
    R, C, md, fd = plan3.R, 21, plan3.max_det, plan3.feat_out.shape[2]
    for b in range(3):
        fo, ro = ops.zeros((1, md, fd)), ops.zeros((1, md), dtype=torch.int32)
        ops.detect_features(plan3.keep[b:b + 1].contiguous(), plan3.keep_cnt[b:b + 1].contiguous(), plan3.fc7[b * R:(b + 1) * R], C, fo, ro)
        assert torch.equal(fo[0], plan3.feat_out[b]) and torch.equal(ro[0], plan3.roi_out[b])
    # batch 1
    for b in range(3):
        res1, plan1 = net.detect_features(blobs[b:b + 1], scales[b:b + 1], orig[b:b + 1])
        check_gather(net, plan1, res1)
        det1, feats1, roi1 = res1[0]
        assert det1.tobytes() == net.detect_batch(blobs[b:b + 1], scales[b:b + 1], orig[b:b + 1])[0][0].tobytes()
        det3, feats3, roi3 = res3[b]
        same = det1.tobytes() == det3.tobytes()
        if same:
            assert np.array_equal(roi1, roi3)
        common, i1, i3 = np.intersect1d(roi1.astype(np.int64) * 32 + det1[:, 5].astype(np.int64),
                                        roi3.astype(np.int64) * 32 + det3[:, 5].astype(np.int64), return_indices=True)
        err = fc7_err(feats1[i1], feats3[i3], feats3)
        print("\n[%s image %d] batch-1 vs batch-3: records identical=%s, common (roi, class) %d/%d, feature rel err %.2e"
              % (net_name, b, same, len(common), det3.shape[0], err))
        assert len(common) >= 0.95 * det3.shape[0] and err < 1e-4
        if same:
            assert err == 0.0


def match_with_oracle(det, want, widx, tol):
    """(gpu row, oracle class, oracle row) of detections matched as in test_e2e_gpu.compare_detections."""
    pairs = []
    cls = det[:, 5].astype(np.int64)
    for j, wj in enumerate(want):
        g = np.where(cls == j)[0]
        if not g.size or not wj.shape[0]:
            continue
        d = np.abs(det[g, None, :4] - wj[None, :, :4]).max(axis=2)
        used = set()
        for a, i in enumerate(g):
            k = int(np.argmin(d[a]))
            if d[a, k] <= tol and k not in used:
                used.add(k)
                pairs.append((i, j, k))
    return pairs


@pytest.mark.parametrize("net_name,hw,tol", [("res101", (600, 800), 5e-3), ("mobile", (600, 800), 4e-3)])
def test_detection_features_match_oracle(cuda, net_name, hw, tol):
    net, w = build(net_name, 81, (4, 8, 16, 32))
    blob = synth.synthetic_blob(*hw)
    o = P.opts(anchor_scales=(4, 8, 16, 32))
    st = P.test_image(net_name, w, blob, np.array([hw[0], hw[1], 1.0], F), 81, o)
    (det, feats, roi), = net.detect_features(blob, [1.0], [hw])[0]
    scores, boxes = P.im_detect_post(st["rois"], st["cls_prob"], st["bbox_pred"], 1.0, hw[0], hw[1])
    want, widx = RO.test_net_post_indexed(scores, boxes, o)
    pairs = match_with_oracle(det, want, widx, tol)
    n_want = sum(x.shape[0] for x in want)
    got = np.stack([feats[i] for i, _, _ in pairs])
    ref = np.stack([st["fc7"][widx[j][k]] for _, j, k in pairs])
    err = fc7_err(got, ref, st["fc7"])
    print("\n[%s %dx%d] detections gpu %d oracle %d matched %d | feature of matched detections: max abs err / max|fc7| = %.2e"
          % (net_name, hw[0], hw[1], det.shape[0], n_want, len(pairs), err))
    assert len(pairs) >= 0.95 * n_want
    assert err < 1e-4


def test_score_boxes_own_rois_at_scale_1(cuda):
    net, w = build("res101", 81, (4, 8, 16, 32))
    hw = (320, 480)
    blob = synth.synthetic_blob(*hw)
    o = P.opts(anchor_scales=(4, 8, 16, 32))
    st = P.test_image("res101", w, blob, np.array([hw[0], hw[1], 1.0], F), 81, o)
    boxes = np.ascontiguousarray(st["rois"][:, 1:5])
    (scores, pred_boxes, feats), = net.score_boxes(blob, [1.0], [hw], [boxes])[0]
    plan = net.plan_for(hw[0], hw[1], 1, cap=engine.box_capacity(boxes.shape[0]))
    n = boxes.shape[0]
    rois, bbox_pred = plan.rois[:n].cpu().numpy(), plan.bbox_pred[:n].cpu().numpy()
    assert scores.shape == (n, 81) and pred_boxes.shape == (n, 324) and feats.shape == st["fc7"].shape
    assert np.array_equal(rois, st["rois"]) and int(plan.num_rois[0]) == n
    e_prob, e_bbox = float(np.abs(scores - st["cls_prob"]).max()), float(np.abs(bbox_pred - st["bbox_pred"]).max())
    e_fc7 = fc7_err(feats, st["fc7"], st["fc7"])
    _, want_pred = P.im_detect_post(rois, scores, bbox_pred, 1.0, hw[0], hw[1])
    print("\n[res101 %dx%d, %d oracle RoIs as boxes] cls_prob abs %.2e bbox_pred abs %.2e fc7 rel %.2e" % (hw[0], hw[1], n, e_prob, e_bbox, e_fc7))
    assert e_prob < 1e-4 and e_bbox < 1e-4 and e_fc7 < 1e-4
    assert np.abs(pred_boxes - want_pred).max() < 1e-4


def random_boxes(rng, n, h, w):
    xy = rng.uniform(0, [w * 0.8, h * 0.8], (n, 2))
    wh = rng.uniform(8, [w * 0.5, h * 0.5], (n, 2))
    return np.hstack([xy, xy + wh]).astype(F)


def test_score_boxes_scaled_matches_oracle(cuda):
    net, w = build("res50", 21, (8, 16, 32))
    hw, scale = (224, 304), 1.25
    orig = (179, 243)
    blob = synth.synthetic_blob(*hw)
    boxes = random_boxes(np.random.default_rng(11), 150, *orig)
    (scores, pred_boxes, feats), = net.score_boxes(blob, [scale], [orig], [boxes])[0]
    sb = RO.score_boxes("res50", w, blob, boxes, scale, orig, P.opts())
    plan = net.plan_for(hw[0], hw[1], 1, cap=engine.box_capacity(boxes.shape[0]))
    rois, bbox_pred = plan.rois[:150].cpu().numpy(), plan.bbox_pred[:150].cpu().numpy()
    assert np.array_equal(rois, sb["rois"])
    e_prob, e_bbox = float(np.abs(scores - sb["cls_prob"]).max()), float(np.abs(bbox_pred - sb["bbox_pred"]).max())
    e_fc7 = fc7_err(feats, sb["fc7"], sb["fc7"])
    print("\n[res50 scale %.2f, 150 boxes] cls_prob abs %.2e bbox_pred abs %.2e fc7 rel %.2e" % (scale, e_prob, e_bbox, e_fc7))
    assert e_prob < 1e-4 and e_bbox < 1e-4 and e_fc7 < 1e-4
    _, want_pred = P.im_detect_post(rois, scores, bbox_pred, scale, orig[0], orig[1])
    assert np.abs(pred_boxes - want_pred).max() < 1e-4


def test_score_boxes_counts_and_batch(cuda):
    """Counts 0, 1 and cap in one batch of 3: exactly n_i rows back per image, zero RoI rows past each count, each image
    equal to its single-image run (bit for bit through boxes_to_rois, to 1e-4 through the whole network)."""
    net, w = build("res50", 21, (8, 16, 32))
    hw = (224, 304)
    rng = np.random.default_rng(5)
    blobs = np.concatenate([synth.synthetic_blob(hw[0], hw[1], s) for s in (1, 2, 3)], axis=0)
    scales, orig = [1.0, 1.25, 0.8], [(224, 304), (179, 243), (280, 380)]
    for counts in ((0, 1, 64), (64, 0, 17)):
        boxes = [random_boxes(rng, n, *orig[b]) for b, n in enumerate(counts)]
        res, plan = net.score_boxes(blobs, scales, orig, boxes)
        assert plan.R == 64 and plan.num_rois.cpu().tolist() == list(counts)
        rois = plan.rois.cpu().numpy().reshape(3, 64, 5)
        for b, n in enumerate(counts):
            assert res[b][0].shape == (n, 21) and res[b][1].shape == (n, 84) and res[b][2].shape[0] == n
            assert not rois[b, n:].any() and (rois[b, :n, 0] == b).all()
            # boxes_to_rois on this image alone gives the same rows
            r1, n1 = ops.zeros((64, 5)), ops.zeros(1, dtype=torch.int32)
            ops.boxes_to_rois(plan.boxes[b:b + 1].contiguous(), plan.box_counts[b:b + 1].contiguous(),
                              plan.im_meta[b:b + 1].contiguous(), r1, n1)
            r1 = r1.cpu().numpy()
            r1[:n, 0] = b
            assert np.array_equal(r1, rois[b]) and int(n1[0]) == n
            single, _ = net.score_boxes(blobs[b:b + 1], scales[b:b + 1], orig[b:b + 1], [boxes[b]])
            for got, want in zip(res[b], single[0]):
                assert got.shape == want.shape
                if n:
                    assert np.abs(got - want).max() <= 1e-4 * max(np.abs(want).max(), 1.0)


def test_im_detect_with_boxes(cuda):
    import cv2
    import model.test as MT
    net, w = build("res50", 21, (8, 16, 32))
    im = cv2.blur(np.random.default_rng(9).integers(0, 256, (240, 320, 3), dtype=np.uint8), (5, 5))
    boxes = random_boxes(np.random.default_rng(3), 40, 240, 320).astype(np.float64)    # im_detect takes any real dtype
    s0, b0 = MT.im_detect(None, net, im, boxes=boxes)
    blobs, im_scales = MT._get_blobs(im)
    (scores, pred_boxes, _), = net.score_boxes(blobs["data"], [im_scales[0]], [im.shape[:2]], [boxes.astype(F)])[0]
    assert s0.shape == (40, 21) and np.array_equal(s0, scores) and np.array_equal(b0, pred_boxes)
    MT.DEVICE_PREPROCESS = True
    try:
        s1, b1 = MT.im_detect(None, net, im, boxes=boxes)
    finally:
        MT.DEVICE_PREPROCESS = False
    H, W, f = MT.blob_geometry(im.shape)
    dev_blob = net.plan_for(H, W, 1, cap=64).image.cpu().numpy()
    (scores, pred_boxes, _), = net.score_boxes(dev_blob, [f], [im.shape[:2]], [boxes.astype(F)])[0]
    assert np.array_equal(s1, scores) and np.array_equal(b1, pred_boxes)
    assert np.abs(s0 - s1).max() < 1e-3 and np.abs(b0 - b1).max() < 0.5


def test_extract_features_tool_matches_api(cuda, tmp_path):
    import cv2
    from datasets.factory import get_imdb
    from model.test import _get_blobs
    imdb = get_imdb("synthetic_4_21")
    rng = np.random.default_rng(2)
    given = {i: random_boxes(rng, 10 + 7 * i, 375, 500) for i in range(4)}
    with open(tmp_path / "boxes.pkl", "wb") as f:
        pickle.dump(given, f)
    tool = os.path.join(ROOT, "tools", "extract_features.py")
    for mode, extra in (("det", []), ("boxes", ["--boxes", str(tmp_path / "boxes.pkl")])):
        r = subprocess.run([sys.executable, tool, "--imdb", "synthetic_4_21", "--net", "res50", "--batch", "2",
                            "--out", str(tmp_path / mode)] + extra, capture_output=True, text=True, cwd=ROOT)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    net, w = build("res50", 21, (8, 16, 32))
    ims = [cv2.imread(imdb.image_path_at(i)) for i in range(4)]
    prep = [_get_blobs(im) for im in ims]
    for g in ((0, 1), (2, 3)):                         # the tool's grouping: equal blob shapes, --batch 2
        blobs = np.concatenate([prep[i][0]["data"] for i in g], axis=0)
        scales, hws = [float(prep[i][1][0]) for i in g], [ims[i].shape[:2] for i in g]
        res, _ = net.detect_features(blobs, scales, hws)
        for i, (det, feats, roi) in zip(g, res):
            z = np.load(tmp_path / "det" / ("%d.npz" % i))
            assert np.array_equal(z["boxes"], det[:, :4]) and np.array_equal(z["scores"], det[:, 4])
            assert np.array_equal(z["classes"], det[:, 5].astype(np.int32)) and np.array_equal(z["features"], feats)
            assert np.array_equal(z["roi_index"], roi) and (int(z["image_h"]), int(z["image_w"])) == (375, 500)
        res, _ = net.score_boxes(blobs, scales, hws, [given[i] for i in g])
        for i, (scores, _, feats) in zip(g, res):
            z = np.load(tmp_path / "boxes" / ("%d.npz" % i))
            assert np.array_equal(z["boxes"], given[i]) and np.array_equal(z["scores"], scores)
            assert np.array_equal(z["features"], feats)


def test_bench_features_tool_runs(cuda):
    """tools/bench_features.py at a tiny setting: one JSON line with both throughputs and the gather kernel's bandwidth."""
    import json
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "bench_features.py"), "--net", "mobile", "--batch", "1",
                        "--steps", "2", "--warmup", "1", "--rounds", "1"], capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    line = json.loads([x for x in r.stdout.splitlines() if x.startswith("{")][-1])
    assert line["detect"]["value"] > 0 and line["features"]["value"] > 0
    k = line["kernel"]
    assert k["feature_dim"] == 1024 and k["max_det"] == 256 and 0 < k["detections"] <= 256 and k["achieved_gbs"] > 0 and k["us"] > 0
