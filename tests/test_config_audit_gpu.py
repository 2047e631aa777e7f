"""The `detect` graph audited step by step (graph_audit.run_audit: poisoned replay, every step against float64 or its exact
model on its own device inputs, then the eager re-run bit-equal) at the architecture and pooling options the production
configs do not set: MobileNet depth multipliers, RPN_CHANNELS, anchor sets of 1 and 25 anchors, POOLING_SIZE 1 to 16 in the
three pooling modes, RESNET.MAX_POOL, and VGG16 at POOLING_SIZE 14 and 4.  Each config names the path it is there for and
asserts it from the tape (output shapes, ConvPlan.info()); test_config_space.py checks the same claims without a GPU.

A MobileNet depth that is not a multiple of 32 runs zero-padded to one (nets/mobilenet_v1.py, pad_depths): the audit holds
the pad channels to exactly 0.  Two corruptions each fail at their layer: one element in the second M tile of a RoI whose
14 x 14 head map straddles two tiles, and one Conv2d_0 weight channel >= 8 of a MobileNet at multiplier 0.5 moved in the
engine's weights.  A MobileNet at multiplier 0.5 also matches the oracle's own chain end to end (test_e2e_gpu's criteria).

Observed worst err / bound per config and the module's runtime: tests/README.md."""
import numpy as np
import pytest
import torch

import conv_split_model as M
import net_ref64 as R
from graph_audit import build, run_audit
from oracle import pipeline as P
from tf_faster_rcnn_b200 import synth

pytestmark = pytest.mark.gpu
F = np.float32
HW, SMALL = (600, 800), (304, 400)
COCO4 = (4, 8, 16, 32)


def facts(rec):
    """{tape label: (output shape, ConvPlan.info() or None)}; the last record of a label wins (max_pool repeats)."""
    return {label: (tuple(out.shape), None if cp is None else cp.info()) for label, out, cp in rec}


def rows(info):
    return info["tile_n"] * info["tile_h"] * info["tile_w"]


def depth(f, label):
    return f[label][0][-1]


MB = "MobilenetV1/Conv2d_%d"
R101 = "resnet_v1_101/block4/unit_%d/bottleneck_v1/conv%d"


# (id, net, classes, anchor scales, anchor ratios, blob H x W, batch, cfg updates, build options, the path,
#  covers(facts, checkpoint, network))
CONFIGS = [
    ("mobile_dm025", "mobile", 81, COCO4, (0.5, 1, 2), HW, 1, {}, dict(depth_multiplier=0.25),
     "Conv2d_0 at 8 channels and Conv2d_1_pointwise's K of 8 channels, each zero-padded to one 32-channel k-block",
     lambda f, w, net: w[MB % 0 + "/weights"].shape[3] == 8 and depth(f, "conv_first:" + MB % 0) == 32
     and depth(f, "conv:" + MB % 1 + "_pointwise") == 32 and w[MB % 1 + "_pointwise/weights"].shape[2:] == (8, 16)),
    ("mobile_dm05_b2", "mobile", 81, COCO4, (0.5, 1, 2), HW, 2, {}, dict(depth_multiplier=0.5),
     "Conv2d_0 at 16 channels padded to 32, batch 2",
     lambda f, w, net: w[MB % 0 + "/weights"].shape[3] == 16 and depth(f, "conv_first:" + MB % 0) == 32
     and f["conv_first:" + MB % 0][0][0] == 2),
    ("mobile_dm075", "mobile", 81, COCO4, (0.5, 1, 2), SMALL, 1, {}, dict(depth_multiplier=0.75),
     "depths 24 and 48 padded to 32 and 64; K = 96 is three k-blocks",
     lambda f, w, net: depth(f, "conv_first:" + MB % 0) == 32 and depth(f, "conv:" + MB % 1 + "_pointwise") == 64
     and depth(f, "conv:" + MB % 2 + "_pointwise") == 96 and w[MB % 1 + "_pointwise/weights"].shape[3] == 48),
    ("mobile_dm125", "mobile", 81, COCO4, (0.5, 1, 2), SMALL, 1, {}, dict(depth_multiplier=1.25),
     "Conv2d_0 at 40 channels padded to 64 (conv_first's two-group path), depth 80 padded to 96",
     lambda f, w, net: w[MB % 0 + "/weights"].shape[3] == 40 and depth(f, "conv_first:" + MB % 0) == 64
     and depth(f, "conv:" + MB % 1 + "_pointwise") == 96 and depth(f, "conv:" + MB % 13 + "_pointwise") == 1280),
    ("res50_rpn256", "res50", 81, COCO4, (0.5, 1, 2), SMALL, 1, {}, dict(rpn_channels=256),
     "rpn_conv/3x3 with cout 256, the fused RPN heads with K = 256",
     lambda f, w, net: depth(f, "conv:resnet_v1_50/rpn_conv/3x3") == 256 and w["resnet_v1_50/rpn_cls_score/weights"].shape[2] == 256),
    ("vgg16_rpn128", "vgg16", 21, (8, 16, 32), (0.5, 1, 2), SMALL, 1, {}, dict(rpn_channels=128),
     "rpn_conv/3x3 with cout 128, the fused RPN heads with K = 128",
     lambda f, w, net: depth(f, "conv:vgg_16/rpn_conv/3x3") == 128 and w["vgg_16/rpn_bbox_pred/weights"].shape[2] == 128),
    ("res101_a1", "res101", 81, (8,), (1,), SMALL, 1, {}, {},
     "A = 1: the fused RPN head is 8 columns (cls 2 | pad 2 | bbox 4)",
     lambda f, w, net: depth(f, "conv:resnet_v1_101/rpn_heads") == 8),
    ("res101_a25", "res101", 81, (2, 4, 8, 16, 32), (0.25, 0.5, 1, 2, 4), HW, 1, {}, {},
     "A = 25: the fused RPN head is 152 columns (cls 50 | pad 2 | bbox 100), more than one N tile",
     lambda f, w, net: depth(f, "conv:resnet_v1_101/rpn_heads") == 152 and f["conv:resnet_v1_101/rpn_heads"][1]["block_n"] < 152),
    ("res101_crop14", "res101", 81, COCO4, (0.5, 1, 2), SMALL, 1, {"POOLING_SIZE": 14}, {},
     "crop P = 14: 196 rows per RoI, so RoIs straddle M tiles and the mean epilogue's groups span tiles",
     lambda f, w, net: f["conv:" + R101 % (1, 1)][0][1:3] == (14, 14)
     and rows(f["conv:" + R101 % (1, 1)][1]) < 196 and rows(f["conv:" + R101 % (3, 3)][1]) < 196
     and f["conv:" + R101 % (3, 3)][0] == (300, 2048)),
    ("res101_crop2", "res101", 81, COCO4, (0.5, 1, 2), SMALL, 1, {"POOLING_SIZE": 2}, {},
     "crop P = 2: 2 x 2 head maps, one M tile of the 3 x 3 convs holds many RoIs",
     lambda f, w, net: f["conv:" + R101 % (1, 2)][0][1:3] == (2, 2) and f["conv:" + R101 % (1, 2)][1]["tile_n"] > 1),
    ("res101_align1", "res101", 81, COCO4, (0.5, 1, 2), SMALL, 1, {"POOLING_MODE": "align", "POOLING_SIZE": 1}, {},
     "align P = 1: 1 x 1 head maps, every 3 x 3 tap but the centre is padding",
     lambda f, w, net: f["conv:" + R101 % (1, 2)][0][1:3] == (1, 1) and f["conv:" + R101 % (1, 2)][1]["tile_n"] > 1),
    ("res101_pool16", "res101", 81, COCO4, (0.5, 1, 2), SMALL, 1, {"POOLING_MODE": "pool", "POOLING_SIZE": 16}, {},
     "pool P = 16: 256 rows per RoI, the largest pooled size, over two M tiles",
     lambda f, w, net: f["conv:" + R101 % (1, 1)][0][1:3] == (16, 16) and rows(f["conv:" + R101 % (1, 1)][1]) <= 128),
    ("res101_maxpool", "res101", 81, COCO4, (0.5, 1, 2), SMALL, 1, {"RESNET.MAX_POOL": True}, {},
     "RESNET.MAX_POOL: ResNet takes the crop 14 + 2 x 2 max pool path at C = 1024",
     lambda f, w, net: net.crop_pre_pool() and f["conv:" + R101 % (1, 1)][0][1:] == (7, 7, 512)),
    ("vgg16_align14", "vgg16", 21, (8, 16, 32), (0.5, 1, 2), SMALL, 1, {"POOLING_MODE": "align", "POOLING_SIZE": 14}, {},
     "align P = 14: fc6 K = 14 * 14 * 512 = 100 352 (1568 k-blocks), four times the longest K of the production configs",
     lambda f, w, net: w["vgg_16/fc6/weights"].shape == (100352, 4096) and f["conv:vgg_16/fc6"][0] == (1, 1, 300, 4096)),
    ("vgg16_crop4", "vgg16", 21, (8, 16, 32), (0.5, 1, 2), SMALL, 1, {"POOLING_SIZE": 4}, {},
     "crop P = 4: an 8 x 8 crop + 2 x 2 max pool, fc6 K = 8192",
     lambda f, w, net: w["vgg_16/fc6/weights"].shape == (8192, 4096)),
    ("mobile_pool3", "mobile", 81, COCO4, (0.5, 1, 2), SMALL, 1, {"POOLING_MODE": "pool", "POOLING_SIZE": 3}, {},
     "pool P = 3: the head's depthwise and pointwise layers and the spatial mean on 3 x 3 maps",
     lambda f, w, net: f["depthwise:" + MB % 12 + "_depthwise"][0][1:3] == (3, 3) and f["spatial_mean"][0] == (300, 1024)),
]


def free(net, rec):
    """Release a network's plans and the recorded step outputs now: sixteen 600 x 800 networks do not fit at once."""
    rec.clear()
    for plan in net._plans.values():
        plan.release()
    net._plans.clear()
    net._aug_plans.clear()
    torch.cuda.empty_cache()


@pytest.mark.parametrize("cid,net_name,C,scales,ratios,hw,B,cfg_updates,arch,path,covers", CONFIGS, ids=[c[0] for c in CONFIGS])
def test_config_audit(cuda, monkeypatch, cid, net_name, C, scales, ratios, hw, B, cfg_updates, arch, path, covers):
    net, w, rec = build(monkeypatch, net_name, C, scales, cfg_updates, None, anchor_ratios=ratios, **arch)
    try:
        rows_ = run_audit(net_name, C, scales, hw, B, net, w, rec, M.F16X3, cid)
        worst = max(r.ratio for r in rows_)
        print("  %s -- %s; worst err/bound over all steps %.3f" % (cid, path, worst))
        assert covers(facts(rec), w, net), "%s no longer covers its path: %s" % (cid, path)
        assert worst <= 1
    finally:
        free(net, rec)


TEETH_P14 = "resnet_v1_50/block4/unit_1/bottleneck_v1/conv1"


def test_audit_names_a_corrupted_straddling_roi(cuda, monkeypatch):
    """Crop P = 14: RoI 0's 196 head rows fill the first M tile and part of the second.  One element of that second part moved
    by 1e-3 relative after the replay: the audit fails at that layer."""
    net, w, rec = build(monkeypatch, "res50", 21, (8, 16, 32), {"POOLING_SIZE": 14}, None)

    def corrupt(walk, steps):
        i = [l.key for l in walk].index(TEETH_P14)
        out, cp = steps[i][1]["out"], steps[i][2]
        tile = rows(cp.info())
        assert out.shape[1:3] == (14, 14) and tile < 196, (out.shape, cp.info())
        row = out.view(-1, out.shape[3])[tile + 10]              # RoI 0, in its second M tile
        j = int(torch.argmax(row.abs()))
        row[j] *= 1 + 1e-3
    try:
        with pytest.raises(R.Finding) as e:
            run_audit("res50", 21, (8, 16, 32), SMALL, 1, net, w, rec, M.F16X3, "corrupted straddling RoI", corrupt)
        print("\n" + str(e.value))
        assert str(e.value).startswith("conv:" + TEETH_P14 + ":"), str(e.value)
    finally:
        free(net, rec)


def test_audit_names_a_perturbed_first_layer_channel(cuda, monkeypatch):
    """Multiplier 0.5: Conv2d_0 has 16 channels.  Its channel 11 scaled by 1 + 1e-3 in the engine's weights only, the
    reference keeps the true tensors: the audit fails at conv_first."""
    key = "MobilenetV1/Conv2d_0/weights"

    def perturbed(w):
        w2 = dict(w)
        a = np.array(w[key], copy=True)
        a[..., 11] *= F(1 + 1e-3)
        w2[key] = a
        return w2
    net, w, rec = build(monkeypatch, "mobile", 21, (8, 16, 32), {}, None, weights=perturbed, depth_multiplier=0.5)
    try:
        assert w[key].shape[3] == 16
        with pytest.raises(R.Finding) as e:
            run_audit("mobile", 21, (8, 16, 32), SMALL, 1, net, w, rec, M.F16X3, "perturbed Conv2d_0")
        print("\n" + str(e.value))
        assert str(e.value).startswith("conv_first:MobilenetV1/Conv2d_0:"), str(e.value)
    finally:
        free(net, rec)


def test_depth_multiplier_detections_match_oracle(cuda, monkeypatch):
    """MobileNet at DEPTH_MULTIPLIER 0.5, 600 x 800: Network.detect against the oracle's own chain test_image -> im_detect_post
    -> test_net_post on the unpadded checkpoint, with test_e2e_gpu's criteria."""
    from test_e2e_gpu import compare_detections, fmt_report
    net, w, rec = build(monkeypatch, "mobile", 81, COCO4, {}, None, depth_multiplier=0.5)
    try:
        blob = synth.synthetic_blob(*HW)
        im_info = np.array([HW[0], HW[1], 1.0], F)
        o = P.opts(anchor_scales=COCO4)
        st = P.test_image("mobile", w, blob, im_info, 81, o)
        _, cls_prob, bbox_pred, rois = net.test_image(None, blob, im_info)
        plan = net.plan_for(*HW)
        keep = plan.roi_keep.cpu().numpy()[:rois.shape[0]]
        common, ia, ib = np.intersect1d(keep, st["roi_keep"], return_indices=True)
        e_prob = float(np.abs(cls_prob[ia] - st["cls_prob"][ib]).max())
        e_bbox = float(np.abs(bbox_pred[ia] - st["bbox_pred"][ib]).max())
        det, _ = net.detect(blob, im_info, HW)
        scores, boxes = P.im_detect_post(st["rois"], st["cls_prob"], st["bbox_pred"], 1.0, HW[0], HW[1])
        rep = compare_detections(det, P.test_net_post(scores, boxes, o))
        print("\n[mobile dm 0.5] RoIs gpu %d oracle %d common %d | cls_prob abs %.2e, bbox_pred abs %.2e | %s"
              % (rois.shape[0], st["rois"].shape[0], len(common), e_prob, e_bbox, fmt_report(rep)))
        assert len(common) >= 0.97 * len(st["roi_keep"])
        assert e_prob < 1e-4 and e_bbox < 1e-4
        assert rep["matched"] >= 0.95 * rep["n_want"] and rep["score_err"] < 1e-4 and rep["box_err"] < 4e-3
    finally:
        free(net, rec)
