"""POOLING_MODE 'align' / 'pool' on the GPU: frcnn_roi_align / frcnn_roi_pool against the numpy models bit for bit (outputs
between sentinel guard bands, inputs unchanged), the largest grid the caller-box bound admits, non-finite maps, and whole
networks at 600x800: pool5 on the GPU's own feature map and RoIs, the detection records against the oracle's post of the GPU's
own outputs, the oracle-alone chain, a batch of 3, detect_features, score_boxes and test-time augmentation with a flip."""
import os
import sys

import cv2
import numpy as np
import pytest
import torch

from oracle import nets as ON
from oracle import pipeline as P

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import aug_oracle as AO  # noqa: E402
import roi_pool_oracle as RP  # noqa: E402
from test_e2e_gpu import compare_detections, fmt_report  # noqa: E402
from tf_faster_rcnn_b200 import ops, synth

pytestmark = pytest.mark.gpu
F = np.float32
GUARD = 4096
SENT = F(-7.25e33)


@pytest.fixture(scope="module", autouse=True)
def _restore_network_registry():
    from nets import network
    before = list(network._REGISTRY)
    yield
    network._REGISTRY[:] = before


@pytest.fixture
def pool_cfg():
    from model.config import cfg
    saved = (cfg.POOLING_MODE, cfg.POOLING_SIZE, dict(cfg.ROI_ALIGN), dict(cfg.TEST.BBOX_AUG), tuple(cfg.TEST.SCALES),
             cfg.USE_GPU_NMS)
    yield cfg
    cfg.POOLING_MODE, cfg.POOLING_SIZE = saved[:2]
    cfg.ROI_ALIGN.update(saved[2])
    cfg.TEST.BBOX_AUG.update(saved[3])
    cfg.TEST.SCALES, cfg.USE_GPU_NMS = saved[4:]


def run(mode, feat, rois, pooled, sr=0, aligned=False):
    """One launch into a buffer between sentinel guard bands; the guards and both inputs are checked afterwards."""
    fd, rd = torch.from_numpy(np.ascontiguousarray(feat)).cuda(), torch.from_numpy(np.ascontiguousarray(rois)).cuda()
    R, C = rois.shape[0], feat.shape[3]
    n = R * pooled * pooled * C
    buf = torch.full((n + 2 * GUARD,), float(SENT), dtype=torch.float32, device="cuda")
    out = buf[GUARD:GUARD + n].view(R, pooled, pooled, C)
    if mode == "align":
        ops.roi_align(fd, rd, pooled, 1.0 / 16, sr, aligned, out)
    else:
        ops.roi_pool(fd, rd, pooled, 1.0 / 16, out)
    torch.cuda.synchronize()
    b = buf.cpu().numpy()
    assert (b[:GUARD] == SENT).all() and (b[GUARD + n:] == SENT).all(), "write outside the output"
    assert fd.cpu().numpy().tobytes() == np.ascontiguousarray(feat).tobytes() and rd.cpu().numpy().tobytes() == rois.tobytes()
    return b[GUARD:GUARD + n].reshape(R, pooled, pooled, C)


def model(mode, feat, rois, pooled, sr=0, aligned=False):
    return RP.roi_align_model(feat, rois, pooled, sr, aligned) if mode == "align" else RP.roi_pool_model(feat, rois, pooled)


def same(got, want):
    """Bit for bit, except that any NaN equals any NaN (the device's NaN is the canonical one, numpy keeps payloads)."""
    nan = np.isnan(got) & np.isnan(want)
    return bool((nan | ((got == want) & (np.signbit(got) == np.signbit(want)))).all())


MODES = [("align", 0, False), ("align", 2, True), ("align", 0, True), ("align", 4, False), ("pool", 0, False)]


def batch_rois(rng, h, w, n_random):
    rois = RP.edge_rois(h, w, rng, n_random)
    rois[:, 0] = np.resize(np.array([-1, 0, 1, 2, 5], F), rois.shape[0])     # image index clamp: -1 -> 0, 5 -> 2
    return rois


@pytest.mark.parametrize("C", [4, 64, 512, 1024, 2048])
def test_kernels_equal_model(cuda, C):
    rng = np.random.default_rng(C)
    feat = rng.standard_normal((3, 38, 50, C)).astype(F)
    rois = batch_rois(rng, 38, 50, 40 if C <= 512 else 16)
    sizes = (1, 2, 7, 14, 16) if C <= 64 else (7,)
    for pooled in sizes:
        for mode, sr, aligned in MODES:
            got = run(mode, feat, rois, pooled, sr, aligned)
            assert got.tobytes() == model(mode, feat, rois, pooled, sr, aligned).tobytes(), (pooled, mode, sr, aligned)


@pytest.mark.parametrize("hw,box,sizes", [
    ((38, 50), (-800, -608, 1600, 1216), (1, 7, 16)),        # whole [-W, 2W] x [-H, 2H]: up to 150 x 114 samples per bin at P=1
    ((4, 200), (-3200, -64, 6400, 128), (1, 2)),             # 600 samples per bin across: the x table is walked in passes
])
def test_largest_grid_the_bound_admits(cuda, hw, box, sizes):
    rng = np.random.default_rng(hw[1])
    feat = rng.standard_normal((1,) + hw + (4,)).astype(F)
    rois = np.array([[0] + list(box), [0, 10, 10, 300, 200]], F)
    for pooled in sizes:
        for mode, sr, aligned in ((m, 0, a) for m, a in (("align", False), ("align", True), ("pool", False))):
            got = run(mode, feat, rois, pooled, sr, aligned)
            assert got.tobytes() == model(mode, feat, rois, pooled, sr, aligned).tobytes(), (pooled, mode, aligned)


def test_non_finite_map(cuda):
    """NaN / +-Inf in the map, cell (0,0) included: the kernels follow the model's rule (an out-of-range sample is not read;
    the RoIPool max skips NaN), which differs from torchvision only where that cell is non-finite (test_roi_pool.py)."""
    rng = np.random.default_rng(8)
    feat = rng.standard_normal((2, 9, 13, 8)).astype(F)
    feat[:, 0, 0, :4] = [np.nan, np.inf, -np.inf, np.nan]
    feat[0, 4, 6, 2:6] = [np.inf, np.nan, -np.inf, np.nan]
    feat[1, 8, 12, :] = np.nan
    rois = batch_rois(rng, 9, 13, 40)
    for pooled in (2, 7):
        for mode, sr, aligned in MODES:
            got = run(mode, feat, rois, pooled, sr, aligned)
            assert same(got, model(mode, feat, rois, pooled, sr, aligned)), (pooled, mode, sr, aligned)


# ---- whole networks ---------------------------------------------------------------------------------------------------------
_NETS = {}


def network(net_name, C, scales, cfg, mode, sr=0, aligned=False):
    """The network of net_name (built once per module) re-created for the pooling mode; its weights and the oracle's front half
    (backbone, RPN, proposals: independent of the pooling) are kept."""
    from nets.vgg16 import vgg16
    from nets.resnet_v1 import resnetv1
    from nets.mobilenet_v1 import mobilenetv1
    cfg.TEST.HAS_RPN = True
    cfg.POOLING_MODE = mode
    cfg.ROI_ALIGN.update(SAMPLING_RATIO=sr, ALIGNED=aligned)
    if net_name not in _NETS:
        net = vgg16() if net_name == "vgg16" else mobilenetv1() if net_name == "mobile" else resnetv1(num_layers=int(net_name[3:]))
        net.create_architecture("TEST", C, tag="default", anchor_scales=scales, anchor_ratios=(0.5, 1, 2))
        w = synth.make(net_name, C, 3 * len(scales))
        net.load_weights(w)
        _NETS[net_name] = [net, w, None]
    net, w, _ = _NETS[net_name]
    net.create_architecture("TEST", C, tag="default", anchor_scales=scales, anchor_ratios=(0.5, 1, 2))
    net.options["use_gpu_nms"] = False                  # the cpu_nms predicate of the oracle's test_net_post
    return net, w


def own_outputs(plan, b):
    R, n = plan.R, int(plan.num_rois[b].item())
    return plan.cls_prob[b * R:b * R + n].cpu().numpy(), plan.pred_boxes[b * R:b * R + n].cpu().numpy()


def records_from(out):
    rows = [np.hstack([d, np.full((d.shape[0], 1), j, F)]) for j, d in enumerate(out) if d.shape[0]]
    return np.vstack(rows).astype(F) if rows else np.zeros((0, 6), F)


def check_pool5(plan, pool):
    """The plan's pool5 is the model applied to the plan's own feature map and RoI rows (all of them), bit for bit."""
    assert plan.pool5.cpu().numpy().tobytes() == pool(plan.feat.cpu().numpy(), plan.rois.cpu().numpy()).tobytes()


# the end-to-end box bounds of test_e2e_gpu.FULL_CONFIGS at 600x800
BOX_TOL = {"res101": 5e-3, "vgg16": 9e-3, "mobile": 4e-3}
NET_CONFIGS = [
    ("res101", "align", 0, False), ("res101", "align", 0, True), ("res101", "align", 2, False), ("res101", "pool", 0, False),
    ("vgg16", "align", 0, False), ("vgg16", "pool", 0, False), ("mobile", "align", 0, False), ("mobile", "pool", 0, False),
]


@pytest.mark.parametrize("net_name,mode,sr,aligned", NET_CONFIGS, ids=["%s-%s-sr%d%s" % (c[0], c[1], c[2], "-aligned" if c[3] else "")
                                                                       for c in NET_CONFIGS])
def test_whole_network(cuda, pool_cfg, net_name, mode, sr, aligned):
    C, scales, hw = 81, (4, 8, 16, 32), (600, 800)
    net, w = network(net_name, C, scales, pool_cfg, mode, sr, aligned)
    pool = RP.pool_stage(mode, 7, sr, aligned)
    o = P.opts(anchor_scales=scales, use_gpu_nms=False)
    blob = synth.synthetic_blob(*hw)
    im_info = np.array([hw[0], hw[1], 1.0], F)
    # test_image: pool5 on the GPU's own map and RoIs bit for bit, fc7 against the oracle head on that pool5
    _, _, _, rois = net.test_image(None, blob, im_info)
    plan = net.plan_for(*hw)
    assert [s[0] for s in plan.tape.steps].count("roi_" + mode) == 1 and "crop_pool" not in [s[0] for s in plan.tape.steps]
    check_pool5(plan, pool)
    r = rois.shape[0]
    fc7_want = ON.head_to_tail(net_name, w, plan.pool5[:r].cpu().numpy())
    fc7 = plan.fc7[:r].cpu().numpy()
    e_fc7 = float(np.abs(fc7 - fc7_want).max() / np.abs(fc7_want).max())
    # detect: the records are the oracle's post of the GPU's own outputs
    det, plan = net.detect(blob, im_info, hw)
    prob, pred = own_outputs(plan, 0)
    assert det.shape[0] > 0 and det.tobytes() == records_from(P.test_net_post(prob, pred, o)).tobytes()
    # the oracle alone (nothing of the GPU run fed to it)
    ent = _NETS[net_name]
    if ent[2] is None:
        ent[2] = RP.front(net_name, w, blob, im_info, o)
    st = RP.head(net_name, w, ent[2], C, o, pool)
    scores, boxes = P.im_detect_post(st["rois"], st["cls_prob"], st["bbox_pred"], 1.0, hw[0], hw[1])
    rep = compare_detections(det, P.test_net_post(scores, boxes, o), tol=BOX_TOL[net_name])
    print("\n[%s %s sr=%d aligned=%s 600x800] fc7 rel err %.2e | %s" % (net_name, mode, sr, aligned, e_fc7, fmt_report(rep)))
    assert e_fc7 < 1e-4
    assert rep["matched"] == rep["n_want"] == rep["n_got"] and rep["score_err"] < 1e-4
    # a batch of 3 through one graph replay
    blobs = np.concatenate([synth.synthetic_blob(hw[0], hw[1], seed) for seed in (1, 2, 3)], axis=0)
    dets3, plan3 = net.detect_batch(blobs, [1.0] * 3, [hw] * 3)
    check_pool5(plan3, pool)
    feat3, rois3, pool53 = plan3.feat, plan3.rois, plan3.pool5.cpu().numpy()
    R = plan3.R
    for b in range(3):
        prob, pred = own_outputs(plan3, b)
        assert dets3[b].tobytes() == records_from(P.test_net_post(prob, pred, o)).tobytes(), b
        # the pooling kernel over the batch == the kernel over image b alone
        rb = rois3[b * R:(b + 1) * R].cpu().numpy().copy()
        assert (rb[:, 0] == b).all()
        rb[:, 0] = 0
        one = run(mode, np.ascontiguousarray(feat3[b:b + 1].cpu().numpy()), rb, 7, sr, aligned)
        assert one.tobytes() == pool53[b * R:(b + 1) * R].tobytes(), b
        single, _ = net.detect(blobs[b:b + 1], im_info, hw)
        rep = compare_detections(dets3[b], [single[single[:, 5] == j, :5] for j in range(C)])
        assert rep["matched"] >= 0.95 * max(single.shape[0], 1) and rep["score_err"] < 1e-4, fmt_report(rep)


# ---- the other detection paths, once each in align mode ------------------------------------------------------------------
def test_detect_features_align(cuda, pool_cfg):
    net, w = network("res50", 21, (8, 16, 32), pool_cfg, "align", 2, True)
    hw = (224, 304)
    blobs = np.concatenate([synth.synthetic_blob(hw[0], hw[1], seed) for seed in (4, 5)], axis=0)
    scales, orig = [1.0, 1.25], [(224, 304), (179, 243)]
    res, plan = net.detect_features(blobs, scales, orig)
    check_pool5(plan, RP.pool_stage("align", 7, 2, True))
    fc7, R = plan.fc7.cpu().numpy(), plan.R
    o = P.opts(use_gpu_nms=False)
    for b, (det, feats, roi) in enumerate(res):
        prob, pred = own_outputs(plan, b)
        assert det.shape[0] > 0 and det.tobytes() == records_from(P.test_net_post(prob, pred, o)).tobytes()
        assert np.array_equal(feats, fc7[b * R + roi])
    for (det, _, _), want in zip(res, net.detect_batch(blobs, scales, orig)[0]):
        assert det.tobytes() == want.tobytes()


def test_score_boxes_align(cuda, pool_cfg):
    net, w = network("res50", 21, (8, 16, 32), pool_cfg, "align", 0, False)
    pool = RP.pool_stage("align", 7, 0, False)
    hw, scale = (224, 304), 1.25
    blob = synth.synthetic_blob(hw[0], hw[1], 6)
    orig = (179, 243)
    rng = np.random.default_rng(6)
    xy = rng.uniform(-60, 230, (40, 2)); wh = rng.uniform(1, 150, (40, 2))
    boxes = np.hstack([xy, xy + wh]).astype(F)
    boxes[0] = [-179, -143, 2 * 243 - 1, 2 * 179 - 1]        # near the [-W, 2W] x [-H, 2H] bound of the blob
    out, plan = net.score_boxes(blob, [scale], [orig], [boxes])
    n = boxes.shape[0]
    assert plan.pool5[:n].cpu().numpy().tobytes() == pool(plan.feat.cpu().numpy(), plan.rois[:n].cpu().numpy()).tobytes()
    st = RP.score_boxes("res50", w, blob, boxes, scale, orig, P.opts(), pool)
    scores, pred, feats = out[0]
    assert np.abs(scores - st["scores"]).max() < 1e-4 and np.abs(pred - st["pred_boxes"]).max() < 5e-3
    assert np.abs(feats - st["fc7"]).max() < 1e-4 * np.abs(st["fc7"]).max()
    with pytest.raises(ValueError):
        net.score_boxes(blob, [scale], [orig], [np.array([[0, 0, 600, 10]], F)])


def test_tta_flip_align(cuda, pool_cfg):
    from model.test import _run_aug, _set_post_options
    net, w = network("res50", 21, (8, 16, 32), pool_cfg, "align", 0, False)
    pool_cfg.TEST.SCALES = (288,)
    pool_cfg.USE_GPU_NMS = False
    pool_cfg.TEST.BBOX_AUG.update(ENABLED=True, H_FLIP=True)
    _set_post_options(net, 0.0, 100)
    im = cv2.blur(np.random.default_rng(2).integers(0, 256, (240, 320, 3), dtype=np.uint8), (5, 5))
    aug = _run_aug(net, [im], detect=True)
    pool = RP.pool_stage("align", 7, 0, False)
    sc, bx = [], []
    for v, (h, wd, _) in enumerate(aug.views):
        p = aug.subs[(h, wd)]
        check_pool5(p, pool)
        k = aug.view_slot[v] * aug.batch
        n, R = int(p.num_rois[k].item()), p.R
        sc.append(p.cls_prob[k * R:k * R + n].cpu().numpy()); bx.append(p.pred_boxes[k * R:k * R + n].cpu().numpy())
    assert [v[2] for v in aug.views] == [True, False]
    s, x = AO.union(sc, bx, [v[2] for v in aug.views], im.shape[1])
    want = records_from(AO.post(s, x, P.opts(use_gpu_nms=False, nms_thresh=pool_cfg.TEST.NMS)))
    recs = aug.records()[0]
    assert recs.shape[0] > 0 and recs.tobytes() == want.tobytes()
