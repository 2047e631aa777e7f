"""Soft-NMS on the GPU: nms_wrapper.soft_nms and frcnn_detect_post_soft against the sequential C oracle, bit for bit; `hard`
against the greedy post; the whole network through detect / detect_batch / detect_features / the Python loop; and option
toggles on one shape plan (no stale graph is replayed)."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import pipeline as P

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import soft_nms_oracle as SO  # noqa: E402
from test_e2e_gpu import compare_detections, fmt_report  # noqa: E402
from test_soft_nms import PARAMS, make_set  # noqa: E402
from tf_faster_rcnn_b200 import engine, ops, synth

pytestmark = pytest.mark.gpu
F = np.float32


@pytest.mark.parametrize("n", [1, 2, 63, 64, 65, 300, 1000, 5000, 8192])
def test_wrapper_matches_oracle(cuda, n):
    from model.nms_wrapper import soft_nms
    rng = np.random.default_rng(n)
    families = ("clustered", "tied", "duplicates", "degenerate", "mixed")
    picks = PARAMS if n <= 1000 else PARAMS[::5]
    for k, (m, s, nt, thr) in enumerate(picks):
        d = make_set(rng, n, families[k % len(families)])
        want_rows, want_keep = SO.soft_nms_c(d, m, s, nt, thr)
        rows, keep = soft_nms(d, sigma=s, overlap_thresh=nt, score_thresh=thr, method=m)
        assert np.array_equal(keep, want_keep), (n, m, s, nt, thr)
        assert rows.dtype == F and rows.tobytes() == want_rows.tobytes(), (n, m, s, nt, thr)
    rows, keep = soft_nms(np.zeros((0, 5), F))
    assert rows.shape == (0, 5) and keep == []


def stage_inputs(seed, r, C, batch=1):
    """Synthetic cls_prob [batch*r, C] (softmax rows) and pred_boxes [batch*r, 4C] with clustered boxes per class."""
    rng = np.random.default_rng(seed)
    prob = rng.dirichlet(np.full(C, 0.3), batch * r).astype(F)
    boxes = np.zeros((batch * r, C, 4), F)
    for j in range(C):
        for b in range(batch):
            d = make_set(rng, r, ("clustered", "duplicates")[j % 2])
            boxes[b * r:(b + 1) * r, j] = d[:, :4]
    return prob, boxes.reshape(batch * r, 4 * C)


def run_post(prob, pred, r, C, batch, nroi, thresh, soft, mpi, nt=0.3):
    max_det = 2 * mpi + 56 if mpi > 0 else r * (C - 1)
    cp, pb = torch.from_numpy(prob).cuda(), torch.from_numpy(pred).cuda()
    num = torch.tensor(nroi, dtype=torch.int32).cuda()
    det = ops.zeros((batch, max_det, 6)); ndet = ops.zeros((batch,), dtype=torch.int32)
    keep = ops.zeros((batch, C, r), dtype=torch.int32); cnt = ops.zeros((batch, C), dtype=torch.int32); ks = ops.zeros((batch, C, r))
    if soft is None:
        t32, flags = engine.nms_threshold(nt, True)
        ops.detect_post(cp, pb, num, C, thresh, t32, flags, mpi, det, ndet, keep, cnt, ks, ops.detect_post_workspace(r, C, batch), batch)
    else:
        code, s32, p32 = engine.soft_nms_args(*soft)
        ops.detect_post_soft(cp, pb, num, C, thresh, code, s32, float(F(nt)), p32, mpi, det, ndet, keep, cnt, ks, batch)
    torch.cuda.synchronize()
    ndet = ndet.cpu().numpy()
    assert (ndet <= max_det).all()
    dets = [det[b, :ndet[b]].cpu().numpy() for b in range(batch)]
    return dets, keep.cpu().numpy(), cnt.cpu().numpy()


def records_from(out):
    rows = [np.hstack([d, np.full((d.shape[0], 1), j, F)]) for j, d in enumerate(out) if d.shape[0]]
    return np.vstack(rows).astype(F) if rows else np.zeros((0, 6), F)


@pytest.mark.parametrize("r,C", [(300, 21), (300, 81), (1000, 81), (5000, 21)])
def test_post_stage_matches_oracle(cuda, r, C):
    thresh = 0.0 if r <= 1000 else 0.02
    prob, pred = stage_inputs(r + C, r, C)
    nroi = [r - 7]
    for soft, mpi in ((("linear", 0.5, 0.001), 100), (("gaussian", 0.5, 0.001), 0), (("hard", 0.5, 0.001), 100),
                      (("gaussian", 0.1, 0.1), 100)):
        (det,), keep, cnt = run_post(prob, pred, r, C, 1, nroi, thresh, soft, mpi)
        out, idx = SO.test_net_post_soft(prob[:nroi[0]], pred[:nroi[0]], soft, 0.3, mpi, thresh)
        assert det.tobytes() == records_from(out).tobytes(), soft
        for j in range(C):
            assert cnt[0, j] == idx[j].shape[0] and np.array_equal(keep[0, j, :cnt[0, j]], idx[j]), (soft, j)
            assert (keep[0, j, cnt[0, j]:] == -1).all()


@pytest.mark.parametrize("r,C", [(300, 81), (1000, 21), (5000, 21)])
def test_post_stage_batch_equals_single_images(cuda, r, C):
    thresh = 0.0 if r <= 1000 else 0.02
    prob, pred = stage_inputs(7 * r + C, r, C, batch=3)
    nroi = [r, r - 50, r // 2]
    soft = ("linear", 0.5, 0.001)
    dets3, keep3, cnt3 = run_post(prob, pred, r, C, 3, nroi, thresh, soft, 100)
    for b in range(3):
        (det,), keep, cnt = run_post(prob[b * r:(b + 1) * r], pred[b * r:(b + 1) * r], r, C, 1, nroi[b:b + 1], thresh, soft, 100)
        assert det.tobytes() == dets3[b].tobytes() and np.array_equal(cnt[0], cnt3[b]) and np.array_equal(keep[0], keep3[b])


@pytest.mark.parametrize("r,C", [(300, 81), (5000, 21)])
def test_hard_equals_greedy_post_on_distinct_scores(cuda, r, C):
    prob, pred = stage_inputs(3 * r + C, r, C)
    rng = np.random.default_rng(r)
    for j in range(C):                               # distinct scores per class
        prob[:, j] = (rng.permutation(r) + 1).astype(F) / F(r + 1)
    thresh = 0.001 if r <= 1000 else 0.02            # candidates above the prune threshold: only overlap can drop them
    for mpi in (100, 0):
        soft, _, _ = run_post(prob, pred, r, C, 1, [r], thresh, ("hard", 0.5, 0.001), mpi)
        greedy, _, _ = run_post(prob, pred, r, C, 1, [r], thresh, None, mpi)
        assert soft[0].tobytes() == greedy[0].tobytes()


def build(net_name, num_classes, scales):
    from model.config import cfg
    from nets.resnet_v1 import resnetv1
    from nets.mobilenet_v1 import mobilenetv1
    cfg.TEST.HAS_RPN = True
    net = mobilenetv1() if net_name == "mobile" else resnetv1(num_layers=int(net_name[3:]))
    net.create_architecture("TEST", num_classes, tag="default", anchor_scales=scales, anchor_ratios=(0.5, 1, 2))
    w = synth.make(net_name, num_classes, 3 * len(scales))
    net.load_weights(w)
    return net, w


def own_outputs(plan, b):
    """The GPU's own cls_prob / pred_boxes rows of image b after a launch."""
    R = plan.R
    n = int(plan.num_rois[b].item())
    return plan.cls_prob[b * R:b * R + n].cpu().numpy(), plan.pred_boxes[b * R:b * R + n].cpu().numpy()


@pytest.fixture
def soft_cfg():
    from model.config import cfg
    sn = cfg.TEST.SOFT_NMS
    saved = dict(sn)
    yield sn
    sn.update(saved)


@pytest.mark.parametrize("net_name,box_tol", [("res101", 5e-3), ("mobile", 4e-3)])
def test_whole_network_detect_and_detect_batch(cuda, soft_cfg, net_name, box_tol):
    from model.test import _detections_python_loop, _set_post_options
    import model.test as T
    C, scales, hw = 81, (4, 8, 16, 32), (600, 800)
    net, w = build(net_name, C, scales)
    soft_cfg.update(ENABLED=True, METHOD="linear")
    _set_post_options(net, 0.0, 100)
    soft = net.options["soft_nms"]
    blobs = [synth.synthetic_blob(hw[0], hw[1], seed) for seed in (1, 2)]
    im_info = np.array([hw[0], hw[1], 1.0], F)
    det, plan = net.detect(blobs[0], im_info, hw)
    scores, boxes = own_outputs(plan, 0)
    out, _ = SO.test_net_post_soft(scores, boxes, soft, 0.3, 100)
    assert det.shape[0] >= 100 and det.tobytes() == records_from(out).tobytes()
    # the FUSED_POST = False loop over nms_wrapper.soft_nms gives the same records
    assert T.FUSED_POST
    loop = _detections_python_loop(scores, boxes, C, 0.0, 100)
    assert records_from(loop).tobytes() == det.tobytes()
    # against the oracle-alone chain: the end-to-end matching rules of test_e2e_gpu
    o = P.opts(anchor_scales=scales)
    st = P.test_image(net_name, w, blobs[0], im_info, C, o)
    sc_o, bx_o = P.im_detect_post(st["rois"], st["cls_prob"], st["bbox_pred"], 1.0, hw[0], hw[1])
    rep = compare_detections(det, SO.test_net_post_soft(sc_o, bx_o, soft, 0.3, 100)[0])
    print("\n[%s 600x800 soft-NMS linear vs oracle chain] %s" % (net_name, fmt_report(rep)))
    assert rep["matched"] >= 0.95 * rep["n_want"] and rep["score_err"] < 1e-4 and rep["box_err"] < box_tol
    # batch of 2 through one replay, gaussian
    soft_cfg.update(METHOD="gaussian")
    _set_post_options(net, 0.0, 100)
    dets, plan2 = net.detect_batch(np.concatenate(blobs, axis=0), [1.0, 1.0], [hw, hw])
    for b in range(2):
        scores, boxes = own_outputs(plan2, b)
        out, _ = SO.test_net_post_soft(scores, boxes, net.options["soft_nms"], 0.3, 100)
        assert dets[b].tobytes() == records_from(out).tobytes(), b


def test_features_and_option_toggles(cuda, soft_cfg):
    from model.test import _set_post_options
    C, scales, hw = 21, (8, 16, 32), (224, 304)
    net, _ = build("res50", C, scales)
    blobs = np.concatenate([synth.synthetic_blob(hw[0], hw[1], seed) for seed in (1, 2, 3)], axis=0)
    sc, orig = [1.0, 1.25, 0.8], [(224, 304), (179, 243), (280, 380)]
    soft_cfg.update(ENABLED=True, METHOD="gaussian")
    _set_post_options(net, 0.0, 100)
    res, plan = net.detect_features(blobs, sc, orig)
    fc7 = plan.fc7.cpu().numpy()
    for b, ((det, feats, roi), want) in enumerate(zip(res, net.detect_batch(blobs, sc, orig)[0])):
        assert det.shape[0] > 0 and det.tobytes() == want.tobytes()
        assert np.array_equal(feats, fc7[b * plan.R + roi])
    # enabled -> disabled -> gaussian -> linear on one plan: each launch computes what a direct call of its post computes
    for enabled, method in ((True, "linear"), (False, "linear"), (True, "gaussian"), (True, "linear")):
        soft_cfg.update(ENABLED=enabled, METHOD=method)
        _set_post_options(net, 0.0, 100)
        dets, plan = net.detect_batch(blobs, sc, orig)
        for b in range(3):
            prob, pred = own_outputs(plan, b)
            n = prob.shape[0]
            (direct,), _, _ = run_post(prob, pred, n, C, 1, [n], 0.0, net.options["soft_nms"], 100)
            assert dets[b].tobytes() == direct.tobytes(), (enabled, method, b)
            if enabled:
                out, _ = SO.test_net_post_soft(prob, pred, net.options["soft_nms"], 0.3, 100)
                assert dets[b].tobytes() == records_from(out).tobytes()
