"""Box voting on the GPU: nms_wrapper.box_voting / frcnn_box_vote_host and frcnn_detect_post_vote / _soft_vote against the C
oracle bit for bit (outputs guard-banded, inputs checked unchanged); the ID invariants; the whole network through detect,
detect_batch, detect_features, test-time augmentation and the Python loop; and option toggles on one shape plan."""
import os
import sys

import cv2
import numpy as np
import pytest
import torch

from oracle import pipeline as P

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import box_vote_oracle as BV  # noqa: E402
from stage_ref64 import check_guarded, guarded_out  # noqa: E402
from test_box_vote import METHODS, make_vote_case  # noqa: E402
from test_e2e_gpu import compare_detections, fmt_report  # noqa: E402
from test_soft_nms_gpu import build, own_outputs, records_from, stage_inputs  # noqa: E402
from tf_faster_rcnn_b200 import engine, ops, synth

pytestmark = pytest.mark.gpu
F = np.float32


@pytest.fixture(scope="module", autouse=True)
def _restore_network_registry():
    from nets import network
    before = list(network._REGISTRY)
    yield
    network._REGISTRY[:] = before


@pytest.fixture
def vote_cfg():
    from model.config import cfg
    saved = (dict(cfg.TEST.BBOX_VOTE), dict(cfg.TEST.SOFT_NMS), dict(cfg.TEST.BBOX_AUG), tuple(cfg.TEST.SCALES), cfg.USE_GPU_NMS)
    yield cfg.TEST.BBOX_VOTE
    cfg.TEST.BBOX_VOTE.update(saved[0]); cfg.TEST.SOFT_NMS.update(saved[1]); cfg.TEST.BBOX_AUG.update(saved[2])
    cfg.TEST.SCALES, cfg.USE_GPU_NMS = saved[3:]


@pytest.mark.parametrize("n", [1, 31, 33, 300, 1024, 1025, 5000, 8192])
def test_wrapper_matches_oracle(cuda, n):
    from model.nms_wrapper import box_voting
    rng = np.random.default_rng(n)
    fams = ("clustered", "tied", "duplicates", "degenerate", "mixed")
    for k, m in enumerate(METHODS):
        th, b = (0.5, 0.8, 1.0)[k % 3], (0.5, 1.0, 2.0)[(k // 3) % 3]
        top, a = make_vote_case(rng, max(n - 4, 0), fams[k % len(fams)])
        a = a[:n]
        top0, a0 = top.copy(), a.copy()
        got = box_voting(top, a, th, m, b)
        assert np.array_equal(top, top0) and np.array_equal(a, a0)
        want = BV.box_vote_c(top, a, th, m, b)
        assert got.dtype == F and got.tobytes() == want.tobytes(), (n, m, th, b)
    assert box_voting(np.zeros((0, 5), F), np.zeros((3, 5), F), 0.8).shape == (0, 5)


def run_post(prob, pred, r, C, batch, nroi, thresh, soft, mpi, vote, nt=0.3):
    """The post entries on guard-banded outputs; vote = (VOTE_TH, METHOD, BETA) or None.  -> (records per image, keep, keep_cnt,
    keep_score, ndet)."""
    max_det = 2 * mpi + 56 if mpi > 0 else r * (C - 1)
    cp, pb = torch.from_numpy(prob).cuda(), torch.from_numpy(pred).cuda()
    num = torch.tensor(nroi, dtype=torch.int32).cuda()
    ins = [t.clone() for t in (cp, pb, num)]
    gd, det = guarded_out((batch, max_det, 6), 0.0)
    gn, ndet_f = guarded_out((batch,), 0.0)
    ndet = ndet_f.view(torch.int32)
    gk, keep_f = guarded_out((batch, C, r), 0.0)
    keep = keep_f.view(torch.int32)
    gc, cnt_f = guarded_out((batch, C), 0.0)
    cnt = cnt_f.view(torch.int32)
    gs, ks = guarded_out((batch, C, r), 0.0)
    gv, vb = guarded_out((batch, C, r, 4), float("nan"))
    v = None if vote is None else (*engine.box_vote_args(*vote), vb)
    if soft is None:
        t32, flags = engine.nms_threshold(nt, True)
        ops.detect_post(cp, pb, num, C, thresh, t32, flags, mpi, det, ndet, keep, cnt, ks, ops.detect_post_workspace(r, C, batch), batch,
                        vote=v)
    else:
        code, s32, p32 = engine.soft_nms_args(*soft)
        ops.detect_post_soft(cp, pb, num, C, thresh, code, s32, float(F(nt)), p32, mpi, det, ndet, keep, cnt, ks, batch, vote=v)
    torch.cuda.synchronize()
    for g, t in ((gd, det), (gn, ndet), (gk, keep), (gc, cnt), (gs, ks), (gv, vb)):
        check_guarded(g, t.numel())
    for a, b in zip(ins, (cp, pb, num)):
        assert torch.equal(a, b), "input changed"
    nd = ndet.cpu().numpy()
    assert (nd <= max_det).all()
    return [det[b, :nd[b]].cpu().numpy() for b in range(batch)], keep.cpu().numpy(), cnt.cpu().numpy(), ks.cpu().numpy(), nd


def check_against_oracle(det, keep, cnt, prob, pred, vote, soft, mpi, thresh, what):
    out, idx = BV.test_net_post_vote(prob, pred, vote, 0.3, mpi, thresh, soft=soft)
    assert det.tobytes() == records_from(out).tobytes(), what
    for j in range(prob.shape[1]):
        assert cnt[j] == idx[j].shape[0] and np.array_equal(keep[j, :cnt[j]], idx[j]), (what, j)
        assert (keep[j, cnt[j]:] == -1).all()


VOTES = [(0.8, "ID", 1.0), (0.5, "AVG", 1.0), (0.8, "IOU_AVG", 1.0), (0.6, "GENERALIZED_AVG", 2.0), (0.8, "QUASI_SUM", 0.5),
         (1.0, "TEMP_AVG", 0.5)]


@pytest.mark.parametrize("r,C", [(300, 21), (300, 81), (1000, 81), (5000, 21)])
@pytest.mark.parametrize("soft", [None, ("linear", 0.5, 0.001)])
def test_post_stage_matches_oracle(cuda, r, C, soft):
    thresh = 0.0 if r <= 1000 else 0.02
    prob, pred = stage_inputs(r + C, r, C)
    nroi = [r - 7]
    for k, vote in enumerate(VOTES if r <= 1000 else VOTES[::2]):
        mpi = 0 if k == 2 else 100
        (det,), keep, cnt, _, _ = run_post(prob, pred, r, C, 1, nroi, thresh, soft, mpi, vote)
        check_against_oracle(det, keep[0], cnt[0], prob[:nroi[0]], pred[:nroi[0]], vote, soft, mpi, thresh, (vote, soft))


@pytest.mark.parametrize("soft", [None, ("gaussian", 0.5, 0.001)])
def test_post_stage_batch_equals_single_images(cuda, soft):
    r, C = 300, 81
    prob, pred = stage_inputs(11 * r + C, r, C, batch=3)
    nroi = [0, 137, 300]
    vote = (0.7, "AVG", 1.0)
    dets3, keep3, cnt3, _, nd3 = run_post(prob, pred, r, C, 3, nroi, 0.0, soft, 100, vote)
    assert nd3[0] == 0
    for b in range(3):
        (det,), keep, cnt, _, _ = run_post(prob[b * r:(b + 1) * r], pred[b * r:(b + 1) * r], r, C, 1, nroi[b:b + 1], 0.0, soft, 100, vote)
        assert det.tobytes() == dets3[b].tobytes() and np.array_equal(cnt[0], cnt3[b]) and np.array_equal(keep[0], keep3[b])


@pytest.mark.parametrize("soft", [None, ("linear", 0.5, 0.001)])
def test_id_moves_boxes_only(cuda, soft):
    """ID: scores, classes, counts and the kept RoIs equal the unvoted post's; only boxes move, and a top box whose voters are
    itself or exact duplicates of itself keeps its box bit for bit."""
    r, C = 300, 21
    prob, pred = stage_inputs(5 * r, r, C)
    pred[10:14, 4:8] = np.array([3000, 3000, 3040.25, 3030.5], F)   # exact duplicates in class 1, away from the others
    prob[10:14, 1] = np.array([0.97, 0.5, 0.4, 0.3], F)
    pred[20, 8:12] = np.array([5000, 5000, 5020, 5020], F)  # an isolated box in class 2
    prob[20, 2] = 0.96
    (plain,), keep0, cnt0, _, _ = run_post(prob, pred, r, C, 1, [r], 0.0, soft, 0, None)
    (voted,), keep1, cnt1, _, _ = run_post(prob, pred, r, C, 1, [r], 0.0, soft, 0, (0.8, "ID", 1.0))
    assert voted[:, 4:].tobytes() == plain[:, 4:].tobytes() and np.array_equal(keep0, keep1) and np.array_equal(cnt0, cnt1)
    assert (voted[:, :4] != plain[:, :4]).any(axis=1).sum() > 10
    for roi, c in ((10, 1), (20, 2)):
        j = int(np.where(keep1[0, c, :cnt1[0, c]] == roi)[0][0])
        row = int(cnt1[0, 1:c].sum()) + j
        assert voted[row, :4].tobytes() == pred[roi, 4 * c:4 * c + 4].tobytes() == plain[row, :4].tobytes()


@pytest.mark.parametrize("net_name,box_tol", [("res101", 5e-3), ("mobile", 4e-3)])
def test_whole_network_detect_and_detect_batch(cuda, vote_cfg, net_name, box_tol):
    from model.config import cfg
    from model.test import _detections_python_loop, _set_post_options
    C, scales, hw = 81, (4, 8, 16, 32), (600, 800)
    net, w = build(net_name, C, scales)
    blobs = [synth.synthetic_blob(hw[0], hw[1], seed) for seed in (1, 2)]
    im_info = np.array([hw[0], hw[1], 1.0], F)
    o = P.opts(anchor_scales=scales)
    st = P.test_image(net_name, w, blobs[0], im_info, C, o)
    sc_o, bx_o = P.im_detect_post(st["rois"], st["cls_prob"], st["bbox_pred"], 1.0, hw[0], hw[1])
    for soft_on in (False, True):
        for method in ("ID", "AVG"):
            cfg.TEST.SOFT_NMS.update(ENABLED=soft_on, METHOD="linear")
            vote_cfg.update(ENABLED=True, SCORING_METHOD=method, VOTE_TH=0.7)
            _set_post_options(net, 0.0, 100)
            soft, vote = net.options["soft_nms"], net.options["box_vote"]
            det, plan = net.detect(blobs[0], im_info, hw)
            scores, boxes = own_outputs(plan, 0)
            out, _ = BV.test_net_post_vote(scores, boxes, vote, 0.3, 100, soft=soft)
            assert det.shape[0] >= 100 and det.tobytes() == records_from(out).tobytes(), (soft_on, method)
            loop = _detections_python_loop(scores, boxes, C, 0.0, 100)
            assert records_from(loop).tobytes() == det.tobytes(), (soft_on, method)
            rep = compare_detections(det, BV.test_net_post_vote(sc_o, bx_o, vote, 0.3, 100, soft=soft)[0])
            print("\n[%s 600x800 %s + box voting %s vs oracle chain] %s" % (net_name, "soft-NMS" if soft_on else "greedy", method,
                                                                          fmt_report(rep)))
            assert rep["matched"] >= 0.95 * rep["n_want"] and rep["box_err"] < box_tol
            dets, plan2 = net.detect_batch(np.concatenate(blobs, axis=0), [1.0, 1.0], [hw, hw])
            for b in range(2):
                scores, boxes = own_outputs(plan2, b)
                out, _ = BV.test_net_post_vote(scores, boxes, vote, 0.3, 100, soft=soft)
                assert dets[b].tobytes() == records_from(out).tobytes(), (soft_on, method, b)


def test_features_toggles_and_tta(cuda, vote_cfg):
    from model.config import cfg
    from model.test import _run_aug, _set_post_options
    C, scales, hw = 21, (8, 16, 32), (224, 304)
    net, _ = build("res50", C, scales)
    blobs = np.concatenate([synth.synthetic_blob(hw[0], hw[1], seed) for seed in (1, 2, 3)], axis=0)
    sc, orig = [1.0, 1.25, 0.8], [(224, 304), (179, 243), (280, 380)]
    # detect_features with a re-sorting method: feats[k] = fc7 of roi_out[k], the records those of detect_batch
    vote_cfg.update(ENABLED=True, SCORING_METHOD="TEMP_AVG", VOTE_TH=0.6)
    _set_post_options(net, 0.0, 100)
    res, plan = net.detect_features(blobs, sc, orig)
    fc7 = plan.fc7.cpu().numpy()
    for b, ((det, feats, roi), want) in enumerate(zip(res, net.detect_batch(blobs, sc, orig)[0])):
        assert det.shape[0] > 0 and det.tobytes() == want.tobytes()
        assert np.array_equal(feats, fc7[b * plan.R + roi])
        prob, pred = own_outputs(plan, b)
        _, idx = BV.test_net_post_vote(prob, pred, net.options["box_vote"], 0.3, 100)
        assert np.array_equal(roi, np.concatenate(idx[1:]))
    # toggles on one plan: each launch computes what a direct call of its post computes
    for enabled, method, soft_on in ((True, "AVG", False), (False, "AVG", False), (True, "ID", True), (True, "QUASI_SUM", True),
                                     (False, "ID", True)):
        vote_cfg.update(ENABLED=enabled, SCORING_METHOD=method)
        cfg.TEST.SOFT_NMS.update(ENABLED=soft_on)
        _set_post_options(net, 0.0, 100)
        dets, plan = net.detect_batch(blobs, sc, orig)
        assert (plan.vote_box is not None) == enabled
        for b in range(3):
            prob, pred = own_outputs(plan, b)
            n = prob.shape[0]
            (direct,), _, _, _, _ = run_post(prob, pred, n, C, 1, [n], 0.0, net.options["soft_nms"], 100,
                                             net.options["box_vote"])
            assert dets[b].tobytes() == direct.tobytes(), (enabled, method, soft_on, b)
    # test-time augmentation + voting: the records are the oracle's voted post of the GPU's own union
    cfg.TEST.SCALES, cfg.USE_GPU_NMS = (288,), False
    cfg.TEST.BBOX_AUG.update(ENABLED=True, H_FLIP=True)
    net.options["use_gpu_nms"] = False
    im = cv2.blur(np.random.default_rng(4).integers(0, 256, (240, 320, 3), dtype=np.uint8), (5, 5))
    for soft_on in (False, True):
        cfg.TEST.SOFT_NMS.update(ENABLED=soft_on)
        vote_cfg.update(ENABLED=True, SCORING_METHOD="AVG", VOTE_TH=0.8)
        _set_post_options(net, 0.0, 100)
        aug = _run_aug(net, [im], detect=True)
        recs = aug.records()[0]
        n = int(aug.num_rois[0].item())
        s, x = aug.cls_prob[:n].cpu().numpy(), aug.pred_boxes[:n].cpu().numpy()
        out, _ = BV.test_net_post_vote(s, x, net.options["box_vote"], cfg.TEST.NMS, 100, soft=net.options["soft_nms"], use_gpu_nms=False)
        assert recs.shape[0] > 0 and recs.tobytes() == records_from(out).tobytes(), soft_on
    net.options["use_gpu_nms"] = True
