"""Detectors with more than 1024 classes on the GPU, bit for bit against the oracles: the four post entries (greedy with both
predicates, Soft-NMS, voting behind each) and detect_features at 1025 to 4096 classes, the class boundary at 1024, the bottom-up
regions' overlap-mask path, and a synthetic 1601-class, 12-anchor ResNet-101 (the bottom-up-attention Visual Genome layout).
Outputs sit between sentinel guard bands and inputs are checked unchanged (the helpers of test_post_edges_gpu / test_regions_gpu)."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import post_ref64 as R  # noqa: E402
import regions_oracle as RO  # noqa: E402
import stage_ref64 as S  # noqa: E402
from test_post_edges_gpu import SOFTS, check_post, dev, guarded_int, post, same_bits, unchanged  # noqa: E402
from test_regions_gpu import _release_networks, build, check_net, guarded, make_batch  # noqa: E402,F401
from oracle import pipeline as P  # noqa: E402
from tf_faster_rcnn_b200 import engine, ops  # noqa: E402

pytestmark = pytest.mark.gpu
F = np.float32
G = 64


def greedy_post(prob, pred, r, C, nroi, gpu_nms, mpi, max_det):
    """frcnn_detect_post on guard-banded outputs, inputs checked unchanged, each image against oracle.pipeline.test_net_post on its
    valid rows -> (records [B, max_det, 6], ndet [B], keep [B, C, r], keep_cnt [B, C])."""
    B = len(nroi)
    cp, pb, num = dev(prob), dev(pred), dev(np.asarray(nroi, np.int32))
    gd, det = S.guarded_out((B, max_det, 6))
    gn, ndet = guarded_int((B,))
    gk, keep = guarded_int((B, C, r))
    gc, cnt = guarded_int((B, C))
    gs, ks = S.guarded_out((B, C, r))
    t32, flags = engine.nms_threshold(0.3, gpu_nms)
    ops.detect_post(cp, pb, num, C, 0.0, t32, flags, mpi, det, ndet, keep, cnt, ks, ops.detect_post_workspace(r, C, B), B)
    torch.cuda.synchronize()
    for g, t, what in ((gd, det, "det"), (gn, ndet, "ndet"), (gk, keep, "keep"), (gc, cnt, "keep_cnt"), (gs, ks, "keep_score")):
        S.check_guarded(g, t.numel(), what)
    unchanged(cp, prob, "cls_prob"); unchanged(pb, pred, "pred_boxes"); unchanged(num, np.asarray(nroi, np.int32), "num_rois")
    det, nd, cnt_h = det.cpu().numpy(), ndet.cpu().numpy(), cnt.cpu().numpy()
    for b, n in enumerate(nroi):
        n = min(max(n, 0), r)
        want = P.test_net_post(prob[b * r:b * r + n], pred[b * r:b * r + n], P.opts(nms_thresh=0.3, use_gpu_nms=gpu_nms, max_per_image=mpi))
        S.check_records(det[b], int(nd[b]), cnt_h[b], want, max_det, "C %d image %d" % (C, b))
    return det, nd, keep.cpu().numpy(), cnt_h


def case(rng, r, C, B=3):
    prob = S.quantised_probs(rng, B * r, C, weights=S.SPARSE_TOP)
    pred = np.vstack([S.clustered_pred(rng, r, C) for _ in range(B)])
    return prob, pred


POSTS = [(1025, 300), (1025, 1000), (1204, 300), (1204, 1000), (1601, 300), (1601, 1000), (1601, 5000), (4096, 300), (4096, 1000)]


@pytest.mark.parametrize("C,r", POSTS)
def test_posts_many_classes(cuda, C, r):
    """Batch 3 with num_rois 0, 137 and r: greedy with both predicates, Soft-NMS, and voting behind greedy and behind Soft-NMS."""
    rng = np.random.default_rng(C + r)
    nroi = [0, 137, r]
    prob, pred = case(rng, r, C)
    for gpu_nms in (True, False):
        _, nd, _, _ = greedy_post(prob, pred, r, C, nroi, gpu_nms, 100, 256)
        assert nd[0] == 0 and nd[2] >= 100
    if r > 1000:
        return                                       # TEST.MODE 'top': the greedy post (the oracles of the others take minutes here)
    for soft, vote in ((SOFTS[1], None), (None, (0.8, "AVG", 1.0)), (SOFTS[0], (0.6, "IOU_AVG", 1.0))):
        res = post(prob, pred, r, C, nroi, soft, vote, 100, 256)
        counts = check_post(res, prob, pred, r, C, nroi, soft, vote, 100, 256)
        assert counts[0] == 0 and counts[2] >= 100


def test_post_ties_at_the_cap_across_1024(cuda):
    """60 records above the 100th score and 80 tied at it, spread over classes below and above 1024 (all 140 kept); then 300 tied:
    ndet 360 reported, nothing stored past max_det 256; max_per_image 0 keeps every record."""
    rng = np.random.default_rng(1601)
    r, C = 300, 1601
    prob, pred = S.cap_tie_probs(rng, r, C, 60, 80), S.grid_pred(r, C)
    tied = np.argwhere(prob == F(0.5))[:, 1]
    assert (tied < 1024).any() and (tied >= 1024).any()
    _, nd, _, _ = greedy_post(prob, pred, r, C, [r], True, 100, 256)
    assert nd.tolist() == [140]
    prob2 = S.cap_tie_probs(rng, r, C, 60, 300)
    _, nd, _, _ = greedy_post(prob2, pred, r, C, [r], False, 100, 256)
    assert nd.tolist() == [360]
    _, nd, _, _ = greedy_post(prob2, pred, r, C, [r], True, 0, r * (C - 1))
    assert nd.tolist() == [360]
    res = post(prob2, pred, r, C, [r], SOFTS[2], None, 0, r * (C - 1))
    check_post(res, prob2, pred, r, C, [r], SOFTS[2], None, 0, r * (C - 1))


def test_class_boundary_1025_equals_1024(cuda):
    """A 1025-class input whose last class scores 0 gives the records of the same input without that class."""
    rng = np.random.default_rng(1024)
    r = 300
    prob, pred = case(rng, r, 1024, B=2)
    prob1 = np.hstack([prob, np.zeros((prob.shape[0], 1), F)])
    pred1 = np.hstack([pred, pred[:, -4:]])
    for gpu_nms in (True, False):
        a = greedy_post(prob, pred, r, 1024, [r, 200], gpu_nms, 100, 256)
        b = greedy_post(prob1, pred1, r, 1025, [r, 200], gpu_nms, 100, 256)
        assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes()


@pytest.mark.parametrize("C", [1601, 4096])
def test_detect_features_many_classes(cuda, C):
    rng = np.random.default_rng(C)
    keep, cnt = R.features_case(rng, C)
    B, _, r = keep.shape
    fc7 = rng.standard_normal((B * r, 64)).astype(F)
    kd, cd, fd = dev(keep), dev(cnt), dev(fc7)
    for max_det in (7, 100, 256):
        gf, feat = S.guarded_out((B, max_det, 64))
        gr, roi = guarded_int((B, max_det))
        ops.detect_features(kd, cd, fd, C, feat, roi)
        torch.cuda.synchronize()
        S.check_guarded(gf, feat.numel(), "features"); S.check_guarded(gr, roi.numel(), "roi_out")
        wf, wr = R.features_ref(keep, cnt, fc7, max_det)
        assert np.array_equal(roi.cpu().numpy(), wr), max_det
        same_bits(feat.cpu().numpy(), wf, "features max_det %d" % max_det)
    unchanged(kd, keep, "keep"); unchanged(cd, cnt, "keep_cnt"); unchanged(fd, fc7, "fc7")


# ---- bottom-up regions, the overlap-mask path ---------------------------------------------------------------------------------
def run_regions(probs, rois, fc7, nrois, scales, gpu_pred, conf, mn, mx):
    """frcnn_detect_regions at C > 1024 (no keep lists, one box per row, the mask workspace) -> per image dicts; guards, padding
    rows and unchanged inputs checked."""
    B = len(nrois)
    Rr, C = probs.shape[0] // B, probs.shape[1]
    assert C > ops.REGIONS_CLASS_NMS_MAX
    fdim = fc7.shape[1]
    ins = dict(cls_prob=dev(probs), rois=dev(rois), num_rois=dev(np.asarray(nrois, np.int32)),
               im_meta=dev(np.array([[float(F(s)), 600.0, 800.0] for s in scales], F)), fc7=dev(fc7))
    before = {k: v.clone() for k, v in ins.items()}
    M = min(mx, Rr)
    bufs = dict(roi_box=guarded(ops.regions_box_shape(B * Rr, C), torch.float32), key=guarded((B * Rr,), torch.int64),
                boxes=guarded((B, M, 4), torch.float32), features=guarded((B, M, fdim), torch.float32),
                conf=guarded((B, M), torch.float32), classes=guarded((B, M), torch.int32), roi_index=guarded((B, M), torch.int32),
                count=guarded((B,), torch.int32))
    guards = {k: (b[:G].clone(), b[-G:].clone()) for k, (b, _) in bufs.items()}
    ws = ops.detect_regions_workspace(Rr, C, B)
    thr, flags = engine.nms_threshold(0.3, gpu_pred)
    t32, mn, mx = engine.region_args(conf, mn, mx)
    out = {k: v for k, (_, v) in bufs.items() if k not in ("roi_box", "key")}
    ops.detect_regions(ins["cls_prob"], ins["rois"], ins["num_rois"], ins["im_meta"], ins["fc7"], C, thr, flags, t32, mn, mx, None, None,
                       None, ws, bufs["roi_box"][1], bufs["key"][1], out, batch=B)
    torch.cuda.synchronize()
    for k, (b, _) in bufs.items():
        assert torch.equal(b[:G], guards[k][0]) and torch.equal(b[-G:], guards[k][1]), "guard band of %s overwritten" % k
    for k in ins:
        assert torch.equal(ins[k], before[k]), "input %s changed" % k
    host = {k: v.cpu().numpy() for k, v in out.items()}
    res = []
    for b in range(B):
        n = int(host["count"][b])
        assert 0 <= n <= M
        assert (host["roi_index"][b, n:] == -1).all() and not host["boxes"][b, n:].any() and not host["conf"][b, n:].any()
        assert not host["classes"][b, n:].any() and not host["features"][b, n:].any()
        res.append({k: host[k][b, :n] for k in engine.REGION_FIELDS})
    return res


def check_regions(probs, rois, fc7, nrois, scales, gpu_pred, conf, mn, mx):
    B = len(nrois)
    Rr = probs.shape[0] // B
    res = run_regions(probs, rois, fc7, nrois, scales, gpu_pred, conf, mn, mx)
    for b in range(B):
        s = slice(b * Rr, (b + 1) * Rr)
        RO.compare(res[b], RO.image_regions(probs[s], rois[s], nrois[b], F(scales[b]), 0.3, gpu_pred, conf, mn, mx, fc7=fc7[s]))
    return res


@pytest.mark.parametrize("C,Rr,B", [(1025, 300, 2), (1601, 300, 3), (4096, 300, 1), (1025, 1000, 2), (1601, 1000, 1), (4096, 1000, 1),
                                    (1025, 5000, 1)])
def test_regions_mask_path(cuda, C, Rr, B):
    rng = np.random.default_rng(C + Rr + B)
    nrois = [Rr - 17, 0, 5][:B] if B > 1 else [Rr - 3]
    probs, rois, fc7 = make_batch(rng, B, Rr, C, nrois)
    scales = [1.6, 0.8, 1.25][:B]
    for gpu_pred in (True, False):
        for conf, mn, mx in ((0.2, 10, 100), (0.0, 10, 100), (0.2, 36, 36))[:1 if Rr > 1000 else 3]:
            res = check_regions(probs, rois, fc7, nrois, scales, gpu_pred, conf, mn, mx)
            assert res[0]["roi_index"].shape[0] > 0


def test_regions_mask_path_edges(cuda):
    """test_regions_gpu's stage edges at 1601 classes, plus a best class above 1024 tied with one below (the lower wins)."""
    rng = np.random.default_rng(11)
    Rr, C = 300, 1601
    probs, rois, fc7 = make_batch(rng, 1, Rr, C, [Rr], spread=6000.0, size=(10, 20))   # isolated boxes
    probs *= F(0.45)
    half = F(0.5)
    probs[3, 5], probs[4, 1300], probs[5, 7] = half, np.nextafter(half, F(0)), np.nextafter(half, F(1))
    probs[11], probs[12], probs[40] = probs[10], probs[10], probs[10]
    rois[21, 1:] = rois[20, 1:]
    probs[21] = probs[20]
    rois[31, 1:] = rois[30, 1:]
    probs[30] = probs[31] * F(0.5)
    probs[50, 900], probs[50, 1500] = F(0.48), F(0.48)
    for gpu_pred in (True, False):
        res = check_regions(probs, rois, fc7, [Rr], [1.0], gpu_pred, 0.5, 0, 100)
        assert res[0]["roi_index"].tolist() == [3, 5]
        res = check_regions(probs, rois, fc7, [Rr], [1.0], gpu_pred, 0.5, 10, 100)
        idx = res[0]["roi_index"].tolist()
        assert idx[:2] == [5, 3] and len(idx) == 10
        res = check_regions(probs, rois, fc7, [Rr], [1.0], gpu_pred, 0.3, Rr, Rr)
        got = {i: (c, k) for i, c, k in zip(res[0]["roi_index"].tolist(), res[0]["conf"].tolist(), res[0]["classes"].tolist())}
        assert got[21][0] == 0.0 and got[30][0] == 0.0 and got[20][0] > 0 and got[31][0] > 0
        assert got[50][1] == 900 and got[4][1] == 1300
    for nr in (0, 4, 9):
        res = check_regions(probs, rois, fc7, [nr], [1.0], True, 0.2, 10, 100)
        assert res[0]["roi_index"].shape[0] == nr


# ---- network level: the bottom-up-attention layout (1601 classes, 12 anchors) -------------------------------------------------
def test_network_resnet101_1601_classes(cuda):
    net = build("res101", 1601, (4, 8, 16, 32))
    assert net._num_anchors == 12
    hw = (600, 800)
    blobs = np.concatenate([synth_blob(hw, s) for s in (1, 2)], axis=0)
    scales, orig = [1.0, 1.25], [(600, 800), (480, 640)]
    recs, plan = net.detect_batch(blobs, scales, orig)
    B, Rr = plan.batch, plan.R
    probs, pred = plan.cls_prob.cpu().numpy(), plan.pred_boxes.cpu().numpy()
    nroi = plan.num_rois.cpu().numpy()
    o = net.options
    want = []
    for b in range(B):
        s = slice(b * Rr, b * Rr + int(nroi[b]))
        per_class = P.test_net_post(probs[s], pred[s], P.opts(nms_thresh=o["nms_thresh"], use_gpu_nms=o["use_gpu_nms"], max_per_image=100))
        want.append(S.flat_records(per_class))
        S.check_exact(recs[b], want[b], "image %d records" % b)
    assert recs[0].shape[0] > 0
    feats, _ = net.detect_features(blobs, scales, orig)
    fc7 = plan.fc7.cpu().numpy()
    for b, (det, f, ri) in enumerate(feats):
        S.check_exact(det, want[b], "detect_features image %d" % b)
        assert f.tobytes() == fc7[b * Rr + ri.astype(np.int64)].tobytes()
    det1, plan1 = net.detect(blobs[:1], np.array([hw[0], hw[1], 1.0], F), hw)
    p1, x1 = plan1.cls_prob.cpu().numpy(), plan1.pred_boxes.cpu().numpy()
    n1 = int(plan1.num_rois.cpu().numpy()[0])
    S.check_exact(det1, S.flat_records(P.test_net_post(p1[:n1], x1[:n1], P.opts(nms_thresh=o["nms_thresh"],
                                                                                 use_gpu_nms=o["use_gpu_nms"], max_per_image=100))), "detect")
    res, plan2 = net.detect_regions(blobs, scales, orig)
    assert plan2 is plan and plan.reg_box.shape == (B * Rr, 4) and plan.reg_ws is not plan.post_ws
    check_net(net, plan, res, 0.2, 10, 100)


def synth_blob(hw, seed):
    from tf_faster_rcnn_b200 import synth
    return synth.synthetic_blob(hw[0], hw[1], seed)
