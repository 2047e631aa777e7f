"""Test-time augmentation (TEST.BBOX_AUG) on the GPU: frcnn_aug_union against the numpy model bit for bit, the mirrored
preprocess, one view = detect, the flip slot, whole networks against the oracle's post on the GPU's own per-view outputs (bit for
bit) and against the oracle alone (matched and reported), batched TTA over mixed sizes, the Python loop, the alternating record
buffers, an LRU eviction between calls, and the 'top'-mode capacity check."""
import os
import sys

import cv2
import numpy as np
import pytest
import torch

from oracle import pipeline as P

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import aug_oracle as AO  # noqa: E402
from test_bbox_aug import random_views  # noqa: E402
from test_e2e_gpu import compare_detections, fmt_report  # noqa: E402
from test_soft_nms_gpu import build, records_from  # noqa: E402
from tf_faster_rcnn_b200 import ops

pytestmark = pytest.mark.gpu
F = np.float32


@pytest.fixture(scope="module", autouse=True)
def _restore_network_registry():
    """The networks built here leave the process-wide registry afterwards (Saver.restore walks it)."""
    from nets import network
    before = list(network._REGISTRY)
    yield
    network._REGISTRY[:] = before


@pytest.fixture
def aug_cfg():
    from model.config import cfg
    saved = (dict(cfg.TEST.BBOX_AUG), dict(cfg.TEST.SOFT_NMS), tuple(cfg.TEST.SCALES), cfg.TEST.MAX_SIZE, cfg.USE_GPU_NMS, cfg.TEST.MODE)
    yield cfg.TEST.BBOX_AUG
    cfg.TEST.BBOX_AUG.update(saved[0])
    cfg.TEST.SOFT_NMS.update(saved[1])
    cfg.TEST.SCALES, cfg.TEST.MAX_SIZE, cfg.USE_GPU_NMS, cfg.TEST.MODE = saved[2:]


def image(h, w, seed):
    return cv2.blur(np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8), (5, 5))


def own_views(aug, b):
    """The GPU's own per-view im_detect outputs (valid rows) of image b after an augmented launch."""
    sc, bx = [], []
    for v, (h, w, _) in enumerate(aug.views):
        p = aug.subs[(h, w)]
        k = aug.view_slot[v] * aug.batch + b
        n, R = int(p.num_rois[k].item()), p.R
        sc.append(p.cls_prob[k * R:k * R + n].cpu().numpy())
        bx.append(p.pred_boxes[k * R:k * R + n].cpu().numpy())
    return sc, bx


def oracle_records_on_own_outputs(aug, b, orig_w, o, soft=None):
    sc, bx = own_views(aug, b)
    s, x = AO.union(sc, bx, [v[2] for v in aug.views], orig_w)
    return records_from(AO.post(s, x, o, soft)), s, x


@pytest.mark.parametrize("nv", [1, 2, 5, 16])
@pytest.mark.parametrize("C", [21, 81])
def test_union_kernel_matches_model(cuda, nv, C):
    rng = np.random.default_rng(100 * nv + C)
    B = 3
    probs, boxes, counts, flips, rows = random_views(rng, nv, B, C, max_rows=300)
    orig_w = [800, 500, 1333]
    dev = [(torch.from_numpy(p).cuda(), torch.from_numpy(q).cuda(), torch.from_numpy(c).cuda()) for p, q, c in zip(probs, boxes, counts)]
    meta = torch.tensor([[1.0, 600.0, float(w)] for w in orig_w], dtype=torch.float32).cuda()
    ru = sum(p.shape[1] for p in probs)
    up = torch.full((B * ru, C), float("nan"), device="cuda"); ub = torch.full((B * ru, 4 * C), float("nan"), device="cuda")
    num = torch.full((B,), -7, dtype=torch.int32, device="cuda")
    ops.aug_union([(a.data_ptr(), q.data_ptr(), c.data_ptr(), a.shape[1], f) for (a, q, c), f in zip(dev, flips)], C, meta.data_ptr(), up,
                  ub, num)
    torch.cuda.synchronize()
    wp, wb, wn = AO.union_model(probs, boxes, counts, flips, orig_w)
    assert np.array_equal(num.cpu().numpy(), wn)
    assert up.cpu().numpy().tobytes() == wp.reshape(B * ru, C).tobytes()
    assert ub.cpu().numpy().tobytes() == wb.reshape(B * ru, 4 * C).tobytes()


@pytest.mark.parametrize("hw", [(375, 500), (601, 799), (333, 1200)])
def test_mirrored_preprocess(cuda, hw):
    """frcnn_preprocess_hflip(im) == frcnn_preprocess(im[:, ::-1]) bit for bit, and within the preprocess tolerance of
    cv2.resize of the mirrored image."""
    from model.config import cfg
    from model.test import aug_view_blob, blob_geometry
    im = np.random.default_rng(hw[1]).integers(0, 256, hw + (3,), dtype=np.uint8)
    H, W, f = blob_geometry(im.shape)
    means = np.asarray(cfg.PIXEL_MEANS, dtype=np.float64).ravel()
    a = torch.empty((1, H, W, 3), device="cuda"); b = torch.empty_like(a)
    ops.preprocess(torch.from_numpy(im).cuda(), means, f, f, a, hflip=True)
    ops.preprocess(torch.from_numpy(np.ascontiguousarray(im[:, ::-1])).cuda(), means, f, f, b)
    want, g = aug_view_blob(im, cfg.TEST.SCALES[0], cfg.TEST.MAX_SIZE, True)
    assert g == f and want.shape == (1, H, W, 3)
    assert a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes()
    err = float(np.abs(a.cpu().numpy() - want).max())
    print("\n[preprocess hflip %dx%d -> %dx%d] max abs diff vs OpenCV of the mirrored image %.2e" % (hw[0], hw[1], H, W, err))
    assert err < 1e-4


@pytest.fixture(scope="module")
def res50():
    net, w = build("res50", 21, (8, 16, 32))
    net.options["use_gpu_nms"] = False          # the cpu_nms predicate of the oracle's test_net_post
    return net, w


def small(aug_cfg, **update):
    """288-px base view: ResNet-50 tests at a small size; the Python loop's nms() with the cpu_nms predicate too."""
    from model.config import cfg
    cfg.TEST.SCALES = (288,)
    cfg.USE_GPU_NMS = False
    aug_cfg.update(ENABLED=True, **update)


def test_one_view_equals_detect(cuda, res50, aug_cfg):
    from model.test import detect_image, _run_aug
    net, _ = res50
    im = image(240, 320, 1)
    small(aug_cfg)
    for soft in (False, True):
        from model.config import cfg
        cfg.TEST.SOFT_NMS.ENABLED = soft
        aug_cfg.ENABLED = False
        want = detect_image(net, im, 0.0, 100)
        aug_cfg.ENABLED = True
        got = detect_image(net, im, 0.0, 100)
        assert records_from(got).shape[0] > 0 and records_from(got).tobytes() == records_from(want).tobytes(), soft
    aug = _run_aug(net, [im], detect=True)
    assert len(aug.views) == 1 and aug.R == aug.subs[aug.views[0][:2]].R


def test_flip_slot_equals_plain_detect(cuda, res50, aug_cfg):
    """Identity and flip share one batch-2 plan (slots 0 and 1); the flip slot's outputs are those of a plain detect_batch of
    [base blob, blob of the mirrored image] on that plan, bit for bit; the records are the oracle's post of the union."""
    from model.test import _run_aug, _set_post_options, aug_view_blob
    from model.config import cfg
    net, _ = res50
    im = image(240, 320, 2)
    small(aug_cfg, H_FLIP=True)
    _set_post_options(net, 0.0, 100)
    aug = _run_aug(net, [im], detect=True)
    assert [v[2] for v in aug.views] == [True, False] and aug.view_slot == [1, 0] and len(aug.subs) == 1
    plan = aug.subs[aug.views[0][:2]]
    assert plan.batch == 2
    R = plan.R
    got = [(plan.cls_prob[k * R:(k + 1) * R].cpu().numpy(), plan.pred_boxes[k * R:(k + 1) * R].cpu().numpy(),
            int(plan.num_rois[k].item())) for k in range(2)]
    recs = aug.records()[0]
    want, _, _ = oracle_records_on_own_outputs(aug, 0, im.shape[1], P.opts(use_gpu_nms=False, nms_thresh=cfg.TEST.NMS))
    base, f = aug_view_blob(im, 288, 1000, False)
    flip, g = aug_view_blob(im, 288, 1000, True)
    dets, aug2 = net.detect_aug([flip, base], [[g], [f]], [im.shape[:2]], [True, False])    # the public entry, host blobs
    assert aug2 is aug and dets[0].tobytes() == recs.tobytes()
    net.detect_batch(np.concatenate([base, flip]), [f, g], [im.shape[:2]] * 2)
    for k in range(2):
        assert got[k][2] == int(plan.num_rois[k].item())
        assert got[k][0].tobytes() == plan.cls_prob[k * R:(k + 1) * R].cpu().numpy().tobytes()
        assert got[k][1].tobytes() == plan.pred_boxes[k * R:(k + 1) * R].cpu().numpy().tobytes()
    assert recs.shape[0] > 0 and recs.tobytes() == want.tobytes()


@pytest.mark.parametrize("net_name,extra,box_tol", [("res101", (), 5e-3), ("mobile", (480,), 4e-3)])
def test_whole_network_against_oracles(cuda, aug_cfg, net_name, extra, box_tol):
    """600x800, H_FLIP (MobileNet also an extra 480 scale), greedy and Soft-NMS: records == the oracle's post on the numpy union
    of the GPU's own per-view outputs, bit for bit; against the oracle alone, detections are matched and reported."""
    from model.config import cfg
    from model.test import _run_aug, _set_post_options
    C, scales = 81, (4, 8, 16, 32)
    net, w = build(net_name, C, scales)
    net.options["use_gpu_nms"] = False
    cfg.USE_GPU_NMS = False
    aug_cfg.update(ENABLED=True, H_FLIP=True, SCALES=extra)
    im = image(600, 800, 3)
    o = P.opts(anchor_scales=scales, use_gpu_nms=False)
    view_list = AO.views(True, extra, aug_cfg.MAX_SIZE)
    s_or, b_or = AO.im_detect_aug(net_name, w, im, C, o, view_list)
    for soft in (None, ("linear", 0.5, 0.001)):
        cfg.TEST.SOFT_NMS.update(ENABLED=soft is not None, METHOD="linear")
        _set_post_options(net, 0.0, 100)
        aug = _run_aug(net, [im], detect=True)
        assert len(aug.views) == len(view_list) and aug.R == 300 * len(view_list)
        det = aug.records()[0]
        want, s, x = oracle_records_on_own_outputs(aug, 0, im.shape[1], o, soft)
        assert det.shape[0] >= 100 and det.tobytes() == want.tobytes(), soft
        r = int(aug.num_rois[0].item())
        assert r == s.shape[0] and aug.cls_prob[:r].cpu().numpy().tobytes() == s.tobytes()
        assert aug.pred_boxes[:r].cpu().numpy().tobytes() == x.tobytes()
        rep = compare_detections(det, AO.post(s_or, b_or, o, soft))
        print("\n[%s 600x800 TTA %d views, %s, vs the oracle alone] union rows gpu %d oracle %d | %s"
              % (net_name, len(view_list), soft[0] if soft else "greedy", r, s_or.shape[0], fmt_report(rep)))
        assert rep["matched"] >= 0.9 * rep["n_want"] and rep["score_err"] < 1e-4 and rep["box_err"] < box_tol


def test_detect_images_mixed_sizes(cuda, res50, aug_cfg):
    """Batched TTA groups consecutive images with equal view-shape tuples.  Every image's records are the oracle's post of the
    union of that launch's own per-view outputs, bit for bit; a single-image group equals per-image TTA bit for bit.  Images of a
    multi-image group are matched against per-image TTA: the conv plans of batch 2 and batch 1 may split K differently, so the
    head outputs can differ in the last bits."""
    from model.test import detect_images, detect_image, _aug_key, _run_aug
    from model.config import cfg
    net, _ = res50
    small(aug_cfg, H_FLIP=True, SCALES=(224,), MAX_SIZE=1000)
    ims = [image(240, 320, 4), image(240, 320, 5), image(200, 320, 6), image(240, 320, 7)]
    keys = [_aug_key(im) for im in ims]
    assert keys[0] == keys[1] == keys[3] != keys[2]
    got = detect_images(net, ims, 0.0, 100, batch_size=2)
    single = [detect_image(net, im, 0.0, 100) for im in ims]
    o = P.opts(use_gpu_nms=False, nms_thresh=cfg.TEST.NMS)
    for group in ([0, 1], [2], [3]):
        aug = _run_aug(net, [ims[i] for i in group], detect=True)
        for b, i in enumerate(group):
            want, _, _ = oracle_records_on_own_outputs(aug, b, ims[i].shape[1], o)
            assert records_from(got[i]).tobytes() == want.tobytes(), i
            if len(group) == 1:
                assert records_from(got[i]).tobytes() == records_from(single[i]).tobytes(), i
            else:
                rep = compare_detections(records_from(got[i]), single[i])
                print("\n[batched TTA image %d vs per-image TTA] %s" % (i, fmt_report(rep)))
                assert rep["matched"] >= 0.95 * rep["n_want"] and rep["score_err"] < 1e-4


def test_python_loop_equals_fused(cuda, res50, aug_cfg):
    from model.config import cfg
    from model.test import im_detect, detect_image, _detections_python_loop
    net, _ = res50
    small(aug_cfg, H_FLIP=True, SCALES=(224,))
    cfg.USE_GPU_NMS = False
    net.options["use_gpu_nms"] = False
    im = image(240, 320, 8)
    for soft in (False, True):
        cfg.TEST.SOFT_NMS.ENABLED = soft
        scores, boxes = im_detect(None, net, im)
        assert scores.shape[0] > 300 and boxes.shape == (scores.shape[0], 4 * 21)
        fused = detect_image(net, im, 0.0, 100)
        loop = _detections_python_loop(scores, boxes, 21, 0.0, 100)
        assert records_from(loop).tobytes() == records_from(fused).tobytes(), soft


def test_im_detect_with_device_preprocess(cuda, res50, aug_cfg):
    """DEVICE_PREPROCESS fills each view's image slice with the preprocess kernels (mirrored for flipped views): the union has
    the host path's size and differs only by the preprocess tolerance carried through the network."""
    import model.test as MT
    net, _ = res50
    small(aug_cfg, H_FLIP=True, SCALES=(224,))
    im = image(240, 320, 14)
    s0, b0 = MT.im_detect(None, net, im)
    MT.DEVICE_PREPROCESS = True
    try:
        s1, b1 = MT.im_detect(None, net, im)
    finally:
        MT.DEVICE_PREPROCESS = False
    print("\n[TTA im_detect, device vs host preprocess] union rows %d / %d, scores %.2e, boxes %.2e px"
          % (s0.shape[0], s1.shape[0], np.abs(s0 - s1).max() if s0.shape == s1.shape else -1,
             np.abs(b0 - b1).max() if b0.shape == b1.shape else -1))
    assert s0.shape == s1.shape and np.abs(s0 - s1).max() < 1e-3 and np.abs(b0 - b1).max() < 0.5


def test_detect_record_alternates_buffers(cuda, res50, aug_cfg):
    from model.test import _detect_record, detect_image
    net, _ = res50
    small(aug_cfg, H_FLIP=True)
    ims = [image(240, 320, 9), image(240, 320, 10), image(240, 320, 11)]
    recs = [_detect_record(net, im, 0.0, 100) for im in ims]
    assert recs[0].data_ptr() != recs[1].data_ptr() and recs[2].data_ptr() == recs[0].data_ptr()
    torch.cuda.synchronize()
    from tf_faster_rcnn_b200 import engine
    aug = list(net._aug_plans.values())[-1]                     # the plan of the last call
    assert aug.double_buffer and sorted(r.data_ptr() for r in recs[:2]) == sorted(r.data_ptr() for r in aug.recs)
    host = [r.cpu() for r in recs[1:]]                          # recs[1] still holds image 1 after image 2 ran
    for k in (1, 2):
        det = engine.split_host_records(host[k - 1][None], aug.max_det)[0]
        assert det.shape[0] > 0 and det.tobytes() == records_from(detect_image(net, ims[k], 0.0, 100)).tobytes()


def test_lru_eviction_between_calls(cuda, res50, aug_cfg):
    from model.test import detect_image, _run_aug
    net, _ = res50
    small(aug_cfg, H_FLIP=True)
    im = image(240, 320, 12)
    first = records_from(detect_image(net, im, 0.0, 100))
    aug = _run_aug(net, [im], detect=True)
    old = dict(aug.subs)
    saved = net.MAX_PLANS
    try:
        net.MAX_PLANS = 2
        net.plan_for(160, 224); net.plan_for(224, 160)                  # evicts the augmented call's batch-2 plan
        assert all(k[:3] != (288, 384, 2) for k in net._plans)
        again = records_from(detect_image(net, im, 0.0, 100))
    finally:
        net.MAX_PLANS = saved
    assert aug.subs[(288, 384)] is not old[(288, 384)]
    assert again.shape[0] > 0 and again.tobytes() == first.tobytes()


def test_top_mode_two_views_raises_before_device_work(cuda, aug_cfg):
    from model.config import cfg
    from model.test import detect_image
    cfg.TEST.MODE = "top"
    net, _ = build("mobile", 21, (8, 16, 32))
    aug_cfg.update(ENABLED=True, H_FLIP=True)
    with pytest.raises(ValueError, match="8192"):
        detect_image(net, image(240, 320, 13), 0.0, 100)
    assert net._plans == {} and net._aug_plans == {}
