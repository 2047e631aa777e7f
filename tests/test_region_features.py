"""Region features and caller-box scoring, host side: argument checks that must fire before any device work, the oracle's
indexed test_net tail and Fast R-CNN box scoring, and the compiled gather / box kernels' register use."""
import os
import re
import sys

import numpy as np
import pytest

from oracle import pipeline as P

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import region_oracle as RO  # noqa: E402
from tf_faster_rcnn_b200 import engine, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = np.float32


def small_net(max_per_image=100):
    from model.config import cfg
    from nets.mobilenet_v1 import mobilenetv1
    cfg.TEST.HAS_RPN = True
    net = mobilenetv1()
    net.create_architecture("TEST", 5, tag="default", anchor_scales=(8, 16, 32), anchor_ratios=(0.5, 1, 2))
    net.load_weights(synth.make("mobile", 5, 9))
    net.options["max_per_image"] = max_per_image
    return net


def test_box_capacity_buckets():
    assert [engine.box_capacity(n) for n in (0, 1, 64, 65, 128, 129, 300, 512, 513, 1024)] == \
        [64, 64, 64, 128, 128, 256, 512, 512, 1024, 1024]
    with pytest.raises(ValueError, match="1025 boxes"):
        engine.box_capacity(1025)


def test_check_boxes_rejects_wrong_shape_dtype_and_count():
    ok = np.zeros((3, 4), F)
    assert engine.check_boxes([ok, np.zeros((0, 4), F)], 2)[0].shape == (3, 4)
    with pytest.raises(ValueError, match="shape"):
        engine.check_boxes([np.zeros((3, 5), F)], 1)
    with pytest.raises(ValueError, match="shape"):
        engine.check_boxes([np.zeros(4, F)], 1)
    with pytest.raises(TypeError, match="float32"):
        engine.check_boxes([np.zeros((3, 4), np.float64)], 1)
    with pytest.raises(ValueError, match="2 box arrays for 1 images"):
        engine.check_boxes([ok, ok], 1)


def test_public_calls_reject_bad_input_before_device_work():
    """The checks run before a plan is built, so they answer the same with and without a GPU."""
    net = small_net()
    img = np.zeros((1, 64, 96, 3), F)
    with pytest.raises(ValueError, match="1025 boxes"):
        net.score_boxes(img, [1.0], [(64, 96)], [np.zeros((1025, 4), F)])
    with pytest.raises(ValueError, match="shape"):
        net.score_boxes(img, [1.0], [(64, 96)], [np.zeros((4, 2), F)])
    with pytest.raises(TypeError, match="float32"):
        net.score_boxes(img, [1.0], [(64, 96)], [np.zeros((4, 4), np.float64)])
    from model.test import im_detect
    with pytest.raises(ValueError, match="shape"):
        im_detect(None, net, np.zeros((64, 96, 3), np.uint8), boxes=np.zeros((2, 3)))
    net0 = small_net(max_per_image=0)
    with pytest.raises(ValueError, match="max_per_image > 0"):
        net0.detect_features(img, [1.0], [(64, 96)])


def test_oracle_indexed_test_net_post_matches_test_net_post():
    rng = np.random.default_rng(7)
    r, C = 300, 21
    xy = rng.uniform(0, 300, (r, C, 2)); wh = rng.uniform(8, 120, (r, C, 2))
    boxes = np.concatenate([xy, xy + wh], axis=2).reshape(r, 4 * C).astype(F)
    scores = rng.dirichlet(np.ones(C), r).astype(F)
    for mpi in (100, 0):
        o = P.opts(max_per_image=mpi)
        want = P.test_net_post(scores, boxes, o)
        got, idx = RO.test_net_post_indexed(scores, boxes, o)
        assert sum(d.shape[0] for d in got) > (100 if mpi == 0 else 50)
        for j in range(C):
            assert np.array_equal(got[j], want[j]), j
            assert idx[j].shape[0] == got[j].shape[0]
            if j:
                assert np.array_equal(got[j][:, :4], boxes[idx[j], 4 * j:4 * j + 4])
                assert np.array_equal(got[j][:, 4], scores[idx[j], j])


def test_oracle_score_boxes_reproduces_test_image_on_its_own_rois():
    hw, C = (96, 128), 5
    w = synth.make("mobile", C, 9)
    blob = synth.synthetic_blob(*hw)
    o = P.opts(rpn_post_nms_top_n=50)
    st = P.test_image("mobile", w, blob, np.array([hw[0], hw[1], 1.0], F), C, o)
    sb = RO.score_boxes("mobile", w, blob, st["rois"][:, 1:5], 1.0, hw, o)
    assert np.array_equal(sb["rois"], st["rois"])
    for k in ("fc7", "cls_prob", "bbox_pred"):
        assert np.array_equal(sb[k], st[k]), k
    want = P.im_detect_post(st["rois"], st["cls_prob"], st["bbox_pred"], 1.0, hw[0], hw[1])
    assert np.array_equal(sb["pred_boxes"], want[1])


INSTANTIATIONS = {"conv_gemm_kernel": 6}      # 2 block_n x 3 arithmetic modes; every other kernel: 1


@pytest.mark.parametrize("obj,kernel", [("nms", "detect_features_kernel"), ("simt_ops", "boxes_to_rois_kernel"),
                                        ("conv_gemm", "conv_gemm_kernel")])
def test_new_kernels_do_not_spill(obj, kernel):
    """ptxas -v output written by the build (one log per object), for every instantiation of the kernel."""
    log = open(os.path.join(ROOT, "tf_faster_rcnn_b200", "csrc", "_obj", obj + ".o.log")).read()
    found = re.findall(r"Function properties for \S*%s\S*\s*\n([^\n]*)" % kernel, log)
    assert len(found) == INSTANTIATIONS.get(kernel, 1), "ptxas reports for %s: %d" % (kernel, len(found))
    for line in found:
        assert "0 bytes spill stores, 0 bytes spill loads" in line, line
