"""Detectors with up to 4096 classes, without a GPU: the class-count refusals of the Python layer and of every C entry that takes C,
the overlap-mask walk of frcnn_detect_regions (C > 1024) restated in numpy against tests/regions_oracle.py, plausible mistakes the
comparison catches, and the ptxas report of the new and changed kernels."""
import ctypes
import os
import re
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
import regions_oracle as RO  # noqa: E402
from oracle import nms as NMS  # noqa: E402

F = np.float32
ERR_ARG, ERR_CAPACITY = -2, -5


# ---- refusals -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C", [4097, 1, 0, -3, 2.0, "81", True])
def test_create_architecture_refuses_class_count(C):
    from nets.resnet_v1 import resnetv1
    net = resnetv1(num_layers=50)
    with pytest.raises(ValueError, match="num_classes"):
        net.create_architecture("TEST", C, tag="default")


def test_create_architecture_accepts_4096_classes():
    from nets.resnet_v1 import resnetv1
    net = resnetv1(num_layers=101)
    net.create_architecture("TEST", np.int64(4096), tag="default", anchor_scales=(4, 8, 16, 32))
    assert net.num_classes == 4096 and type(net.num_classes) is int and net._num_anchors == 12


def _entries():
    """name -> call(r, batch, C) of every C entry that takes a class count, with non-null pointers that are never dereferenced."""
    from tf_faster_rcnn_b200 import _native as N
    L, p = N.lib(), ctypes.c_void_p(4096)
    return {
        "detect_post": lambda r, b, C: L.frcnn_detect_post(p, p, p, r, b, C, 0.05, 0.3, 1, 100, 256, p, p, 0, p, p, p, p, 1 << 40, None),
        "detect_post_vote": lambda r, b, C: L.frcnn_detect_post_vote(p, p, p, r, b, C, 0.05, 0.3, 1, 100, 256, p, p, 0, p, p, p, p, 1 << 40,
                                                                     0.8, 1, 1.0, p, None),
        "detect_post_soft": lambda r, b, C: L.frcnn_detect_post_soft(p, p, p, r, b, C, 0.001, 1, 0.5, 0.3, 0.001, 100, 256, p, p, 0, p, p, p,
                                                                     None, 0, None),
        "detect_post_soft_vote": lambda r, b, C: L.frcnn_detect_post_soft_vote(p, p, p, r, b, C, 0.001, 1, 0.5, 0.3, 0.001, 100, 256, p, p,
                                                                               0, p, p, p, None, 0, 0.8, 1, 1.0, p, None),
        "detect_features": lambda r, b, C: L.frcnn_detect_features(p, p, p, r, b, C, 64, 256, p, p, None),
        "detect_regions": lambda r, b, C: L.frcnn_detect_regions(p, p, p, p, p, r, b, C, 64, 0.3, 1, 0.2, 10, 100, p, p, p, p, 1 << 40, p,
                                                                 p, p, p, p, p, p, p, None),
        "bbox_decode": lambda r, b, C: L.frcnn_bbox_decode(p, p, r * b, C, b, p, p, None),
    }


CLASS_ENTRIES = ["detect_post", "detect_post_vote", "detect_post_soft", "detect_post_soft_vote", "detect_features", "detect_regions"]


@pytest.mark.parametrize("name", CLASS_ENTRIES)
def test_c_entry_refuses_4097_classes(name):
    from tf_faster_rcnn_b200 import _native as N
    call = _entries()[name]
    assert call(300, 1, 4097) == ERR_ARG
    assert "4096" in N.last_error()


# r * C (or r * batch) past INT_MAX: refused before any CUDA call.  The post entries hold at most 8192 RoIs per image, so there the
# product cannot overflow and the RoI capacity refuses first.
@pytest.mark.parametrize("name,r,b,C,rc", [("bbox_decode", 1 << 19, 1, 4096, ERR_ARG), ("bbox_decode", 1 << 16, 8, 4096, ERR_ARG),
                                           ("detect_features", 1 << 19, 1, 4096, ERR_ARG), ("detect_features", 600000, 2, 3600, ERR_ARG),
                                           ("detect_regions", 8192, (1 << 18) + 1, 1601, ERR_ARG),
                                           ("detect_post", 1 << 19, 1, 4096, ERR_CAPACITY),
                                           ("detect_post_soft", 1 << 19, 1, 4096, ERR_CAPACITY),
                                           ("detect_post_vote", 1 << 19, 1, 4096, ERR_CAPACITY),
                                           ("detect_post_soft_vote", 1 << 19, 1, 4096, ERR_CAPACITY),
                                           ("detect_regions", 1 << 19, 1, 4096, ERR_CAPACITY)])
def test_c_entry_refuses_int_overflowing_sizes(name, r, b, C, rc):
    from tf_faster_rcnn_b200 import _native as N
    assert _entries()[name](r, b, C) == rc
    assert N.last_error()


def test_regions_mask_path_workspace():
    """C > 1024: the masks (r * ceil(r/32) words per image) and nothing of the per-class path; keep / keep_cnt / keep_score may be
    NULL there, but not below; a short workspace is refused."""
    from tf_faster_rcnn_b200 import _native as N, ops
    L, p = N.lib(), ctypes.c_void_p(4096)
    for r, b in ((300, 4), (1000, 1), (5000, 2), (8192, 1)):
        assert ops.detect_regions_workspace_bytes(r, 1601, b) >= b * r * ((r + 31) // 32) * 4
        assert ops.detect_regions_workspace_bytes(r, 1024, b) == L.frcnn_detect_post_workspace_bytes(r, 1024, b)
    for bad in ((0, 1601, 1), (300, 4097, 1), (300, 1601, 0)):
        with pytest.raises(RuntimeError, match="status -2"):
            ops.detect_regions_workspace_bytes(*bad)

    def call(C, keep, ws_bytes, ws=p):
        return L.frcnn_detect_regions(p, p, p, p, p, 300, 4, C, 64, 0.3, 1, 0.2, 10, 100, keep, keep, keep, ws, ws_bytes, p, p, p, p, p,
                                      p, p, p, None)
    need = ops.detect_regions_workspace_bytes(300, 1601, 4)
    assert call(1601, p, need - 1) == ERR_ARG and "workspace" in N.last_error()
    assert call(1601, p, need, ws=None) == ERR_ARG
    assert call(1601, p, need, ws=ctypes.c_void_p(4098)) == ERR_ARG
    assert call(1024, None, need) == ERR_ARG and "null" in N.last_error()


# ---- the overlap mask and the per-class walk, restated in numpy ------------------------------------------------------------------
def overlap_mask(boxes, thresh, use_gpu_nms, plus_one=True, swap=False):
    """[n, n] bool: row i suppresses row j, the '+1' predicate of oracle_nms_plus1 in fp32.  swap: an asymmetric mistake (the union
    uses area_i twice)."""
    inclusive = not use_gpu_nms
    t = NMS.thresh_f32(thresh, inclusive)
    x1, y1, x2, y2 = (boxes[:, k] for k in range(4))
    one = F(1) if plus_one else F(0)
    area = ((x2 - x1) + one) * ((y2 - y1) + one)
    with np.errstate(invalid="ignore", divide="ignore"):
        w = np.maximum(F(0), (np.minimum(x2[:, None], x2[None]) - np.maximum(x1[:, None], x1[None])) + one)
        h = np.maximum(F(0), (np.minimum(y2[:, None], y2[None]) - np.maximum(y1[:, None], y1[None])) + one)
        inter = w * h
        aj = np.broadcast_to(area[:, None], inter.shape) if swap else area[None]
        ovr = inter / ((area[:, None] + aj) - inter)
        return (ovr >= t) if inclusive else (ovr > t)


def mask_walk(boxes, probs, thresh, use_gpu_nms, mask=None, ties_high=False):
    """frcnn_detect_regions' C > 1024 algorithm: per class the rows in score order (ties to the lower row), each kept unless a kept
    row's mask row removed it; per row the largest kept score and the lowest class reaching it (the atomicMax of score << 32 | ~c)."""
    n, C = probs.shape
    M = overlap_mask(boxes, thresh, use_gpu_nms) if mask is None else mask
    best = np.zeros(n, np.uint64)
    rows = np.arange(n)
    for c in range(1, C):
        s = probs[:, c]
        order = np.lexsort((-rows if ties_high else rows, -s.astype(np.float64)))
        removed = np.zeros(n, bool)
        for i in order:
            if removed[i]:
                continue
            k = np.uint64((int(s[i].view(np.uint32)) << 32) | (~c & 0xffffffff))
            best[i] = max(best[i], k)
            removed |= M[i]
    conf = (best >> np.uint64(32)).astype(np.uint32).view(F)
    cls = np.where(conf > 0, np.uint64(0xffffffff) - (best & np.uint64(0xffffffff)), 0).astype(np.int32)
    return conf, cls


def tied_case(rng, n, C, degenerate=True):
    """n >= 64 rows of C > 1000 classes: random boxes and peaked scores, with ties, a class above 1024 tied with one below, and pairs
    placed where each mistake of test_mistakes_fail_the_comparison changes a result."""
    probs = rng.dirichlet(np.full(C, 0.05), n).astype(F)
    xy = rng.uniform(0, 300, (n, 2))
    wh = rng.uniform(10, 120, (n, 2))
    boxes = np.hstack([xy, xy + wh]).astype(F)
    boxes[5] = boxes[4]                                               # identical boxes
    boxes[9] = boxes[8] + F(1)                                        # overlapping boxes with tied scores in every class
    probs[9] = probs[8]
    probs[20:24, C - 1] = F(0.99)                                     # a top class above 1024, tied across four rows
    probs[30, 1000], probs[30, C - 1] = F(0.995), F(0.995)            # a best class above 1024 tied with one below: 1000 wins
    boxes[50], boxes[51] = [1000, 0, 1009, 9], [1000, 5, 1009, 14]    # IoU 1/3 with '+1' areas, 2/7 without
    probs[51] = probs[50] * F(0.5)
    boxes[60], boxes[61] = [2000, 0, 2009, 9], [2000, 0, 2039, 9]     # IoU 1/4; 1 or 1/7 when one area is used twice
    probs[61] = probs[60] * F(0.5)
    if degenerate:
        boxes[40] = [50, 50, 49, 49]                                  # zero '+1' area
        boxes[41] = [60, 60, 40, 40]                                  # negative area
        boxes[42] = [70, 70, 70, 70]                                  # one pixel
    return boxes, probs


@pytest.mark.parametrize("C", [1025, 1601])
@pytest.mark.parametrize("use_gpu_nms", [True, False])
def test_mask_walk_equals_oracle(C, use_gpu_nms):
    rng = np.random.default_rng(C + use_gpu_nms)
    boxes, probs = tied_case(rng, 120, C)
    want = RO.best_kept_class(boxes, probs, 0.3, use_gpu_nms)
    got = mask_walk(boxes, probs, 0.3, use_gpu_nms)
    assert got[0].tobytes() == want[0].tobytes() and got[1].tobytes() == want[1].tobytes()
    assert want[1][30] == 1000 and (want[1] >= 1024).any()


def test_mask_is_symmetric_with_degenerate_boxes():
    boxes, _ = tied_case(np.random.default_rng(3), 200, 1025)
    for gpu in (True, False):
        M = overlap_mask(boxes, 0.3, gpu)
        assert np.array_equal(M, M.T)


@pytest.mark.parametrize("mistake", ["asymmetric", "no_plus_one", "ties_high"])
def test_mistakes_fail_the_comparison(mistake):
    rng = np.random.default_rng(17)
    boxes, probs = tied_case(rng, 120, 1025, degenerate=False)
    want = RO.best_kept_class(boxes, probs, 0.3, False)
    if mistake == "asymmetric":
        got = mask_walk(boxes, probs, 0.3, False, mask=overlap_mask(boxes, 0.3, False, swap=True))
    elif mistake == "no_plus_one":
        got = mask_walk(boxes, probs, 0.3, False, mask=overlap_mask(boxes, 0.3, False, plus_one=False))
    else:
        got = mask_walk(boxes, probs, 0.3, False, ties_high=True)
    assert got[0].tobytes() != want[0].tobytes() or got[1].tobytes() != want[1].tobytes()


# ---- ptxas --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kernel,count", [("regions_mask_kernel", 1), ("regions_walk_kernel", 2), ("cap_emit_kernel", 2),
                                          ("detect_features_kernel", 1), ("regions_select_kernel", 1)])
def test_new_and_changed_kernels_do_not_spill(kernel, count):
    log = open(os.path.join(ROOT, "tf_faster_rcnn_b200", "csrc", "_obj", "nms.o.log")).read()
    found = re.findall(r"Function properties for \S*%s\S*\s*\n([^\n]*)" % kernel, log)
    assert len(found) == count, "ptxas reports for %s: %d" % (kernel, len(found))
    for line in found:
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in line, line
