"""Test-time augmentation (TEST.BBOX_AUG) on the host: config keys and merges, every ValueError before device work, the view
list and blob shapes, the grouping of views into shape plans, the numpy model of the union against the oracle's vstack, the
ABI's argument checks, and the absence of spills in the new kernels."""
import ctypes
import os
import re
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import aug_oracle as AO  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
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
    saved = (dict(cfg.TEST.BBOX_AUG), cfg.TEST.MODE, cfg.TEST.BBOX_REG, tuple(cfg.TEST.SCALES), cfg.TEST.MAX_SIZE)
    yield cfg.TEST.BBOX_AUG
    cfg.TEST.BBOX_AUG.update(saved[0])
    cfg.TEST.MODE, cfg.TEST.BBOX_REG, cfg.TEST.SCALES, cfg.TEST.MAX_SIZE = saved[1:]


def net_for_options(**cfg_test):
    from model.config import cfg
    from nets.mobilenet_v1 import mobilenetv1
    for k, v in cfg_test.items():
        cfg.TEST[k] = v
    net = mobilenetv1()
    net.create_architecture("TEST", 5, tag="default")
    return net


def test_config_defaults_and_merges(aug_cfg, tmp_path):
    from model.config import cfg_from_file, cfg_from_list
    from tf_faster_rcnn_b200 import engine
    assert dict(aug_cfg) == dict(ENABLED=False, H_FLIP=False, SCALES=(), MAX_SIZE=2000)
    assert engine.bbox_aug_option(aug_cfg) is None
    cfg_from_list(["TEST.BBOX_AUG.ENABLED", "True", "TEST.BBOX_AUG.H_FLIP", "True", "TEST.BBOX_AUG.SCALES", "(400, 800)",
                   "TEST.BBOX_AUG.MAX_SIZE", "1333"])
    assert engine.bbox_aug_option(aug_cfg) == (True, (400, 800), 1333)
    with pytest.raises(AssertionError):
        cfg_from_list(["TEST.BBOX_AUG.SCALES", "[500]"])             # a list for a tuple key
    y = tmp_path / "aug.yml"
    y.write_text("TEST:\n  BBOX_AUG:\n    ENABLED: false\n    SCALES: [500]\n    H_FLIP: false\n")
    cfg_from_file(str(y))
    assert aug_cfg.SCALES == (500,) and isinstance(aug_cfg.SCALES, tuple) and aug_cfg.ENABLED is False
    with pytest.raises(KeyError):
        y.write_text("TEST:\n  BBOX_AUG:\n    VOTE: true\n")
        cfg_from_file(str(y))


@pytest.mark.parametrize("update,match", [
    (dict(SCALES=(0,)), "positive"), (dict(SCALES=(500, -100)), "positive"), (dict(MAX_SIZE=0), "MAX_SIZE"),
    (dict(H_FLIP=True, SCALES=tuple(range(400, 1200, 100))), "18 views"),
])
def test_invalid_config_raises_before_device_work(aug_cfg, update, match):
    from model.test import detect_image, im_detect
    net = net_for_options()                                   # no weights: any device work would fail differently
    aug_cfg.update(ENABLED=True, **update)
    im = np.zeros((60, 80, 3), np.uint8)
    for call in (lambda: detect_image(net, im), lambda: im_detect(None, net, im)):
        with pytest.raises(ValueError, match=match):
            call()
    assert net._plans == {}


def test_bbox_reg_off_raises(aug_cfg):
    from model.test import im_detect
    net = net_for_options(BBOX_REG=False)
    aug_cfg.update(ENABLED=True, H_FLIP=True)
    with pytest.raises(ValueError, match="BBOX_REG"):
        im_detect(None, net, np.zeros((60, 80, 3), np.uint8))


def test_union_rows_over_capacity_raise(aug_cfg):
    """'top' mode keeps RPN_TOP_N = 5000 RoIs per view: two views are 10 000 union rows, over the post's 8192."""
    from model.test import detect_image, _detect_record
    net = net_for_options(MODE="top")
    aug_cfg.update(ENABLED=True, H_FLIP=True)
    im = np.zeros((60, 80, 3), np.uint8)
    for call in (lambda: detect_image(net, im), lambda: _detect_record(net, im, 0.0, 100)):
        with pytest.raises(ValueError, match="8192"):
            call()
    aug_cfg.update(H_FLIP=False)                              # one view of 5000 rows is allowed: the check is V * R
    from tf_faster_rcnn_b200 import engine
    engine.check_aug_views([(600, 800, False)], 5000, 6)
    with pytest.raises(ValueError, match="8192"):
        engine.check_aug_views([(600, 800, False)] * 14, 600, 6)
    engine.check_aug_views([(600, 800, False)] * 16, 512, 6)     # exactly 8192
    assert net._plans == {}


def test_too_many_shapes_for_the_plan_cache_raise(aug_cfg):
    from model.test import detect_image
    net = net_for_options()
    net.MAX_PLANS = 2
    aug_cfg.update(ENABLED=True, H_FLIP=True, SCALES=(300, 900))       # three blob shapes (identity and flip share one)
    with pytest.raises(ValueError, match="MAX_PLANS"):
        detect_image(net, np.zeros((600, 800, 3), np.uint8))
    aug_cfg.update(SCALES=(300,))
    from tf_faster_rcnn_b200 import engine
    engine.check_aug_views([(600, 800, True), (300, 400, False), (300, 400, True), (600, 800, False)], 300, 2)
    with pytest.raises(ValueError, match="16"):
        engine.check_aug_views([(600, 800, False)] * 17, 300, 6)


def test_caller_boxes_and_features_raise(aug_cfg):
    from model.test import im_detect
    net = net_for_options()
    aug_cfg.update(ENABLED=True)
    blob = np.zeros((1, 64, 96, 3), F)
    with pytest.raises(ValueError, match="caller boxes"):
        im_detect(None, net, np.zeros((64, 96, 3), np.uint8), boxes=np.zeros((2, 4), F))
    with pytest.raises(ValueError, match="caller boxes"):
        net.score_boxes(blob, [1.0], [(64, 96)], [np.zeros((2, 4), F)])
    with pytest.raises(ValueError, match="detect_features"):
        net.detect_features(blob, [1.0], [(64, 96)])
    assert net._plans == {}


@pytest.mark.parametrize("hw", [(375, 500), (500, 375), (333, 1000), (600, 800), (241, 1999)])
def test_view_list_and_blob_shapes(aug_cfg, hw):
    """Union order, per-view scale (MAX_SIZE caps), and blob_geometry == the host blob's shape for every view."""
    from model.test import aug_views, aug_view_blob, blob_geometry, _get_image_blob
    aug_cfg.update(ENABLED=True, H_FLIP=True, SCALES=(400, 900), MAX_SIZE=1200)
    v = aug_views(hw)
    assert v == AO.views(True, (400, 900), 1200) == [(600, 1000, True), (400, 1200, False), (400, 1200, True), (900, 1200, False),
                                                     (900, 1200, True), (600, 1000, False)]
    im = np.random.default_rng(hw[0]).integers(0, 256, hw + (3,), dtype=np.uint8)
    base, scales = _get_image_blob(im)
    for target, max_size, flip in v:
        blob, f = aug_view_blob(im, target, max_size, flip)
        H, W, g = blob_geometry(hw, target, max_size)
        assert blob.shape == (1, H, W, 3) and f == g
        capped = np.round(float(target) / min(hw) * max(hw)) > max_size
        assert f == (float(max_size) / max(hw) if capped else float(target) / min(hw))
        if (target, max_size) == (600, 1000):
            want = base if not flip else aug_view_blob(np.ascontiguousarray(im[:, ::-1]), target, max_size, False)[0]
            assert blob.tobytes() == want.tobytes() and f == scales[0]    # the base view is _get_image_blob's blob


def test_views_group_into_shape_plans():
    """Views of one blob shape share a plan at batch k*B: unflipped views first (identity = slots [0, B), its flip [B, 2B))."""
    from tf_faster_rcnn_b200 import engine
    shapes, slot, counts = engine.aug_groups([(600, 800, True), (400, 533, False), (400, 533, True), (600, 800, False)])
    assert shapes == [(600, 800), (400, 533)] and slot == [1, 0, 1, 0] and counts == {(600, 800): 2, (400, 533): 2}
    shapes, slot, counts = engine.aug_groups([(600, 800, False)])
    assert shapes == [(600, 800)] and slot == [0] and counts == {(600, 800): 1}
    # two extra scales that land on the base shape (a capped long side): three views in one plan
    shapes, slot, counts = engine.aug_groups([(600, 1000, True), (600, 1000, False), (600, 1000, True), (600, 1000, False)])
    assert shapes == [(600, 1000)] and slot == [2, 0, 3, 1] and counts == {(600, 1000): 4}


def random_views(rng, nv, B, C, max_rows=40):
    """nv views of random rows: counts mostly in [-2, R+2] (clamped by the union), else exactly 0 or R."""
    rows = [int(rng.integers(1, max_rows + 1)) for _ in range(nv)]
    probs = [rng.random((B, r, C), dtype=F) for r in rows]
    boxes = [(rng.random((B, r, 4 * C), dtype=F) * F(700)).astype(F) for r in rows]
    counts = [np.array([rng.integers(-2, r + 3) if rng.random() < 0.6 else (0 if rng.random() < 0.5 else r) for _ in range(B)], np.int32)
              for r in rows]
    flips = [bool(rng.random() < 0.5) for _ in range(nv)]
    return probs, boxes, counts, flips, rows


@pytest.mark.parametrize("nv", [1, 2, 3, 7, 16])
def test_union_model_against_the_oracle_vstack(nv):
    """Ragged, zero and out-of-range counts: the model's valid rows are the oracle's vstack (un-flipped), the tail is zero."""
    rng = np.random.default_rng(nv)
    B, C = 3, 21
    probs, boxes, counts, flips, rows = random_views(rng, nv, B, C)
    orig_w = [800, 333, 1000]
    up, ub, num = AO.union_model(probs, boxes, counts, flips, orig_w)
    assert up.shape == (B, sum(rows), C) and ub.shape == (B, sum(rows), 4 * C)
    for b in range(B):
        n = [int(np.clip(c[b], 0, r)) for c, r in zip(counts, rows)]
        s, x = AO.union([p[b, :k] for p, k in zip(probs, n)], [q[b, :k] for q, k in zip(boxes, n)], flips, orig_w[b])
        assert num[b] == sum(n) == s.shape[0]
        assert up[b, :num[b]].tobytes() == s.tobytes() and ub[b, :num[b]].tobytes() == x.tobytes()
        assert not up[b, num[b]:].any() and not ub[b, num[b]:].any()
        off = 0
        for v in range(nv):                                   # row i of view v sits at off_v + i; y never changes
            blk = ub[b, off:off + n[v]].reshape(n[v], C, 4)
            src = boxes[v][b, :n[v]].reshape(n[v], C, 4)
            assert np.array_equal(up[b, off:off + n[v]], probs[v][b, :n[v]])
            assert np.array_equal(blk[..., 1::2], src[..., 1::2])
            if flips[v]:
                assert np.array_equal(blk[..., 0], (F(orig_w[b]) - src[..., 2]) - F(1))
                assert np.array_equal(blk[..., 2], (F(orig_w[b]) - src[..., 0]) - F(1))
            else:
                assert np.array_equal(blk, src)
            off += n[v]


def test_unflip_arithmetic():
    """x1 = (W - x2') - 1, x2 = (W - x1') - 1 with fp32 roundings; exact and an involution on pixel-grid boxes."""
    W = 800
    b = np.array([[0.0, 5.0, 99.0, 60.0, 10.5, 0.0, 799.0, 599.0]], F)
    u = AO.unflip(b, W)
    assert u.tolist() == [[700.0, 5.0, 799.0, 60.0, 0.0, 0.0, 788.5, 599.0]]
    assert AO.unflip(u, W).tobytes() == b.tobytes()
    rng = np.random.default_rng(0)
    x = (rng.random((500, 8), dtype=F) * F(W - 1)).astype(F)
    got = AO.unflip(x, W)
    want = x.copy()
    want[:, 0::4] = (F(W) - x[:, 2::4]) - F(1)
    want[:, 2::4] = (F(W) - x[:, 0::4]) - F(1)
    assert got.tobytes() == want.tobytes() and got.dtype == F
    ref64 = np.float64(W) - x[:, 2::4].astype(np.float64) - 1.0
    assert np.abs(got[:, 0::4] - ref64).max() <= 2 ** -24 * W * 2   # two roundings of values below W


def test_abi_rejects_bad_arguments_without_a_device():
    from tf_faster_rcnn_b200 import _native
    L = _native.lib()
    p = ctypes.c_void_p(64)                 # never dereferenced: the checks come first
    vp = ctypes.c_void_p

    def union(nv=2, batch=1, C=21, rows=(300, 300), flips=(1, 0), ptr=64, out_box=64, null=None):
        arr = (vp * 16)(*([ptr] * 16))
        boxes = (vp * 16)(*([ptr] * 16))
        r = (ctypes.c_int * 16)(*(list(rows) + [300] * (16 - len(rows))))
        f = (ctypes.c_int * 16)(*(list(flips) + [0] * (16 - len(flips))))
        a = [arr, boxes, arr, r, f]
        if null is not None:
            a[null] = None
        return L.frcnn_aug_union(*a, nv, batch, C, p, p, vp(out_box), p, None)
    for bad in (dict(nv=0), dict(batch=0), dict(C=0), dict(rows=(300, 0)), dict(flips=(2, 0)), dict(ptr=0), dict(ptr=72),
                dict(out_box=72), dict(null=0), dict(null=1), dict(null=2), dict(null=3), dict(null=4)):
        assert union(**bad) == -2, bad
        assert _native.last_error()
    assert union(nv=17) == -5 and "capacity" in _native.last_error()
    m = (ctypes.c_double * 3)(1.0, 2.0, 3.0)
    for fn in (L.frcnn_preprocess, L.frcnn_preprocess_hflip):
        assert fn(p, 0, 10, m, 1.0, 1.0, p, 10, 10, None) == -2
        assert fn(p, 10, 10, m, 1.0, -1.0, p, 10, 10, None) == -2
        assert fn(p, 10, 10, None, 1.0, 1.0, p, 10, 10, None) == -2


@pytest.mark.parametrize("kernel", ["aug_union_kernel", "preprocess_kernelILb1E", "preprocess_kernelILb0E"])
def test_new_kernels_do_not_spill(kernel):
    """ptxas -v output written by the build."""
    log = open(os.path.join(ROOT, "tf_faster_rcnn_b200", "csrc", "_obj", "simt_ops.o.log")).read()
    found = re.findall(r"Function properties for \S*%s\S*\s*\n([^\n]*)" % kernel, log)
    assert len(found) == 1, "ptxas reports for %s: %d" % (kernel, len(found))
    assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in found[0], found[0]
