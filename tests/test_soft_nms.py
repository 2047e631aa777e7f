"""Soft-NMS, host side: the C oracle (the sequential definition) against the numpy model of the kernel's parallel formulation,
the swap-with-last order, the properties the record cap relies on, the configuration keys, the argument checks that run before
any device work, and the compiled kernels' register use."""
import ctypes
import os
import re
import sys

import numpy as np
import pytest

from oracle import nms as ONMS

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import soft_nms_model as SM  # noqa: E402
import soft_nms_oracle as SO  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = np.float32
PARAMS = [(m, s, nt, thr) for m in ("linear", "gaussian", "hard") for s in (0.5, 0.1) for nt in (0.3, 0.5) for thr in (0.001, 0.1)]


def make_set(rng, n, family):
    """Candidate rows [n,5]: clustered boxes (pruning chains, tail moves), duplicates, tied scores, degenerate boxes."""
    k = max(1, n // int(rng.integers(3, 12)))
    centres = rng.uniform(0, 400, (k, 2))
    xy = centres[rng.integers(0, k, n)] + rng.normal(0, rng.uniform(2, 20), (n, 2))
    wh = rng.uniform(4, 80, (n, 2))
    s = rng.uniform(0.0005, 1.0, n)
    d = np.hstack([xy, xy + wh, s[:, None]]).astype(F)
    if family in ("tied", "mixed"):
        d[:, 4] = (np.round(d[:, 4] * 6) / 6 + F(0.01)).astype(F)                    # few distinct scores
    if family in ("duplicates", "mixed") and n >= 2:
        src = rng.integers(0, n, n // 3)
        dst = rng.integers(0, n, n // 3)
        d[dst, :4] = d[src, :4]
        d[dst[: len(dst) // 2], 4] = d[src[: len(src) // 2], 4]                     # identical rows too
    if family in ("degenerate", "mixed") and n >= 1:
        bad = rng.integers(0, n, max(1, n // 8))
        d[bad, 2] = d[bad, 0] - F(rng.integers(0, 3))                                # zero / negative '+1' width
        pts = rng.integers(0, n, max(1, n // 16))
        d[pts, 2:4] = d[pts, 0:2]                                                   # single pixel: area 1
    return d


def same(a, b):
    return np.array_equal(a[1], b[1]) and a[0].shape == b[0].shape and a[0].tobytes() == b[0].tobytes()


def test_oracle_equals_parallel_model_on_random_sets():
    rng = np.random.default_rng(2017)
    families = ("clustered", "tied", "duplicates", "degenerate", "mixed")
    moved = 0
    for it in range(2000):
        n = int(rng.integers(0, 301))
        d = make_set(rng, n, families[it % len(families)])
        m, s, nt, thr = PARAMS[it % len(PARAMS)]
        want = SO.soft_nms_c(d, m, s, nt, thr)
        got = SM.soft_nms_model(d, m, s, nt, thr)
        assert same(want, got), (it, n, m, s, nt, thr)
        moved += int(want[1].shape[0] > 1 and np.any(np.diff(want[1]) < 0) and (want[1][1:] != np.sort(want[1][1:])).any())
    assert moved > 500            # the sets exercise reordering, not just identity output


@pytest.mark.parametrize("n,family,params", [(1000, "clustered", PARAMS[0]), (2500, "mixed", PARAMS[9]),
                                             (5000, "clustered", PARAMS[18]), (5000, "tied", PARAMS[5])])
def test_oracle_equals_parallel_model_on_large_sets(n, family, params):
    d = make_set(np.random.default_rng(n + len(family)), n, family)
    want = SO.soft_nms_c(d, *params)
    assert same(want, SM.soft_nms_model(d, *params))
    assert want[0].shape[0] < n or params[0] != "hard"


def test_swap_with_last_order():
    """Behind the selected box: [pruned, kept, pruned, kept, kept] = rows a1..a5 -> the next rows are [a5, a2, a4] (a stable
    compaction would give [a2, a4, a5])."""
    t = [0, 0, 10, 10, 1.0]
    dup = [0, 0, 10, 10, 0.5]                     # IoU 1 with t: linear weight 0 -> pruned
    far = lambda x: [x, 0, x + 10, 10, 0.5]       # noqa: E731  no overlap: kept, score tied
    d = np.array([t, dup, far(100), dup, far(200), far(300)], F)
    for fn in (SO.soft_nms_c, SM.soft_nms_model):
        rows, keep = fn(d, "linear", 0.5, 0.3, 0.001)
        assert keep.tolist() == [0, 5, 2, 4], fn
        assert np.array_equal(rows, d[[0, 5, 2, 4]])
        assert keep.tolist() != [0, 2, 4, 5]


def decay(t, b, s, params):
    """One decay of score s (box b) by the selected box t, the definition's fp32 arithmetic -> (new score, overlapped)."""
    m, sigma, nt, _ = params
    one = F(1)
    iw = (min(F(t[2]), F(b[2])) - max(F(t[0]), F(b[0]))) + one
    if not iw > 0:
        return s, False
    ih = (min(F(t[3]), F(b[3])) - max(F(t[1]), F(b[1]))) + one
    if not ih > 0:
        return s, False
    area = lambda u: ((F(u[2]) - F(u[0])) + one) * ((F(u[3]) - F(u[1])) + one)  # noqa: E731
    inter = iw * ih
    ov = inter / ((area(t) + area(b)) - inter)
    if m == "gaussian":
        w = F(np.exp(-np.float64((ov * ov) / F(sigma))))
    elif m == "linear":
        w = one - ov if ov > F(nt) else one
    else:
        w = F(0) if ov > F(nt) else one
    return F(w * s), True


def test_output_properties():
    rng = np.random.default_rng(5)
    for it in range(120):
        params = PARAMS[it % len(PARAMS)]
        d = make_set(rng, int(rng.integers(1, 120)), ("clustered", "mixed")[it % 2])
        rows, keep = SO.soft_nms_c(d, *params)
        assert (np.diff(rows[:, 4]) <= 0).all()                       # never increasing: the cap's binary search holds
        assert (rows[:, 4] <= d[keep, 4]).all()
        assert (rows[:, 4] > 0).all() or (d[:, 4] <= 0).any()
        assert np.array_equal(rows[:, :4], d[keep, :4])
        # each kept score is the input score decayed by the rows selected before it
        for k in range(min(len(keep), 12)):
            s = F(d[keep[k], 4])
            for t in keep[:k]:
                s = decay(d[t], d[keep[k]], s, params)[0]
            assert s.tobytes() == rows[k, 4].tobytes()
        # every dropped row was pruned: some selection overlapped it and left it below the threshold
        for j in sorted(set(range(d.shape[0])) - set(keep.tolist()))[:12]:
            s, hit = F(d[j, 4]), False
            for t in keep:
                s, ov = decay(d[t], d[j], s, params)
                if ov and s < F(params[3]):
                    hit = True
                    break
            assert hit, (it, j)


def test_hard_equals_greedy_gpu_nms_predicate_on_distinct_scores():
    rng = np.random.default_rng(11)
    for it in range(300):
        d = make_set(rng, int(rng.integers(0, 300)), "clustered")
        d[:, 4] = rng.permutation(d.shape[0]).astype(F) / F(max(d.shape[0], 1)) + F(0.2)       # distinct, above the prune threshold
        for nt in (0.3, 0.5, 0.7):
            rows, keep = SO.soft_nms_c(d, "hard", 0.5, nt, 0.001)
            assert np.array_equal(keep, ONMS.nms_plus1_c(d, nt, inclusive=False)), (it, nt)
            assert np.array_equal(rows, d[keep, :5])


def test_config_defaults_and_overrides():
    from model.config import cfg, cfg_from_list
    from tf_faster_rcnn_b200 import engine
    sn = cfg.TEST.SOFT_NMS
    assert dict(sn) == dict(ENABLED=False, METHOD="linear", SIGMA=0.5, SCORE_THRESH=0.001)
    assert engine.soft_nms_option(sn) is None
    saved = dict(sn)
    try:
        cfg_from_list(["TEST.SOFT_NMS.ENABLED", "True", "TEST.SOFT_NMS.METHOD", "gaussian", "TEST.SOFT_NMS.SIGMA", "0.1",
                       "TEST.SOFT_NMS.SCORE_THRESH", "0.01"])
        assert sn.ENABLED is True and sn.METHOD == "gaussian" and sn.SIGMA == 0.1 and sn.SCORE_THRESH == 0.01
        assert engine.soft_nms_option(sn) == ("gaussian", 0.1, 0.01)
        with pytest.raises(AssertionError):
            cfg_from_list(["TEST.SOFT_NMS.SIGMA", "1"])                   # int for a float key
    finally:
        sn.update(saved)


@pytest.mark.parametrize("key,value,match", [("METHOD", "box_voting", "METHOD"), ("SIGMA", 0.0, "SIGMA"), ("SIGMA", -1.0, "SIGMA"),
                                             ("SIGMA", float("nan"), "SIGMA"), ("SCORE_THRESH", 0.0, "SCORE_THRESH"),
                                             ("SCORE_THRESH", -0.1, "SCORE_THRESH"), ("SCORE_THRESH", 1e-50, "SCORE_THRESH")])
def test_invalid_values_raise_before_device_work(key, value, match):
    """Every check runs on the host first, so the answers are the same with and without a GPU."""
    from model.config import cfg
    from model.nms_wrapper import soft_nms
    from model.test import _set_post_options
    from nets.mobilenet_v1 import mobilenetv1
    sn = cfg.TEST.SOFT_NMS
    saved = dict(sn)
    try:
        sn.ENABLED = True
        sn[key] = value
        with pytest.raises(ValueError, match=match):
            mobilenetv1().create_architecture("TEST", 5, tag="default")
        sn.update(saved)
        net = mobilenetv1()
        net.create_architecture("TEST", 5, tag="default")
        assert net.options["soft_nms"] is None
        sn.ENABLED = True
        sn[key] = value
        with pytest.raises(ValueError, match=match):
            _set_post_options(net, 0.0, 100)
    finally:
        sn.update(saved)
    args = dict(method="linear", sigma=0.5, score_thresh=0.001)
    args[{"METHOD": "method", "SIGMA": "sigma", "SCORE_THRESH": "score_thresh"}[key]] = value
    with pytest.raises(ValueError, match=match):
        soft_nms(np.zeros((3, 5), F), **args)
    with pytest.raises(ValueError, match=match):
        soft_nms(np.zeros((0, 5), F), **args)


def test_soft_nms_option_reaches_the_network():
    from model.config import cfg
    from model.test import _set_post_options
    from nets.mobilenet_v1 import mobilenetv1
    sn = cfg.TEST.SOFT_NMS
    saved = dict(sn)
    try:
        sn.update(ENABLED=True, METHOD="hard")
        net = mobilenetv1()
        net.create_architecture("TEST", 5, tag="default")
        assert net.options["soft_nms"] == ("hard", 0.5, 0.001)
        sn.update(METHOD="gaussian", SIGMA=0.25)
        _set_post_options(net, 0.05, 100)
        assert net.options["soft_nms"] == ("gaussian", 0.25, 0.001)
        sn.ENABLED = False
        _set_post_options(net, 0.05, 100)
        assert net.options["soft_nms"] is None
    finally:
        sn.update(saved)


def test_abi_rejects_bad_parameters_without_a_device():
    from tf_faster_rcnn_b200 import _native
    L = _native.lib()
    p = ctypes.c_void_p(64)                     # never dereferenced: the checks come first

    def post(r=300, method=0, sigma=0.5, nt=0.3, thr=0.001, stride=0):
        return L.frcnn_detect_post_soft(p, p, p, r, 1, 81, 0.0, method, sigma, nt, thr, 100, 256, p, p, stride, p, p, p, None, 0, None)

    def greedy(r=300, stride=0):
        return L.frcnn_detect_post(p, p, p, r, 1, 81, 0.0, 0.3, 0, 100, 256, p, p, stride, p, p, p, None, 0, None)
    dets = np.zeros((8193, 5), F)
    out, keep, num = np.zeros((8193, 5), F), np.zeros(8193, np.int32), ctypes.c_int(7)

    def host(n=4, method=0, sigma=0.5, nt=0.3, thr=0.001):
        return L.frcnn_soft_nms_host(out.ctypes.data_as(_native.fp), keep.ctypes.data_as(_native.ip), ctypes.byref(num),
                                     dets.ctypes.data_as(_native.fp), n, 5, method, sigma, nt, thr, -1)
    for fn in (post, host):
        for bad in (dict(method=3), dict(method=-1), dict(sigma=0.0), dict(sigma=-0.5), dict(sigma=float("nan")), dict(thr=0.0),
                    dict(thr=-1.0), dict(nt=float("nan"))):
            assert fn(**bad) == -2, (fn.__name__, bad)
            assert _native.last_error()
    assert post(r=8193) == -5 and "capacity" in _native.last_error()
    for fn in (post, greedy):                   # both post entries check the record layout and the capacity before any launch
        assert fn(stride=5) == -2 and "record_stride" in _native.last_error(), fn.__name__
        assert fn(r=8193) == -5 and "capacity" in _native.last_error(), fn.__name__
    assert host(n=8193) == -5 and "capacity" in _native.last_error()
    assert host(n=0) == 0 and num.value == 0
    assert L.frcnn_soft_nms_host(None, keep.ctypes.data_as(_native.ip), ctypes.byref(num), None, 0, 5, 0, 0.5, 0.3, 0.001, -1) == -2


@pytest.mark.parametrize("kernel", ["class_soft_nms_kernel", "soft_nms_set_kernel"])
def test_soft_nms_kernels_do_not_spill(kernel):
    """ptxas -v output written by the build, both capacities (256 threads x 4 and 1024 threads x 8 positions)."""
    log = open(os.path.join(ROOT, "tf_faster_rcnn_b200", "csrc", "_obj", "nms.o.log")).read()
    found = re.findall(r"Function properties for \S*%s\S*\s*\n([^\n]*)" % kernel, log)
    assert len(found) == 2, "ptxas reports for %s: %d" % (kernel, len(found))
    for line in found:
        assert "0 bytes spill stores, 0 bytes spill loads" in line, line
