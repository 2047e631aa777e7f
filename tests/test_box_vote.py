"""Box voting, host side: the C oracle (include/frcnn_b200.h's definition) against a float64 numpy restatement of Detectron's
box_voting within a derived bound, for every scoring method, VOTE_TH and beta; one plausible implementation mistake failing the
comparators each; the configuration keys, the argument checks that run before any device work, the C ABI's refusals, and the
compiled kernels' register use."""
import ctypes
import os
import re
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import box_vote_oracle as BV  # noqa: E402
from test_soft_nms import make_set  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = np.float32
METHODS = tuple(BV.METHODS)
U = 2.0 ** -53
PARAMS = [(m, th, b) for m in METHODS for th in (0.5, 0.8, 1.0) for b in (0.5, 1.0, 2.0)]


@pytest.fixture(scope="module", autouse=True)
def _restore_network_registry():
    """The networks built here leave the process-wide registry afterwards (Saver.restore walks it)."""
    from nets import network
    before = list(network._REGISTRY)
    yield
    network._REGISTRY[:] = before


def make_vote_case(rng, n, family):
    """(top [k,5], all [n,5]): candidates from make_set (clusters, duplicates, degenerate boxes) with scores pushed towards 0 and 1,
    plus rows overlapping a top box by exactly 0.5 and 0.8 (in fp32) and an exact duplicate; the top boxes are candidates, rows
    far from every candidate (empty vote sets) and a degenerate box."""
    a = make_set(rng, n, family)
    a[:, 4] = np.minimum(a[:, 4], F(1))                       # probabilities ('tied' adds 0.01)
    if n:
        edge = rng.integers(0, n, max(1, n // 6))
        a[edge, 4] = rng.choice(np.array([1.0, 1 - 2 ** -24, 0.999, 1e-3, 2 ** -20, 0.5], F), edge.shape[0])
    # a 10x10 box (area 100 with '+1') and boxes overlapping it by exactly 0.5 (10x5) and 0.8 (10x8), plus a duplicate
    base = np.array([200, 300, 209, 309], F)
    ties = np.array([base, [200, 300, 209, 304], [200, 300, 209, 307], base], F)
    a = np.vstack([a, np.hstack([ties, rng.uniform(0.05, 1.0, (4, 1)).astype(F)])]).astype(F)
    k = max(1, a.shape[0] // 4)
    top = a[rng.choice(a.shape[0], k, replace=False)].copy()
    top = np.vstack([top, np.hstack([ties[:1], [[0.7]]]).astype(F), [[5000, 5000, 5010, 5010, 0.3]], [[50, 50, 40, 45, 0.2]]]).astype(F)
    return top, a


def overlaps32(t, a, plus1=True):
    """ov(t, a) of the header for every (top, candidate) pair, fp32 op by op (numpy float32 rounds each operation)."""
    one = F(1) if plus1 else F(0)
    t, a = t[:, None, :4].astype(F), a[None, :, :4].astype(F)
    iw = (np.minimum(t[..., 2], a[..., 2]) - np.maximum(t[..., 0], a[..., 0])) + one
    ih = (np.minimum(t[..., 3], a[..., 3]) - np.maximum(t[..., 1], a[..., 1])) + one
    area = lambda u: ((u[..., 2] - u[..., 0]) + one) * ((u[..., 3] - u[..., 1]) + one)  # noqa: E731
    inter = iw * ih
    with np.errstate(invalid="ignore", divide="ignore"):
        ov = inter / ((area(t) + area(a)) - inter)
    return np.where((iw > 0) & (ih > 0), ov, F(0)).astype(F)


def detectron64(top, a, th, method, beta, variant=0):
    """Detectron's box_voting restated in float64 (numpy's pairwise sums), the overlaps in the header's fp32 order, with this
    project's empty-vote-set rule -> (float64 [k,5] voted rows, float64 [k,5] error allowance E, see `check`)."""
    top, a = np.asarray(top, F)[:, :5], np.asarray(a, F)[:, :5]
    out = top.astype(np.float64)
    err = np.zeros_like(out)
    if top.shape[0] == 0 or a.shape[0] == 0:
        return out, err
    ov = overlaps32(top, a)
    th32, b = F(th), float(F(beta))
    for i in range(top.shape[0]):
        v = ov[i] >= th32
        n = int(v.sum())
        if n == 0:
            continue
        s = a[v, 4].astype(np.float64)
        bx = a[v, :4].astype(np.float64)
        S = s.sum()
        g = n * U / (1 - n * U)
        if S != 0:
            out[i, :4] = (s[:, None] * bx).sum(axis=0) / S
            err[i, :4] = g * ((s[:, None] * np.abs(bx)).sum(axis=0) / S + np.abs(out[i, :4])) + 2 * U * np.abs(out[i, :4])
        if method == "ID":
            continue
        if method == "AVG":
            val, e = S / n, (g + 2 * U) * S / n
        elif method == "IOU_AVG":
            w = ov[i, v].astype(np.float64)
            val = (w * s).sum() / w.sum()
            e = (2 * g + 2 * U) * val
        elif method == "GENERALIZED_AVG":
            val = np.log(np.exp(b * s).mean()) / b
            e = (g + 4 * 2 * U) / b + 4 * U * abs(val)
        elif method == "QUASI_SUM":
            val = S / float(n) ** b
            e = (g + 6 * U) * val
        else:                                               # TEMP_AVG
            p = np.vstack([s, 1.0 - s])
            m = p.max(axis=0)
            with np.errstate(divide="ignore"):
                x = np.log(p / m)
            ex = np.exp(x / b)
            val = (ex[0] / ex.sum(axis=0)).mean()
            lg = np.abs(x[np.isfinite(x)]).max() if np.isfinite(x).any() else 0.0
            A = (2 * U * lg + 2 * U) / b + 2 * U * lg / b + 2 * U
            e = (4 * A + g + 4 * U) * val
        out[i, 4], err[i, 4] = val, e
    return out, err


def check(got, want, err, what=""):
    """|got - want| <= ulp32(want)/2 + 2E per element.  The oracle rounds its fp64 result once to fp32 (half an fp32 ulp); E bounds
    one fp64 evaluation's distance from the exact value: a sum of n terms is off by <= gamma_n * sum|term|, gamma_n =
    n*2^-53/(1 - n*2^-53), each division / exp / log / pow adds one or two units of 2^-53 relative, and an exp or log error passes
    to the result as its argument's absolute error (divided by beta for GENERALIZED_AVG and TEMP_AVG).  The oracle's sums and
    numpy's pairwise sums each meet E, so the two fp64 values lie within 2E."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    err = np.broadcast_to(np.asarray(err, np.float64), want.shape)
    ulp = np.spacing(np.abs(want + 2 * err).astype(F)).astype(np.float64)
    bad = (np.abs(got - want) > ulp / 2 + 2 * err) | np.isnan(got) | np.isnan(want)
    if bad.any():
        i = np.unravel_index(np.argmax(bad), bad.shape)
        raise AssertionError("%s: %d elements off, first at %s: got %r, want %r (allowance %r)"
                             % (what, int(bad.sum()), i, got[i], want[i], ulp[i] / 2 + 2 * err[i]))


FAMILIES = ("clustered", "tied", "duplicates", "degenerate", "mixed")


@pytest.mark.parametrize("method", METHODS)
def test_oracle_within_bound_of_float64_detectron(method):
    rng = np.random.default_rng(METHODS.index(method) + 1)
    checked = voted = 0
    for it, (m, th, b) in enumerate([p for p in PARAMS if p[0] == method] * 6):
        n = int(rng.integers(0, 200))
        top, a = make_vote_case(rng, n, FAMILIES[it % len(FAMILIES)])
        got = BV.box_vote_c(top, a, th, m, b)
        want, err = detectron64(top, a, th, m, b)
        check(got, want, err, (m, th, b, n))
        checked += got.shape[0]
        voted += int((got[:, :4] != top[:, :4]).any(axis=1).sum())
    assert voted > checked // 12             # boxes that moved: the sets exercise real votes, not just singletons


def test_definition_edges():
    """Empty vote set: box and score kept.  A top box whose voters are itself or exact duplicates of itself keeps its box bit for
    bit.  A row at exactly VOTE_TH votes."""
    t = np.array([[10, 10, 19, 19, 0.9]], F)
    far = np.array([[100, 100, 110, 110, 0.8]], F)
    for m in METHODS:
        assert BV.box_vote_c(t, far, 0.5, m).tobytes() == t.tobytes()
        dup = np.vstack([t, t[:, :4].tolist()[0] + [0.3], t[:, :4].tolist()[0] + [0.77]]).astype(F)
        assert BV.box_vote_c(t, dup, 0.8, m)[0, :4].tobytes() == t[0, :4].tobytes()
    half = np.array([[10, 10, 19, 19, 0.9], [10, 10, 19, 14, 0.1]], F)      # IoU exactly 0.5
    assert overlaps32(t, half)[0, 1] == F(0.5)
    got = BV.box_vote_c(t, half, 0.5, "AVG")
    assert got[0, 3] != t[0, 3] and got[0, 4] == F((0.9 + np.float64(F(0.1))) / 2)
    assert BV.box_vote_c(t, half, 0.5, "AVG", variant=BV.STRICT)[0, 4] == F(0.9)


@pytest.mark.parametrize("variant", [BV.STRICT, BV.NO_PLUS_ONE, BV.FP32_SUMS])
def test_each_oracle_mistake_fails_the_bound(variant):
    rng = np.random.default_rng(100 + variant)
    caught = 0
    for it, (m, th, b) in enumerate(PARAMS):
        top, a = make_vote_case(rng, 120, FAMILIES[it % len(FAMILIES)])
        got = BV.box_vote_c(top, a, th, m, b, variant=variant)
        want, err = detectron64(top, a, th, m, b)
        try:
            check(got, want, err)
        except AssertionError:
            caught += 1
    assert caught >= len(PARAMS) // 3, caught


def post_inputs(seed, r=200, C=6):
    rng = np.random.default_rng(seed)
    prob = rng.dirichlet(np.full(C, 0.3), r).astype(F)
    boxes = np.zeros((r, C, 4), F)
    for j in range(C):
        boxes[:, j] = make_set(rng, r, ("clustered", "duplicates")[j % 2])[:, :4]
    return prob, boxes.reshape(r, 4 * C)


def restated_post(prob, pred, vote, soft):
    """test_net_post_vote with the float64 restatement as the vote (re-sorted by the fp32 rounding of its scores), no cap."""
    def vote64(top, a, th, m, b, variant):
        out, err = detectron64(top, a, th, m, b)
        restated_post.err.append(err)
        return out
    restated_post.err = []
    out, _ = BV.test_net_post_vote(prob, pred, vote, 0.3, 0, 0.0, soft=soft, vote_fn=vote64,
                                   resort=lambda rows: np.argsort(-rows[:, 4].astype(F), kind="stable"))
    return out, restated_post.err


def post_check(got, want, errs):
    for j in range(1, len(got)):
        assert got[j].shape == want[j].shape, j
        # restated rows were re-sorted like the oracle's: apply the same order to the allowance by matching rows
        check(got[j], want[j], np.max(errs[j - 1]) if errs[j - 1].size else 0.0, j)


@pytest.mark.parametrize("soft", [None, ("linear", 0.5, 0.001)])
def test_post_oracle_within_bound_and_post_mistakes_fail(soft):
    """The oracle's voted post (no cap) against the float64 restatement; votes against the Soft-NMS output (decayed weights, the
    pruned candidates missing) and a re-sort that puts ties in reverse NMS order are caught."""
    prob, pred = post_inputs(7)
    # two far-apart identical clusters in class 1: equal voted scores, different boxes -> the re-sort must keep NMS order
    clus = np.array([[0, 0, 30, 30], [1, 0, 31, 30], [0, 1, 30, 31]], F)
    pred[:3, 4:8], pred[3:6, 4:8] = clus, clus + F(500)
    prob[:6, 1] = np.array([0.9, 0.6, 0.3, 0.9, 0.6, 0.3], F)
    for vote in (("AVG", 0.5), ("TEMP_AVG", 0.8), ("ID", 0.8)):
        v = (vote[1], vote[0], 1.0)
        got, _ = BV.test_net_post_vote(prob, pred, v, 0.3, 0, 0.0, soft=soft)
        want, errs = restated_post(prob, pred, v, soft)
        post_check(got, want, errs)
        if vote[0] == "ID":
            continue
        rev = lambda rows: np.lexsort((-np.arange(rows.shape[0]), -rows[:, 4].astype(np.float64)))  # noqa: E731
        bad, _ = BV.test_net_post_vote(prob, pred, v, 0.3, 0, 0.0, soft=soft, resort=rev)
        with pytest.raises(AssertionError):
            post_check(bad, want, errs)
        if soft is not None:
            bad, _ = BV.test_net_post_vote(prob, pred, v, 0.3, 0, 0.0, soft=soft, weights="decayed")
            with pytest.raises(AssertionError):
                post_check(bad, want, errs)


def test_resorted_lists_stay_sorted_and_nonnegative():
    """What the record cap relies on: after the re-sort every class list is non-increasing and every voted score is >= +0 (never
    -0, never NaN)."""
    rng = np.random.default_rng(3)
    for it, (m, th, b) in enumerate(PARAMS):
        top, a = make_vote_case(rng, 150, FAMILIES[it % len(FAMILIES)])
        top[:, 4] = np.clip(top[:, 4], F(1e-6), F(1))
        a[:, 4] = np.clip(a[:, 4], F(1e-6), F(1))
        rows = BV.box_vote_c(top, a, th, m, b)
        s = rows[BV.stable_resort(rows), 4]
        assert not np.isnan(s).any() and (s.view(np.int32) >= 0).all(), (m, th, b)
        if m != "ID":
            assert (np.diff(s) <= 0).all()


def test_config_defaults_and_overrides():
    from model.config import cfg, cfg_from_list
    from tf_faster_rcnn_b200 import engine
    bv = cfg.TEST.BBOX_VOTE
    assert dict(bv) == dict(ENABLED=False, VOTE_TH=0.8, SCORING_METHOD="ID", SCORING_METHOD_BETA=1.0)
    assert engine.box_vote_option(bv) is None
    saved = dict(bv)
    try:
        cfg_from_list(["TEST.BBOX_VOTE.ENABLED", "True", "TEST.BBOX_VOTE.VOTE_TH", "0.5", "TEST.BBOX_VOTE.SCORING_METHOD", "TEMP_AVG",
                       "TEST.BBOX_VOTE.SCORING_METHOD_BETA", "2.0"])
        assert engine.box_vote_option(bv) == (0.5, "TEMP_AVG", 2.0)
        assert engine.box_vote_args(*engine.box_vote_option(bv)) == (0.5, 5, 2.0)
        with pytest.raises(AssertionError):
            cfg_from_list(["TEST.BBOX_VOTE.VOTE_TH", "1"])                  # int for a float key
    finally:
        bv.update(saved)


def test_yaml_merge(tmp_path):
    from model.config import cfg, cfg_from_file
    from tf_faster_rcnn_b200 import engine
    bv = cfg.TEST.BBOX_VOTE
    saved = dict(bv)
    p = tmp_path / "vote.yml"
    p.write_text("TEST:\n  BBOX_VOTE:\n    ENABLED: True\n    SCORING_METHOD: IOU_AVG\n")
    try:
        cfg_from_file(str(p))
        assert engine.box_vote_option(bv) == (0.8, "IOU_AVG", 1.0)
    finally:
        bv.update(saved)


@pytest.mark.parametrize("key,value,match", [("SCORING_METHOD", "avg", "SCORING_METHOD"), ("SCORING_METHOD", "MAX", "SCORING_METHOD"),
                                             ("VOTE_TH", 0.0, "VOTE_TH"), ("VOTE_TH", -0.5, "VOTE_TH"), ("VOTE_TH", 1.5, "VOTE_TH"),
                                             ("VOTE_TH", float("nan"), "VOTE_TH"), ("VOTE_TH", 1e-50, "VOTE_TH"),
                                             ("SCORING_METHOD_BETA", 0.0, "BETA"), ("SCORING_METHOD_BETA", -1.0, "BETA"),
                                             ("SCORING_METHOD_BETA", float("inf"), "BETA"), ("SCORING_METHOD_BETA", float("nan"), "BETA")])
def test_invalid_values_raise_before_device_work(key, value, match):
    """Every check runs on the host first, so the answers are the same with and without a GPU."""
    from model.config import cfg
    from model.nms_wrapper import box_voting
    from model.test import _set_post_options
    from nets.mobilenet_v1 import mobilenetv1
    bv = cfg.TEST.BBOX_VOTE
    saved = dict(bv)
    try:
        bv.ENABLED = True
        bv[key] = value
        with pytest.raises(ValueError, match=match):
            mobilenetv1().create_architecture("TEST", 5, tag="default")
        bv.update(saved)
        net = mobilenetv1()
        net.create_architecture("TEST", 5, tag="default")
        assert net.options["box_vote"] is None
        bv.ENABLED = True
        bv[key] = value
        with pytest.raises(ValueError, match=match):
            _set_post_options(net, 0.0, 100)
    finally:
        bv.update(saved)
    args = dict(thresh=0.8, scoring_method="ID", beta=1.0)
    args[{"SCORING_METHOD": "scoring_method", "VOTE_TH": "thresh", "SCORING_METHOD_BETA": "beta"}[key]] = value
    for top in (np.zeros((3, 5), F), np.zeros((0, 5), F)):
        with pytest.raises(ValueError, match=match):
            box_voting(top, np.zeros((3, 5), F), **args)


def test_box_vote_option_reaches_the_network():
    from model.config import cfg
    from model.test import _set_post_options
    from nets.mobilenet_v1 import mobilenetv1
    bv = cfg.TEST.BBOX_VOTE
    saved = dict(bv)
    try:
        bv.update(ENABLED=True, SCORING_METHOD="AVG")
        net = mobilenetv1()
        net.create_architecture("TEST", 5, tag="default")
        assert net.options["box_vote"] == (0.8, "AVG", 1.0)
        bv.update(VOTE_TH=0.6)
        _set_post_options(net, 0.05, 100)
        assert net.options["box_vote"] == (0.6, "AVG", 1.0)
        bv.ENABLED = False
        _set_post_options(net, 0.05, 100)
        assert net.options["box_vote"] is None
    finally:
        bv.update(saved)


def test_post_key_default_keeps_existing_constructions():
    from tf_faster_rcnn_b200 import engine
    k = engine.PostKey(0.0, 0.3, True, 100, None)
    assert k.box_vote is None and k == engine.PostKey(0.0, 0.3, True, 100, None, None)
    assert k != k._replace(box_vote=(0.8, 0, 1.0))


def test_abi_rejects_bad_parameters_without_a_device():
    from tf_faster_rcnn_b200 import _native
    L = _native.lib()
    p = ctypes.c_void_p(64)                     # never dereferenced: the checks come first

    def greedy(r=300, th=0.8, method=0, beta=1.0, stride=0, vb=p):
        return L.frcnn_detect_post_vote(p, p, p, r, 1, 81, 0.0, 0.3, 0, 100, 256, p, p, stride, p, p, p, None, 0, th, method, beta, vb,
                                        None)

    def soft(r=300, th=0.8, method=0, beta=1.0, stride=0, vb=p):
        return L.frcnn_detect_post_soft_vote(p, p, p, r, 1, 81, 0.0, 0, 0.5, 0.3, 0.001, 100, 256, p, p, stride, p, p, p, None, 0, th,
                                             method, beta, vb, None)
    a = np.zeros((8193, 5), F)
    out = np.zeros((8193, 5), F)

    def host(n_top=4, n_all=4, th=0.8, method=0, beta=1.0):
        return L.frcnn_box_vote_host(out.ctypes.data_as(_native.fp), a.ctypes.data_as(_native.fp), n_top, 5, a.ctypes.data_as(_native.fp),
                                     n_all, 5, th, method, beta, -1)
    for fn in (greedy, soft, host):
        for bad in (dict(method=6), dict(method=-1), dict(th=0.0), dict(th=-0.1), dict(th=1.0001), dict(th=float("nan")),
                    dict(beta=0.0), dict(beta=-1.0), dict(beta=float("inf")), dict(beta=float("nan"))):
            assert fn(**bad) == -2, (fn.__name__, bad)
            assert _native.last_error()
    for fn in (greedy, soft):
        assert fn(stride=5) == -2 and "record_stride" in _native.last_error(), fn.__name__
        assert fn(r=8193) == -5 and "capacity" in _native.last_error(), fn.__name__
        assert fn(vb=None) == -2 and "vote_box" in _native.last_error(), fn.__name__
        assert fn(vb=ctypes.c_void_p(72)) == -2 and "vote_box" in _native.last_error(), fn.__name__
    assert host(n_all=8193) == -5 and "capacity" in _native.last_error()
    assert host(n_top=0) == 0                                   # nothing to vote: no device work
    assert L.frcnn_box_vote_host(None, a.ctypes.data_as(_native.fp), 4, 5, None, 0, 5, 0.8, 0, 1.0, -1) == -2


@pytest.mark.parametrize("kernel", ["class_vote_kernel", "box_vote_set_kernel", "cap_emit_kernel"])
def test_vote_kernels_do_not_spill(kernel):
    """ptxas -v output written by the build: both capacities (256 threads x 4 and 1024 threads x 8 candidates) of the vote kernels,
    both instantiations of the cap."""
    log = open(os.path.join(ROOT, "tf_faster_rcnn_b200", "csrc", "_obj", "nms.o.log")).read()
    found = re.findall(r"Function properties for \S*%s\S*\s*\n([^\n]*)" % kernel, log)
    assert len(found) == 2, "ptxas reports for %s: %d" % (kernel, len(found))
    for line in found:
        assert "0 bytes spill stores, 0 bytes spill loads" in line, line
