"""The post-processing extensions at their edges, through the C ABI, bit for bit against the C oracles and numpy models:
Soft-NMS on one set (frcnn_soft_nms_host) and per class (frcnn_detect_post_soft), box voting on both posts, the augmentation
union, boxes_to_rois and detect_features.  Every output sits between sentinel guard bands and every input is checked unchanged
afterwards.  NaN scores compare as NaN (the device's NaN bit pattern is not the host's); everything else compares bit for bit."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import aug_oracle as AO  # noqa: E402
import box_vote_oracle as BV  # noqa: E402
import post_ref64 as R  # noqa: E402
import soft_nms_oracle as SO  # noqa: E402
import stage_ref64 as S  # noqa: E402

pytestmark = pytest.mark.gpu
F = np.float32
HOST_GUARD = 16


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def unchanged(d, a, what):
    assert d.cpu().numpy().tobytes() == np.ascontiguousarray(a).tobytes(), "%s was modified" % what


def same_bits(got, want, what):
    """Bit for bit, except that any NaN equals any NaN."""
    got, want = np.asarray(got, F), np.asarray(want, F)
    assert got.shape == want.shape, "%s: shape %s, want %s" % (what, got.shape, want.shape)
    gn, wn = np.isnan(got), np.isnan(want)
    assert np.array_equal(gn, wn), "%s: NaN positions differ" % what
    bad = got.view(np.int32)[~gn] != want.view(np.int32)[~wn]
    assert not bad.any(), "%s: %d values differ" % (what, int(bad.sum()))


def guarded_int(shape):
    buf, t = S.guarded_out(shape, 0.0)
    return buf, t.view(torch.int32)


# ---- Soft-NMS, one set ---------------------------------------------------------------------------------------------------
def soft_set(d, method, sigma, nt, thr):
    """frcnn_soft_nms_host into host buffers with HOST_GUARD sentinel rows past n -> (rows [k,5], keep [k]).  The guard bands
    are on the host side: the entry sizes its device buffers to n itself, so only the copies back can be fenced here."""
    from tf_faster_rcnn_b200 import _native as N, engine
    code, s32, p32 = engine.soft_nms_args(method, sigma, thr)
    d = np.ascontiguousarray(d, F)
    d0 = d.copy()
    n = d.shape[0]
    out = np.full((n + HOST_GUARD, 5), S.SENTINEL, np.int32).view(F)
    keep = np.full(n + HOST_GUARD, -7, np.int32)
    num = ctypes.c_int(-1)
    N.check(N.lib().frcnn_soft_nms_host(out.ctypes.data_as(N.fp), keep.ctypes.data_as(N.ip), ctypes.byref(num), d.ctypes.data_as(N.fp),
                                        n, 5, code, float(s32), float(F(nt)), float(p32), -1), "soft_nms_host")
    k = num.value
    assert 0 < k <= n or (k == 0 and n == 0)
    assert (out[k:].view(np.int32) == S.SENTINEL).all() and (keep[k:] == -7).all(), "store past the kept rows"
    assert d.tobytes() == d0.tobytes(), "input rows were modified"
    return out[:k], keep[:k]


@pytest.mark.parametrize("n", [1, 1023, 1024, 1025, 8191, 8192])
def test_soft_nms_set_edges(cuda, n):
    """Every edge generator in all three methods, on both kernel variants (256 x 4 up to 1024, 1024 x 8 above)."""
    for edge, gen in sorted(R.EDGES.items()):
        d, (method0, sigma, nt, thr) = gen(np.random.default_rng(n), n)
        for method in (method0,) + tuple(m for m in ("linear", "gaussian", "hard") if m != method0):
            want_rows, want_keep = SO.soft_nms_c(d, method, sigma, nt, thr)
            rows, keep = soft_set(d, method, sigma, nt, thr)
            assert np.array_equal(keep, want_keep), (edge, n, method)
            same_bits(rows, want_rows, "%s n=%d %s" % (edge, n, method))


def test_soft_nms_set_nan_head_rule(cuda):
    """The NaN finding's four rows: the device takes [0, 3, 2, 1] as the scan rule does."""
    rows, keep = soft_set(R.NAN_ROWS, "linear", 0.5, 0.3, 0.001)
    assert keep.tolist() == R.NAN_KEEP
    same_bits(rows, R.NAN_ROWS[R.NAN_KEEP], "nan rows")


# ---- the class path: Soft-NMS and voting on both posts -------------------------------------------------------------------
def post(prob, pred, r, C, nroi, soft, vote, mpi, max_det, thresh=0.0):
    """The post entries on guard-banded outputs, inputs checked unchanged.  soft = (method, sigma, prune) or None (greedy, the
    gpu_nms predicate); vote = (VOTE_TH, METHOD, BETA) or None."""
    from tf_faster_rcnn_b200 import engine, ops
    B = len(nroi)
    cp, pb, num = dev(prob), dev(pred), dev(np.asarray(nroi, np.int32))
    gd, det = S.guarded_out((B, max_det, 6), float("nan"))
    gn, ndet = guarded_int((B,))
    gk, keep = guarded_int((B, C, r))
    gc, cnt = guarded_int((B, C))
    gs, ks = S.guarded_out((B, C, r), float("nan"))
    gv, vb = S.guarded_out((B, C, r, 4), float("nan"))
    v = None if vote is None else (*engine.box_vote_args(*vote), vb)
    if soft is None:
        t32, flags = engine.nms_threshold(0.3, True)
        ops.detect_post(cp, pb, num, C, thresh, t32, flags, mpi, det, ndet, keep, cnt, ks, ops.detect_post_workspace(r, C, B), B, vote=v)
    else:
        code, s32, p32 = engine.soft_nms_args(*soft)
        ops.detect_post_soft(cp, pb, num, C, thresh, code, s32, float(F(0.3)), p32, mpi, det, ndet, keep, cnt, ks, B, vote=v)
    torch.cuda.synchronize()
    for g, t, what in ((gd, det, "det"), (gn, ndet, "ndet"), (gk, keep, "keep"), (gc, cnt, "keep_cnt"), (gs, ks, "keep_score"),
                       (gv, vb, "vote_box")):
        S.check_guarded(g, t.numel(), what)
    unchanged(cp, prob, "cls_prob"); unchanged(pb, pred, "pred_boxes"); unchanged(num, np.asarray(nroi, np.int32), "num_rois")
    return det.cpu().numpy(), ndet.cpu().numpy(), keep.cpu().numpy(), cnt.cpu().numpy(), ks.cpu().numpy()


def check_post(res, prob, pred, r, C, nroi, soft, vote, mpi, max_det, thresh=0.0):
    """Each image against the oracle on its valid rows (count clamped to [0, r]): the TRUE record count, the first
    min(count, max_det) records, keep / keep_cnt of every class after the cap (-1 past the count), and keep_score: the class
    stage's whole list before the cap (the cap shortens keep and keep_cnt, not keep_score), +0 past it -> the per-image counts."""
    det, nd, keep, cnt, ks = res
    counts = []

    def oracle(p, x, cap):
        if vote is None:
            return SO.test_net_post_soft(p, x, soft, 0.3, cap, thresh)
        return BV.test_net_post_vote(p, x, vote, 0.3, cap, thresh, soft=soft)
    for b, n in enumerate(nroi):
        n = min(max(n, 0), r)
        p, x = prob[b * r:b * r + n], pred[b * r:b * r + n]
        out, idx = oracle(p, x, mpi)
        whole = oracle(p, x, 0)[0] if mpi > 0 else out
        want = S.flat_records(out)
        assert nd[b] == want.shape[0], "image %d: %d records, want %d" % (b, nd[b], want.shape[0])
        k = min(int(nd[b]), max_det)
        same_bits(det[b, :k], want[:k], "image %d records" % b)
        for j in range(C):
            c = int(cnt[b, j])
            assert c == idx[j].shape[0] and np.array_equal(keep[b, j, :c], idx[j]), (b, j)
            assert (keep[b, j, c:] == -1).all(), (b, j)
            w = whole[j].shape[0]
            same_bits(ks[b, j, :w], whole[j][:, 4], "image %d class %d keep_score" % (b, j))
            assert (ks[b, j, w:].view(np.int32) == 0).all(), "image %d class %d: keep_score past the list is not +0" % (b, j)
        counts.append(want.shape[0])
    return counts


SOFTS = [("linear", 0.5, 0.001), ("gaussian", 0.5, 0.001), ("hard", 0.5, 0.001)]


@pytest.mark.parametrize("C", [2, 1024])
@pytest.mark.parametrize("r", [1024, 1025])
def test_soft_post_capacity_boundary(cuda, r, C):
    """r = 1024 is the last size of the 256 x 4 kernel, 1025 the first of the 1024 x 8 one; C = 2 and 1024 the class limits.
    Batch 3 with num_rois -1, r + 5 (clamped to r) and a partial count; quantised probabilities tie within classes and at the
    100th record score."""
    rng = np.random.default_rng(r * 7 + C)
    nroi = [-1, r + 5, r // 3]
    prob = S.quantised_probs(rng, 3 * r, C, weights=S.SPARSE_TOP)
    pred = np.vstack([S.clustered_pred(rng, r, C) for _ in range(3)])
    for k, soft in enumerate(SOFTS):
        mpi = (100, 0, 100)[k]
        max_det = 2 * 100 + 56 if mpi else r * (C - 1)
        res = post(prob, pred, r, C, nroi, soft, None, mpi, max_det)
        counts = check_post(res, prob, pred, r, C, nroi, soft, None, mpi, max_det)
        assert counts[0] == 0 and counts[1] > 0, (soft, counts)


def test_soft_post_zero_rois_and_ties_at_the_cap(cuda):
    """num_rois 0; 60 records above the 100th score and 80 tied at it (all 140 kept)."""
    rng = np.random.default_rng(140)
    r, C = 300, 81
    prob = np.vstack([S.cap_tie_probs(rng, r, C, 60, 80), S.cap_tie_probs(rng, r, C, 60, 80)])
    pred = np.vstack([S.grid_pred(r, C)] * 2)
    res = post(prob, pred, r, C, [0, r], SOFTS[0], None, 100, 256)
    assert check_post(res, prob, pred, r, C, [0, r], SOFTS[0], None, 100, 256) == [0, 140]


def test_soft_post_ties_past_max_det(cuda):
    """Ties push the true count (360) past max_det (256): ndet reports 360, the first 256 rows are the oracle's, nothing is
    stored past row 256 (guard band) and the host refuses the record."""
    from tf_faster_rcnn_b200 import engine
    rng = np.random.default_rng(360)
    r, C, max_det = 300, 81, 256
    prob, pred = S.cap_tie_probs(rng, r, C, 60, 300), S.grid_pred(r, C)
    res = post(prob, pred, r, C, [r], SOFTS[1], None, 100, max_det)
    assert check_post(res, prob, pred, r, C, [r], SOFTS[1], None, 100, max_det) == [360]
    host = torch.zeros((1, engine.REC_HEADER + max_det * 6), dtype=torch.float32)
    host[0, engine.REC_HEADER:] = torch.from_numpy(res[0][0].reshape(-1))
    host.view(torch.int32)[0, 0] = int(res[1][0])
    with pytest.raises(RuntimeError, match="360 detections"):
        engine.split_host_records(host, max_det)


VOTE_EDGES = [(1.0, "AVG", 1.0),                  # only exact duplicates (IoU 1) vote
              (0.6, "QUASI_SUM", 0.7),            # n^beta through pow
              (0.5, "TEMP_AVG", 0.5),
              (0.5, "GENERALIZED_AVG", 1000.0),   # exp(beta * s) overflows: voted score +Inf, re-sorted first
              (0.8, "ID", 1.0)]


@pytest.mark.parametrize("C", [2, 1024])
@pytest.mark.parametrize("r", [1024, 1025])
def test_vote_posts_capacity_boundary(cuda, r, C):
    """Voting behind greedy NMS and behind Soft-NMS at the same boundaries; probabilities 0.5 and 1 exactly (TEMP_AVG's
    log(0) edge for s = 1), exact duplicate boxes for VOTE_TH = 1."""
    rng = np.random.default_rng(r * 3 + C)
    nroi = [r + 5, r // 2]
    prob = S.quantised_probs(rng, 2 * r, C, levels=(0.0, 0.25, 0.5, 0.75, 1.0), weights=(0.6, 0.1, 0.1, 0.1, 0.1))
    pred = np.vstack([S.clustered_pred(rng, r, C) for _ in range(2)])
    dup = rng.integers(0, 2 * r, (2 * r) // 4)
    pred[dup] = pred[rng.integers(0, 2 * r, dup.shape[0])]      # exact duplicate rows (boxes of every class)
    for k, vote in enumerate(VOTE_EDGES):
        soft = (None, SOFTS[k % 3])[k % 2]
        mpi = 100 if k != 2 else 0
        max_det = 256 if mpi else r * (C - 1)
        res = post(prob, pred, r, C, nroi, soft, vote, mpi, max_det)
        counts = check_post(res, prob, pred, r, C, nroi, soft, vote, mpi, max_det)
        assert counts[0] > 0, (vote, soft)
        if vote[1] == "GENERALIZED_AVG":
            assert np.isposinf(res[0][0, :min(counts[0], max_det), 4]).any()


def test_vote_set_temp_avg_scores_zero_half_one(cuda):
    """frcnn_box_vote_host with candidate scores exactly 0, 0.5 and 1 (TEMP_AVG's log(0) on both sides)."""
    from tf_faster_rcnn_b200 import ops, _native as N
    box = [10, 10, 40, 40]
    a = np.array([box + [0.0], box + [0.5], box + [1.0], [12, 10, 40, 40, 0.5], [500, 500, 520, 520, 0.0]], F)
    top = a[[2, 1, 4]].copy()
    for beta in (0.5, 1.0, 3.0):
        got = ops.box_vote_host(top, a, 0.5, N.BOX_VOTE_METHODS["TEMP_AVG"], beta)
        same_bits(got, BV.box_vote_c(top, a, 0.5, "TEMP_AVG", beta), "TEMP_AVG beta %g" % beta)


# ---- test-time augmentation union ----------------------------------------------------------------------------------------
def test_aug_union_edges_then_soft_post(cuda):
    """16 views (FRCNN_AUG_MAX_VIEWS) of 512 rows: R_union = 8192.  Image 0: counts -3, 0 (between non-empty views), above the
    rows and partial, mirrored boxes at x = 0, W - 1 and +-Inf; image 1: every view empty.  The union against the numpy model,
    then detect_post_soft on it against the oracle."""
    from tf_faster_rcnn_b200 import _native as N, ops
    rng = np.random.default_rng(16)
    nv, rv, B, C = N.AUG_MAX_VIEWS, 512, 2, 21
    flips = [v % 2 == 1 for v in range(nv)]
    probs = [S.quantised_probs(rng, B * rv, C, weights=S.SPARSE_TOP).reshape(B, rv, C) for _ in range(nv)]
    boxes = [np.vstack([S.clustered_pred(rng, rv, C) for _ in range(B)]).reshape(B, rv, 4 * C) for _ in range(nv)]
    orig_w = [800.0, 333.0]
    for v in range(1, nv, 2):                        # mirrored views: edge x coordinates in the first rows
        b = boxes[v][0].reshape(rv, C, 4)
        b[0, :, 0], b[0, :, 2] = 0, orig_w[0] - 1
        b[1, :, 0], b[1, :, 2] = -np.inf, np.inf
        b[2, :, 0], b[2, :, 2] = np.inf, np.inf
    c0 = [200, 0, rv + 7, -3, 37, rv, 1, 0, 90, 300, 0, 12, rv + 1, 5, 64, 111]
    c1 = [0, -3, 0, 0, -1, 0, 0, 0, -3, 0, 0, 0, 0, 0, 0, 0]
    counts = [np.array([c0[v], c1[v]], np.int32) for v in range(nv)]
    devs = [(dev(p), dev(q), dev(c)) for p, q, c in zip(probs, boxes, counts)]
    meta_np = np.array([[1.0, 600.0, w] for w in orig_w], F)
    meta = dev(meta_np)
    ru = nv * rv
    gp, up = S.guarded_out((B, ru, C))
    gb, ub = S.guarded_out((B, ru, 4 * C))
    gn, num = guarded_int((B,))
    ops.aug_union([(p.data_ptr(), q.data_ptr(), c.data_ptr(), rv, f) for (p, q, c), f in zip(devs, flips)], C, meta.data_ptr(), up, ub,
                  num)
    torch.cuda.synchronize()
    S.check_guarded(gp, up.numel(), "union cls_prob"); S.check_guarded(gb, ub.numel(), "union pred_boxes")
    S.check_guarded(gn, num.numel(), "union num_rois")
    for (p, q, c), a, bx, cn in zip(devs, probs, boxes, counts):
        unchanged(p, a, "view cls_prob"); unchanged(q, bx, "view pred_boxes"); unchanged(c, cn, "view num_rois")
    unchanged(meta, meta_np, "im_meta")
    with np.errstate(invalid="ignore"):
        wp, wb, wn = AO.union_model(probs, boxes, counts, flips, orig_w)
    assert num.cpu().numpy().tolist() == wn.tolist() and wn[1] == 0
    same_bits(up.cpu().numpy(), wp, "union cls_prob")
    same_bits(ub.cpu().numpy(), wb, "union pred_boxes")
    # the union straight into the Soft-NMS post at R_union = 8192
    prob, pred, nroi = wp.reshape(B * ru, C), wb.reshape(B * ru, 4 * C), wn.tolist()
    for soft in (SOFTS[0], SOFTS[2]):
        res = post(prob, pred, ru, C, nroi, soft, None, 100, 256)
        counts_ = check_post(res, prob, pred, ru, C, nroi, soft, None, 100, 256)
        assert counts_[0] >= 100 and counts_[1] == 0


# ---- boxes_to_rois -------------------------------------------------------------------------------------------------------
def test_boxes_to_rois_edges(cuda):
    """Counts -3, 0, cap and cap + 5 (clamped), a scale that is not a power of two, NaN and +-Inf boxes passed through
    unclipped, and zero rows past each count."""
    from tf_faster_rcnn_b200 import ops
    rng = np.random.default_rng(5)
    B, cap = 4, 37
    boxes = rng.uniform(-50, 900, (B, cap, 4)).astype(F)
    boxes[:, 3] = [np.nan, 1.0, np.inf, -np.inf]
    boxes[:, 5, 0] = -np.inf
    counts = np.array([-3, 0, cap, cap + 5], np.int32)
    scales = [0.6, 1.7, 0.6, 1.3333334]
    meta_np = np.array([[s, 600.0, 800.0] for s in scales], F)
    bd, cd, md = dev(boxes), dev(counts), dev(meta_np)
    gr, rois = S.guarded_out((B * cap, 5))
    gn, num = guarded_int((B,))
    ops.boxes_to_rois(bd, cd, md, rois, num)
    torch.cuda.synchronize()
    S.check_guarded(gr, rois.numel(), "rois"); S.check_guarded(gn, num.numel(), "num_rois")
    unchanged(bd, boxes, "boxes"); unchanged(cd, counts, "counts"); unchanged(md, meta_np, "im_meta")
    want = np.zeros((B, cap, 5), F)
    n = np.clip(counts, 0, cap)
    for b in range(B):
        want[b, :n[b], 0] = b
        want[b, :n[b], 1:] = boxes[b, :n[b]] * meta_np[b, 0]
    assert num.cpu().numpy().tolist() == n.tolist()
    same_bits(rois.cpu().numpy(), want.reshape(B * cap, 5), "rois")
    assert np.isnan(want[2, 3, 1]) and np.isposinf(want[2, 3, 3]) and np.isneginf(want[2, 3, 4]) and np.isneginf(want[2, 5, 1])


# ---- detect_features -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fdim", [4, 4100])
@pytest.mark.parametrize("C", [2, 1024])
def test_detect_features_edges(cuda, C, fdim):
    """post_ref64.features_case, batch 3: empty classes at 1, in the middle and at C - 1; one image's total above every
    max_det and totals of 5 and 12 that end inside an 8-slot block and before max_det 7 / 8 / 9 / 100; class 0 holding a count
    it never emits.  keep holds valid RoI rows past every count, so a read past a count would show as a feature row where the
    reference has -1 and zeros (tests/test_post_ref64.py shows that for `slot <= total`)."""
    from tf_faster_rcnn_b200 import ops
    rng = np.random.default_rng(C + fdim)
    keep, cnt = R.features_case(rng, C)
    B, _, r = keep.shape
    totals = cnt[:, 1:].sum(1)
    assert sorted(totals.tolist())[:2] == ([0, 5] if C == 2 else [5, 12]) and totals.max() >= 12
    fc7 = rng.standard_normal((B * r, fdim)).astype(F)
    kd, cd, fd = dev(keep), dev(cnt), dev(fc7)
    for max_det in (1, 7, 8, 9, 100):
        gf, feat = S.guarded_out((B, max_det, fdim))
        gr, roi = guarded_int((B, max_det))
        ops.detect_features(kd, cd, fd, C, feat, roi)
        torch.cuda.synchronize()
        S.check_guarded(gf, feat.numel(), "features"); S.check_guarded(gr, roi.numel(), "roi_out")
        wf, wr = R.features_ref(keep, cnt, fc7, max_det)
        assert np.array_equal(roi.cpu().numpy(), wr), max_det
        same_bits(feat.cpu().numpy(), wf, "features max_det %d" % max_det)
    unchanged(kd, keep, "keep"); unchanged(cd, cnt, "keep_cnt"); unchanged(fd, fc7, "fc7")
