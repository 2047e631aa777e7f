"""The detection-tail kernels at their edges, through the C ABI, against the oracle and float64 references (stage_ref64.py).

* value for value (the kernels claim the oracle's fp32 op order): rpn_decode proposals, cls_score, the de-normalised deltas,
  bbox_decode, crop_pool, and the per-class NMS + cap records;
* within a derived per-element bound of a float64 truth: the two softmaxes and the spatial mean (max err / bound printed).
Every output sits between sentinel guard bands and every input is checked unchanged afterwards."""
import numpy as np
import pytest
import torch

from oracle import anchors as OA
from oracle import layers as L
from oracle import nms as ONMS
from oracle import pipeline as P
import stage_ref64 as S

pytestmark = pytest.mark.gpu
F = np.float32


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def unchanged(d, a, what):
    assert np.array_equal(d.cpu().numpy(), a, equal_nan=True), "%s was modified" % what


def blob_feat(h, w):
    return -(-h // 16), -(-w // 16)


# ---- rpn_decode ----------------------------------------------------------------------------------------------------------
def rpn_inputs(rng, B, A, fh, fw, deltas):
    """fused RPN head rows [B*fh*fw, ld] (bg | fg logits, pad, deltas at dcol) and the per-image oracle tensors."""
    dcol = (2 * A + 3) // 4 * 4
    ld = (dcol + 4 * A + 3) // 4 * 4
    x, _ = S.logit_rows(rng, B * fh * fw * A, 2)
    cls = np.concatenate([x[:, 0].reshape(B, fh, fw, A), x[:, 1].reshape(B, fh, fw, A)], axis=3)
    box = deltas.reshape(B, fh, fw, 4 * A)
    fused = np.full((B * fh * fw, ld), np.nan, F)
    fused[:, :2 * A] = cls.reshape(-1, 2 * A)
    fused[:, dcol:dcol + 4 * A] = box.reshape(-1, 4 * A)
    return fused, dcol, cls, box


def run_rpn_decode(fused, dcol, scales, A, B, fh, fw, im_h, im_w):
    from tf_faster_rcnn_b200 import ops
    n = B * fh * fw * A
    base = OA.base_anchors(ratios=(0.5, 1, 2), scales=scales).astype(F)
    fd, bd = dev(fused), dev(base)
    sbuf, scores = S.guarded_out((n,))
    pbuf, props = S.guarded_out((n, 4))
    ops.rpn_decode(fd, dcol, bd, A, fh, fw, im_h, im_w, scores, props, batch=B)
    S.check_guarded(sbuf, n, "scores")
    S.check_guarded(pbuf, 4 * n, "proposals")
    unchanged(fd, fused, "rpn head")
    unchanged(bd, base, "base anchors")
    return scores.cpu().numpy().reshape(B, -1), props.cpu().numpy().reshape(B, -1, 4)


@pytest.mark.parametrize("scales,hw,B", [((8, 16, 32), (601, 799), 1), ((8, 16, 32), (601, 799), 3), ((4, 8, 16, 32), (361, 491), 1),
                                         ((2, 4, 8, 16, 32), (600, 1000), 3)])
def test_rpn_decode_edges(cuda, scales, hw, B):
    A = 3 * len(scales)
    fh, fw = blob_feat(*hw)
    assert (fh * fw * A) % 256
    rng = np.random.default_rng(A * 10 + B)
    fused, dcol, cls, box = rpn_inputs(rng, B, A, fh, fw, S.edge_deltas(rng, B * fh * fw * A, 1))
    scores, props = run_rpn_decode(fused, dcol, scales, A, B, fh, fw, *hw)
    worst = 0.0
    for b in range(B):
        with np.errstate(over="ignore", invalid="ignore"):
            _, want, _ = P.rpn_decode(cls[b:b + 1], box[b:b + 1], np.array([hw[0], hw[1], 1.0], F), P.opts(anchor_scales=scales))
        nan = S.check_boxes_exact(props[b], want, "proposals image %d" % b)
        assert not nan.any()
        p64, bound = S.rpn_fg_ref(cls[b, ..., :A].reshape(-1), cls[b, ..., A:].reshape(-1))
        worst = max(worst, S.check_bounded(scores[b], p64, bound, "fg score image %d" % b))
    print("\n[rpn_decode A=%d %dx%d B=%d] fg score max err/bound %.3f" % (A, hw[0], hw[1], B, worst))


def test_decode_nan_clip(cuda):
    """inf - inf in the decode: numpy propagates the NaN through the clip, the kernels' fminf / fmaxf return the bound.
    The device result is pinned here (DESIGN §2): rpn_decode (two-sided clip) gives (W-1, H-1, W-1, H-1) for x1 = NaN,
    x2 = +inf and (0, 0, W-1, H-1) for x1 = -inf, x2 = NaN; bbox_decode (one-sided) gives (0, 0, W-1, H-1) for both."""
    from tf_faster_rcnn_b200 import ops
    A, fh, fw, H, W = 9, 2, 3, 32, 48
    rng = np.random.default_rng(0)
    fused, dcol, cls, box = rpn_inputs(rng, 1, A, fh, fw, S.nan_deltas(fh * fw * A, 1))
    _, props = run_rpn_decode(fused, dcol, (8, 16, 32), A, 1, fh, fw, H, W)
    with np.errstate(over="ignore", invalid="ignore"):
        _, want, _ = P.rpn_decode(cls, box, np.array([H, W, 1.0], F), P.opts())
    assert np.isnan(want).any(axis=1).all()
    even = np.arange(fh * fw * A) % 2 == 0
    assert (props[0][even] == [W - 1, H - 1, W - 1, H - 1]).all()
    assert (props[0][~even] == [0, 0, W - 1, H - 1]).all()
    R, C = 6, 3
    rois = np.hstack([np.zeros((R, 1)), np.tile([10, 20, 60, 90], (R, 1))]).astype(F)
    buf, pred = S.guarded_out((R, 4 * C))
    ops.bbox_decode(dev(rois), dev(S.nan_deltas(R, C)), C, ops.im_meta_tensor([(1.0, H, W)]), pred)
    S.check_guarded(buf, R * 4 * C)
    assert (pred.cpu().numpy().reshape(-1, 4) == [0, 0, W - 1, H - 1]).all()


# ---- cls_finish ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("r", [1, 7, 9, 300, 1001])
@pytest.mark.parametrize("C", [2, 5, 21, 31, 32, 33, 81, 1024])
def test_cls_finish_edges(cuda, C, r):
    """The production head stride ld = ceil(5C/4)*4 with NaN in the pad columns; every logit row kind; distinct stds and
    non-zero means."""
    from tf_faster_rcnn_b200 import ops
    rng = np.random.default_rng(C * 7 + r)
    ld = -(-5 * C // 4) * 4
    logits, kind = S.logit_rows(rng, r, C, S.ROW_KINDS[r % len(S.ROW_KINDS):] + S.ROW_KINDS[:r % len(S.ROW_KINDS)])
    deltas = S.edge_deltas(rng, r, C)
    head = np.full((r, ld), np.nan, F)
    head[:, :C] = logits
    head[:, C:5 * C] = deltas
    hd = dev(head)
    b1, cs = S.guarded_out((r, C))
    b2, cp = S.guarded_out((r, C))
    b3, bp = S.guarded_out((r, 4 * C))
    ops.cls_finish(hd, C, S.BBOX_STDS, S.BBOX_MEANS, cs, cp, bp)
    for b, t, w in ((b1, cs, "cls_score"), (b2, cp, "cls_prob"), (b3, bp, "bbox_pred")):
        S.check_guarded(b, t.numel(), w)
    unchanged(hd, head, "head")
    S.check_exact(cs.cpu().numpy(), logits, "cls_score")
    S.check_exact(bp.cpu().numpy(), S.denorm_ref(deltas, S.BBOX_STDS, S.BBOX_MEANS), "bbox_pred")
    p64, bound = S.softmax_ref(logits, S.cls_depth(C))
    got = cp.cpu().numpy()
    worst = S.check_bounded(got, p64, bound, "cls_prob")
    per_kind = ["%s %.3f" % (S.ROW_KINDS[(k + r) % len(S.ROW_KINDS)], (np.abs(got[kind == k] - p64[kind == k]) / bound[kind == k]).max())
                for k in range(min(r, len(S.ROW_KINDS)))]
    print("\n[cls_finish C=%d r=%d] cls_prob max err/bound %.3f (%s)" % (C, r, worst, ", ".join(per_kind)))


# ---- bbox_decode ---------------------------------------------------------------------------------------------------------
def decode_rois(rng, R, B, blob_hw=(600, 800)):
    xy = rng.uniform(-50, 1, (R, 2)) + rng.uniform(0, 1, (R, 2)) * (blob_hw[1], blob_hw[0])
    img = rng.integers(0, B, R) if B > 1 else np.zeros(R)
    return np.hstack([img[:, None], xy, xy + rng.uniform(4, 400, (R, 2))]).astype(F)


def run_bbox_decode(rois, deltas, C, meta):
    from tf_faster_rcnn_b200 import ops
    rd, dd = dev(rois), dev(deltas)
    buf, pred = S.guarded_out(deltas.shape)
    ops.bbox_decode(rd, dd, C, ops.im_meta_tensor(meta), pred)
    S.check_guarded(buf, pred.numel())
    unchanged(rd, rois, "rois")
    unchanged(dd, deltas, "deltas")
    return pred.cpu().numpy()


def check_decode_per_image(got, rois, deltas, C, meta):
    reached = np.zeros(2, bool)
    for b, (scale, h, w) in enumerate(meta):
        rows = rois[:, 0] == b
        with np.errstate(over="ignore", invalid="ignore"):
            _, want = P.im_detect_post(rois[rows], np.zeros((int(rows.sum()), C), F), deltas[rows], scale, h, w)
        assert not S.check_boxes_exact(got[rows], want, "bbox_decode image %d" % b).any()
        wb = want.reshape(-1, 4)
        reached |= [(wb[:, 0] > w - 1).any(), (wb[:, 2] < 0).any()]
    assert reached.all(), "no box decoded past a side the one-sided clip leaves open"


@pytest.mark.parametrize("scale", [1.6, 600 / 720, 2.4])
@pytest.mark.parametrize("C", [2, 21, 81])
def test_bbox_decode_edges(cuda, C, scale):
    R = 301
    assert (R * C) % 256
    rng = np.random.default_rng(C + int(scale * 10))
    rois = decode_rois(rng, R, 1)
    deltas = S.edge_deltas(rng, R, C)
    meta = [(scale, int(600 / scale), int(800 / scale))]
    check_decode_per_image(run_bbox_decode(rois, deltas, C, meta), rois, deltas, C, meta)


def test_bbox_decode_batch_meta_rows(cuda):
    """Three images with three different im_meta rows, RoI rows of the images interleaved; each image vs the oracle."""
    C, R = 21, 613
    rng = np.random.default_rng(3)
    rois = decode_rois(rng, R, 3)
    deltas = S.edge_deltas(rng, R, C)
    meta = [(1.6, 375, 500), (600 / 720, 720, 960), (2.4, 250, 333)]
    assert len(set(rois[:, 0].tolist())) == 3
    check_decode_per_image(run_bbox_decode(rois, deltas, C, meta), rois, deltas, C, meta)


# ---- crop_pool -----------------------------------------------------------------------------------------------------------
def crop_want(feat_b, rois, pre_pool):
    nb = P.roi_norm_boxes(feat_b.shape, rois)
    if pre_pool:
        return L.max_pool(L.crop_and_resize(feat_b, nb, 14), 2, 2, "SAME")
    return L.crop_and_resize(feat_b, nb, 7)


def run_crop(feat, rois, pre_pool):
    from tf_faster_rcnn_b200 import ops
    fd, rd = dev(feat), dev(rois)
    buf, out = S.guarded_out((rois.shape[0], 7, 7, feat.shape[3]))
    ops.crop_pool(fd, rd, 7, pre_pool, out)
    S.check_guarded(buf, out.numel())
    unchanged(fd, feat, "feature map")
    unchanged(rd, rois, "rois")
    return out.cpu().numpy()


@pytest.mark.parametrize("fhw", [(38, 50), (2, 3)])
@pytest.mark.parametrize("pre_pool", [0, 1])
@pytest.mark.parametrize("C", [64, 512, 1024])
def test_crop_pool_edges(cuda, C, pre_pool, fhw):
    """Boxes straddling and outside every side (extrapolation to 0), inverted, zero-size and last-sample-on-the-edge boxes;
    C = 512 / 1024 run the channel loop more than once per thread."""
    fh, fw = fhw
    rng = np.random.default_rng(C + pre_pool + fh)
    feat = rng.standard_normal((1, fh, fw, C)).astype(F)
    n = 45
    rois = np.hstack([np.zeros((n, 1), F), S.crop_boxes(rng, fh, fw, n, 14 if pre_pool else 7)])
    S.check_exact(run_crop(feat, rois, pre_pool), crop_want(feat, rois, pre_pool), "crop_pool")


@pytest.mark.parametrize("pre_pool", [0, 1])
def test_crop_pool_batch_and_image_clamp(cuda, pre_pool):
    """Batch 3, RoI column 0 mixed over {0, 1, 2}; out-of-range indices clamp: -1 -> image 0, 5 -> image 2."""
    B, fh, fw, C, n = 3, 19, 27, 512, 64
    rng = np.random.default_rng(30 + pre_pool)
    feat = rng.standard_normal((B, fh, fw, C)).astype(F)
    col0 = rng.integers(0, B, n).astype(F)
    col0[:4] = [-1, 5, -1, 5]
    rois = np.hstack([col0[:, None], S.crop_boxes(rng, fh, fw, n, 14 if pre_pool else 7)]).astype(F)
    got = run_crop(feat, rois, pre_pool)
    img = np.where(col0 == -1, 0, np.where(col0 == 5, 2, col0)).astype(int)
    for b in range(B):
        rows = img == b
        S.check_exact(got[rows], crop_want(feat[b:b + 1], rois[rows], pre_pool), "crop_pool image %d" % b)


# ---- spatial_mean --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("data", ["normal", "offset", "cancel"])
@pytest.mark.parametrize("C", [256, 2048])
@pytest.mark.parametrize("side", [1, 7, 14])
def test_spatial_mean_bound(cuda, side, C, data):
    """N(0,1); 1e4 + N(0,1) (the sum's rounding error is large, the bound binds); +1e4 over the first half of the
    positions and -1e4 over the rest, + N(0,1) (cancellation: the partial sums climb to hw/2 * 1e4 and round, the mean
    ends up small next to sum|x|).  hw = 1 is exact."""
    from tf_faster_rcnn_b200 import ops
    rng = np.random.default_rng(side * C)
    x = rng.standard_normal((9, side, side, C))
    if data == "offset":
        x += 1e4
    elif data == "cancel":
        x += np.where(np.arange(side * side).reshape(1, side, side, 1) < side * side // 2, 1e4, -1e4)
    x = x.astype(F)
    xd = dev(x)
    buf, out = S.guarded_out((9, C))
    ops.spatial_mean(xd, out)
    S.check_guarded(buf, out.numel())
    unchanged(xd, x, "input")
    m64, bound = S.spatial_mean_ref(x)
    r = S.check_bounded(out.cpu().numpy(), m64, bound, "spatial_mean")
    print("\n[spatial_mean hw=%d C=%d %s] max err/bound %.3f" % (side * side, C, data, r))


# ---- detect_post ---------------------------------------------------------------------------------------------------------
def run_post(probs, pred, nrois, C, max_det, gpu_pred=False, mpi=100, score_thresh=0.0):
    """frcnn_detect_post on B = len(nrois) images of R rows each -> (det [B, max_det, 6], ndet [B], keep_cnt [B, C])."""
    from tf_faster_rcnn_b200 import ops, _native as N
    B = len(nrois)
    R = probs.shape[0] // B
    buf, det = S.guarded_out((B, max_det, 6))
    ndet = torch.full((B,), -1, dtype=torch.int32, device="cuda")
    keep = torch.empty((B, C, R), dtype=torch.int32, device="cuda")
    cnt = torch.empty((B, C), dtype=torch.int32, device="cuda")
    ks = torch.empty((B, C, R), dtype=torch.float32, device="cuda")
    pd, bd, nd = dev(probs), dev(pred), dev(np.asarray(nrois, np.int32))
    flags = N.NMS_MODE_GPU_NMS if gpu_pred else N.NMS_MODE_CPU_NMS
    thr = float(ONMS.thresh_f32(0.3, inclusive=not gpu_pred))
    ops.detect_post(pd, bd, nd, C, float(F(score_thresh)), thr, flags, mpi, det, ndet, keep, cnt, ks,
                    workspace=ops.detect_post_workspace(R, C, B) if R > 1024 else None, batch=B)
    S.check_guarded(buf, det.numel(), "record buffer")
    unchanged(pd, probs, "cls_prob")
    unchanged(bd, pred, "pred_boxes")
    return det.cpu().numpy(), ndet.cpu().numpy(), cnt.cpu().numpy()


def post_case(probs, pred, C, nrois=None, max_det=None, gpu_pred=False, mpi=100, score_thresh=0.0):
    """Run the device post and compare every image with the oracle's test_net_post; -> the oracle's per-image counts."""
    R = pred.shape[0] // (len(nrois) if nrois else 1)
    nrois = nrois or [R]
    max_det = max_det or R * (C - 1)
    det, nd, cnt = run_post(probs, pred, nrois, C, max_det, gpu_pred, mpi, score_thresh)
    o = P.opts(use_gpu_nms=gpu_pred, max_per_image=mpi)
    counts = []
    for b, n in enumerate(nrois):
        want = P.test_net_post(probs[b * R:b * R + n], pred[b * R:b * R + n], o, thresh=F(score_thresh))
        S.check_records(det[b], int(nd[b]), cnt[b], want, max_det, "image %d" % b)
        counts.append(sum(d.shape[0] for d in want))
    return counts, det, nd


@pytest.mark.parametrize("gpu_pred", [False, True])
@pytest.mark.parametrize("R,C", [(300, 21), (300, 81), (1000, 21)])
def test_detect_post_quantised_ties(cuda, R, C, gpu_pred):
    """Quantised probabilities over overlapping boxes: per-class ties resolve by RoI index (score desc, index asc)."""
    rng = np.random.default_rng(R + C + gpu_pred)
    probs, pred = S.quantised_probs(rng, R, C, weights=S.SPARSE_TOP), S.clustered_pred(rng, R, C)
    counts, _, _ = post_case(probs, pred, C, gpu_pred=gpu_pred)
    assert counts[0] > 100


def test_detect_post_cap_tie_within_max_det(cuda):
    """60 records above the 100th score and 80 tied at it: all 140 are kept (ties kept, as test.py), within max_det."""
    rng = np.random.default_rng(140)
    R, C, mpi = 300, 81, 100
    counts, _, _ = post_case(S.cap_tie_probs(rng, R, C, 60, 80), S.grid_pred(R, C), C, max_det=2 * mpi + 56, mpi=mpi)
    assert counts == [140]


def test_detect_post_cap_tie_overflow(cuda):
    """Ties push the true count (360) past max_det (256): ndet reports 360, the first 256 rows are the oracle's, nothing is
    stored past row 256 (guard band) and the host refuses the record."""
    from tf_faster_rcnn_b200 import engine
    rng = np.random.default_rng(360)
    R, C, mpi = 300, 81, 100
    max_det = 2 * mpi + 56
    counts, det, nd = post_case(S.cap_tie_probs(rng, R, C, 60, 300), S.grid_pred(R, C), C, max_det=max_det, mpi=mpi)
    assert counts == [360] and int(nd[0]) == 360
    host = torch.zeros((1, engine.REC_HEADER + max_det * 6), dtype=torch.float32)
    host[0, engine.REC_HEADER:] = torch.from_numpy(det[0].reshape(-1))
    host.view(torch.int32)[0, 0] = int(nd[0])
    with pytest.raises(RuntimeError, match="360 detections"):
        engine.split_host_records(host, max_det)


@pytest.mark.parametrize("gpu_pred", [False, True])
def test_detect_post_batch_partial_counts(cuda, gpu_pred):
    """Batch 3 with num_rois = (0, 137, R); the rows past each count hold large finite garbage that must never be read."""
    rng = np.random.default_rng(137 + gpu_pred)
    R, C, nrois = 300, 21, [0, 137, 300]
    probs = S.quantised_probs(rng, 3 * R, C, weights=S.SPARSE_TOP)
    pred = np.vstack([S.clustered_pred(rng, R, C) for _ in range(3)])
    for b, n in enumerate(nrois):
        probs[b * R + n:(b + 1) * R] = F(1e30)
        pred[b * R + n:(b + 1) * R] = rng.choice([F(-1e30), F(1e30)], pred[b * R + n:(b + 1) * R].shape)
    counts, _, nd = post_case(probs, pred, C, nrois=nrois, gpu_pred=gpu_pred)
    assert counts[0] == 0 and int(nd[0]) == 0 and counts[1] > 0 and counts[2] > 0


@pytest.mark.parametrize("C", [2, 1024])
def test_detect_post_class_limits(cuda, C):
    """The ABI's class limits: one foreground class, and 1023 (one thread per class in the cap kernel)."""
    rng = np.random.default_rng(C)
    R = 300
    counts, _, _ = post_case(S.quantised_probs(rng, R, C, weights=S.SPARSE_TOP), S.clustered_pred(rng, R, C), C)
    assert counts[0] > (100 if C > 2 else 0)


def test_detect_post_no_cap(cuda):
    """max_per_image = 0: no cap at all."""
    rng = np.random.default_rng(0)
    R, C = 300, 21
    counts, _, _ = post_case(S.quantised_probs(rng, R, C), S.clustered_pred(rng, R, C), C, mpi=0)
    assert counts[0] > 100


def test_detect_post_score_thresh_strict(cuda):
    """score_thresh = 0.05 with probabilities exactly fp32(0.05) (not candidates: `>` is strict) and one ulp above (are)."""
    rng = np.random.default_rng(5)
    R, C = 300, 21
    t = F(0.05)
    levels = (0.0, t, np.nextafter(t, F(1)), 0.125, 0.5)
    probs = S.quantised_probs(rng, R, C, levels=levels, weights=(0.3, 0.3, 0.2, 0.15, 0.05))
    counts, det, nd = post_case(probs, S.clustered_pred(rng, R, C), C, mpi=0, score_thresh=0.05)
    rec = det[0][:int(nd[0])]
    assert (rec[:, 4] > t).all() and (rec[:, 4] == np.nextafter(t, F(1))).any()


def test_detect_post_top_mode_ties(cuda):
    """TEST.MODE 'top': 5000 RoIs per image, the kept sets in the global workspace, with quantised ties."""
    rng = np.random.default_rng(5000)
    R, C = 5000, 21
    counts, _, _ = post_case(S.quantised_probs(rng, R, C, weights=S.SPARSE_TOP), S.clustered_pred(rng, R, C), C)
    assert counts[0] > 100
