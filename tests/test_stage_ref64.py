"""The comparators of stage_ref64.py have teeth: a numpy model of each kernel's fp32 op order passes its comparator (the
softmaxes with expf perturbed by up to ±2 ulp), and each plausible kernel mistake below fails it.  CPU only."""
import numpy as np
import pytest
import torch

from oracle import boxes as OB
from oracle import layers as L
from oracle import pipeline as P
import stage_ref64 as S

F = np.float32


def expf_2ulp(d, rng):
    """fp32 exp moved by a random -2..+2 ulp per element from the correctly rounded value, then pulled back by one step
    wherever that lands more than 2 ulp from the exact value (the CUDA expf accuracy: at most 2 ulp from exp(d))."""
    exact = np.exp(d.astype(np.float64))
    cr = exact.astype(F)
    e = cr
    k = rng.integers(-2, 3, e.shape)
    for s in (1, 2):
        e = np.where(k >= s, np.nextafter(e, F(np.inf)), e)
        e = np.where(k <= -s, np.nextafter(e, F(0)), e)
    far = np.abs(e.astype(np.float64) - exact) > 2 * np.spacing(e).astype(np.float64)
    return np.where(far, np.where(e > cr, np.nextafter(e, F(0)), np.nextafter(e, F(np.inf))), e)


def cls_softmax_model(x, rng):
    """cls_finish_kernel's softmax: lane c % 32 adds its logits' expf in column order from 0, then 5 xor-shuffle adds."""
    r, C = x.shape
    m = x.max(axis=1, keepdims=True)
    e = expf_2ulp((x - m).astype(F), rng)
    lanes = np.zeros((r, 32), F)
    for c in range(C):
        lanes[:, c % 32] = lanes[:, c % 32] + e[:, c]
    for o in (16, 8, 4, 2, 1):
        lanes = lanes + lanes[:, np.arange(32) ^ o]
    return (e / lanes[:, :1]).astype(F)


def rpn_softmax_model(bg, fg, rng):
    m = np.maximum(bg, fg)
    e0, e1 = expf_2ulp((bg - m).astype(F), rng), expf_2ulp((fg - m).astype(F), rng)
    return (e1 / (e0 + e1)).astype(F)


def spatial_mean_model(x):
    r, h, w, c = x.shape
    s = np.zeros((r, c), F)
    for v in x.reshape(r, h * w, c).transpose(1, 0, 2):
        s = s + v
    return (s / F(h * w)).astype(F)


def bbox_decode_model(rois, deltas, C, meta, fma=False, two_sided=False):
    """bbox_decode_kernel in numpy fp32, one rounding per operation; fma: pcx / pcy through a float64 fma rounded once."""
    meta = np.asarray(meta, F)
    bi = np.clip(rois[:, 0].astype(np.int64), 0, meta.shape[0] - 1)
    s, ymax, xmax = meta[bi, 0:1], meta[bi, 1:2] - F(1), meta[bi, 2:3] - F(1)
    x1, y1, x2, y2 = (rois[:, k:k + 1] / s for k in range(1, 5))
    w, h = (x2 - x1) + F(1), (y2 - y1) + F(1)
    cx, cy = x1 + F(0.5) * w, y1 + F(0.5) * h
    d = deltas.reshape(rois.shape[0], C, 4)
    if fma:
        pcx = (d[..., 0].astype(np.float64) * w + cx).astype(F)
        pcy = (d[..., 1].astype(np.float64) * h + cy).astype(F)
    else:
        pcx, pcy = d[..., 0] * w + cx, d[..., 1] * h + cy
    pw, ph = OB.exp_f32(d[..., 2]) * w, OB.exp_f32(d[..., 3]) * h
    o = np.stack([pcx - F(0.5) * pw, pcy - F(0.5) * ph, pcx + F(0.5) * pw, pcy + F(0.5) * ph], axis=-1)
    if two_sided:
        o[..., 0::2] = np.minimum(o[..., 0::2], xmax[..., None])
        o[..., 1::2] = np.minimum(o[..., 1::2], ymax[..., None])
        o = np.maximum(o, F(0))
    else:
        o[..., :2] = np.maximum(o[..., :2], F(0))
        o[..., 2] = np.minimum(o[..., 2], xmax)
        o[..., 3] = np.minimum(o[..., 3], ymax)
    return o.reshape(rois.shape[0], 4 * C).astype(F)


def crop_clamped(feat, nb, crop):
    """crop_and_resize with the sample coordinates clamped into the map instead of extrapolating to 0."""
    _, H, W, _ = feat.shape
    y1, x1, y2, x2 = nb[:, 0], nb[:, 1], nb[:, 2], nb[:, 3]
    idx = np.arange(crop, dtype=F)
    in_y = (y1 * F(H - 1))[:, None] + idx[None, :] * ((y2 - y1) * F(H - 1) / F(crop - 1))[:, None]
    in_x = (x1 * F(W - 1))[:, None] + idx[None, :] * ((x2 - x1) * F(W - 1) / F(crop - 1))[:, None]
    iy, ix = np.clip(in_y, F(0), F(H - 1)), np.clip(in_x, F(0), F(W - 1))
    top, bot, lef, rig = (np.floor(iy).astype(int), np.ceil(iy).astype(int), np.floor(ix).astype(int), np.ceil(ix).astype(int))
    yl = (iy - np.floor(iy)).astype(F)[:, :, None, None]
    xl = (ix - np.floor(ix)).astype(F)[:, None, :, None]
    f = feat[0]
    t = f[top[:, :, None], lef[:, None, :]] + (f[top[:, :, None], rig[:, None, :]] - f[top[:, :, None], lef[:, None, :]]) * xl
    b = f[bot[:, :, None], lef[:, None, :]] + (f[bot[:, :, None], rig[:, None, :]] - f[bot[:, :, None], lef[:, None, :]]) * xl
    return (t + (b - t) * yl).astype(F)


# ---- the models pass ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C", [2, 5, 21, 31, 32, 33, 81, 1024])
def test_cls_softmax_model_within_bound(C):
    rng = np.random.default_rng(C)
    x, kind = S.logit_rows(rng, 60, C)
    p64, bound = S.softmax_ref(x, S.cls_depth(C))
    for trial in range(3):
        S.check_bounded(cls_softmax_model(x, rng), p64, bound, "cls softmax model C=%d" % C)
    # the bound's regimes are reached: probabilities below 1e-6 and fp32 subnormals (spike rows)
    assert (p64 < 1e-6).any() and (p64[kind == S.ROW_KINDS.index("spike100")] < 1e-38).any()


def test_rpn_softmax_model_within_bound():
    rng = np.random.default_rng(2)
    x, _ = S.logit_rows(rng, 6000, 2)
    bg, fg = x[:, 0], x[:, 1]
    p64, bound = S.rpn_fg_ref(bg, fg)
    S.check_bounded(rpn_softmax_model(bg, fg, rng), p64, bound, "rpn softmax model")


@pytest.mark.parametrize("hw", [1, 49, 196])
@pytest.mark.parametrize("data", ["normal", "offset", "cancel"])
def test_spatial_mean_model_within_bound(hw, data):
    rng = np.random.default_rng(hw)
    s = int(np.sqrt(hw))
    x = rng.standard_normal((5, s, s, 64))
    if data == "offset":
        x += 1e4
    elif data == "cancel":
        x += np.where(np.arange(hw).reshape(1, s, s, 1) < hw // 2, 1e4, -1e4)
    x = x.astype(F)
    m64, bound = S.spatial_mean_ref(x)
    got = spatial_mean_model(x)
    S.check_bounded(got, m64, bound, "spatial mean model")
    if hw > 1 and data != "normal":
        assert (np.abs(got - m64) > 4 * S.U * np.abs(m64)).any()     # rounding well past the division's share: the sum term binds


def _decode_case(seed=0, C=21, R=97):
    rng = np.random.default_rng(seed)
    xy = rng.uniform(0, 800, (R, 2))
    rois = np.hstack([np.zeros((R, 1)), xy, xy + rng.uniform(8, 300, (R, 2))]).astype(F)
    return rois, S.edge_deltas(rng, R, C), C, [(1.6, 375, 500)]


def test_bbox_decode_model_is_the_oracle():
    rois, deltas, C, meta = _decode_case()
    with np.errstate(over="ignore", invalid="ignore"):
        want = P.im_detect_post(rois, np.zeros((rois.shape[0], C), F), deltas, meta[0][0], meta[0][1], meta[0][2])[1]
        S.check_boxes_exact(bbox_decode_model(rois, deltas, C, meta), want, "bbox_decode model")
        assert np.isinf(OB.exp_f32(deltas[:, 2::4])).any()        # exp overflow is reached
    # and so are the outcomes that separate the one-sided clip from a two-sided one
    b = want.reshape(-1, 4)
    assert (b[:, 0] > 499).any() and (b[:, 2] < 0).any() and (b[:, 1] > 374).any() and (b[:, 3] < 0).any()


def test_crop_boxes_reach_every_edge():
    for fh, fw, crop in ((38, 50, 7), (38, 50, 14), (2, 3, 7), (2, 3, 14)):
        b = S.crop_boxes(np.random.default_rng(0), fh, fw, 40, crop)
        assert S.crop_last_sample(b[15, 0], b[15, 2], fw, crop)[1] == F(fw - 1)
        assert S.crop_last_sample(b[15, 1], b[15, 3], fh, crop)[1] == F(fh - 1)
        feat = np.ones((1, fh, fw, 4), F)
        out = L.crop_and_resize(feat, P.roi_norm_boxes(feat.shape, np.hstack([np.zeros((40, 1), F), b])), crop)
        assert (out[4:8] == 0).all() and (out[:4] == 0).any() and (out[:4] == 1).any()   # outside: 0; straddling: both


def test_split_host_records_raises_past_max_det():
    from tf_faster_rcnn_b200 import engine
    max_det = 4
    host = torch.zeros((2, engine.REC_HEADER + max_det * 6), dtype=torch.float32)
    host.view(torch.int32)[:, 0] = torch.tensor([max_det, max_det + 1], dtype=torch.int32)
    with pytest.raises(RuntimeError, match="produced 5 detections"):
        engine.split_host_records(host, max_det)
    host.view(torch.int32)[1, 0] = 2
    assert [d.shape for d in engine.split_host_records(host, max_det)] == [(4, 6), (2, 6)]


# ---- the mutants fail -----------------------------------------------------------------------------------------------
def _mutant_fma_decode():
    rois, deltas, C, meta = _decode_case(1)
    with np.errstate(over="ignore", invalid="ignore"):
        S.check_boxes_exact(bbox_decode_model(rois, deltas, C, meta, fma=True), bbox_decode_model(rois, deltas, C, meta))


def _mutant_two_sided_clip():
    rois, deltas, C, meta = _decode_case(2)
    with np.errstate(over="ignore", invalid="ignore"):
        want = P.im_detect_post(rois, np.zeros((rois.shape[0], C), F), deltas, meta[0][0], meta[0][1], meta[0][2])[1]
        S.check_boxes_exact(bbox_decode_model(rois, deltas, C, meta, two_sided=True), want)


def _denorm_case():
    rng = np.random.default_rng(3)
    return (rng.standard_normal((50, 4 * 21)) * 0.5).astype(F)


def _mutant_swapped_xy_stds():
    d = _denorm_case()
    sx, sy, sw, sh = S.BBOX_STDS
    S.check_exact(S.denorm_ref(d, (sy, sx, sw, sh), S.BBOX_MEANS), S.denorm_ref(d, S.BBOX_STDS, S.BBOX_MEANS))


def _mutant_zero_mean():
    d = _denorm_case()
    S.check_exact(S.denorm_ref(d, S.BBOX_STDS, (0, 0, 0, 0)), S.denorm_ref(d, S.BBOX_STDS, S.BBOX_MEANS))


def _softmax_case():
    x, _ = S.logit_rows(np.random.default_rng(4), 60, 81)
    return x, S.softmax_ref(x, S.cls_depth(81))


def _mutant_flush_below_1e6():
    x, (p64, bound) = _softmax_case()
    p = cls_softmax_model(x, np.random.default_rng(5))
    S.check_bounded(np.where(p < 1e-6, F(0), p), p64, bound)


def _mutant_one_percent():
    x, (p64, bound) = _softmax_case()
    S.check_bounded((cls_softmax_model(x, np.random.default_rng(6)) * F(1.01)).astype(F), p64, bound)


def _mutant_crop_clamps():
    fh, fw = 38, 50
    feat = np.random.default_rng(7).standard_normal((1, fh, fw, 8)).astype(F)
    b = S.crop_boxes(np.random.default_rng(7), fh, fw, 60, 7)
    nb = P.roi_norm_boxes(feat.shape, np.hstack([np.zeros((60, 1), F), b]))
    S.check_exact(crop_clamped(feat, nb, 7), L.crop_and_resize(feat, nb, 7))


def _cap_case():
    rng = np.random.default_rng(8)
    R, C = 300, 21
    return S.cap_tie_probs(rng, R, C, 60, 80), S.grid_pred(R, C)


def _mutant_cap_drops_ties():
    probs, pred = _cap_case()
    want = P.test_net_post(probs, pred, P.opts())
    uncapped = P.test_net_post(probs, pred, P.opts(max_per_image=0))
    th = np.sort(np.hstack([d[:, 4] for d in uncapped[1:]]))[-100]
    mutant = [uncapped[0]] + [d[d[:, 4] > th] for d in uncapped[1:]]
    got = S.flat_records(mutant)
    S.check_records(got, got.shape[0], [d.shape[0] for d in mutant], want, 256)


def _mutant_ties_toward_higher_index():
    rng = np.random.default_rng(9)
    R, C = 300, 21
    probs, pred = S.quantised_probs(rng, R, C), S.clustered_pred(rng, R, C)
    want = P.test_net_post(probs, pred, P.opts())
    mutant = P.test_net_post(probs[::-1].copy(), pred[::-1].copy(), P.opts())     # RoI order reversed: ties -> higher index
    got = S.flat_records(mutant)
    S.check_records(got, got.shape[0], [d.shape[0] for d in mutant], want, 256)


MUTANTS = {
    "fma_decode": _mutant_fma_decode,
    "two_sided_clip": _mutant_two_sided_clip,
    "swapped_xy_stds": _mutant_swapped_xy_stds,
    "zero_mean": _mutant_zero_mean,
    "probs_below_1e-6_flushed": _mutant_flush_below_1e6,
    "probs_1pct_error": _mutant_one_percent,
    "crop_clamps": _mutant_crop_clamps,
    "cap_drops_ties": _mutant_cap_drops_ties,
    "ties_toward_higher_index": _mutant_ties_toward_higher_index,
}


@pytest.mark.parametrize("mutant", list(MUTANTS))
def test_mutant_fails_its_comparator(mutant):
    with pytest.raises(AssertionError):
        MUTANTS[mutant]()
