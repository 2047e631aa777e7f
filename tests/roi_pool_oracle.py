"""Oracle for POOLING_MODE 'align' / 'pool' (test infrastructure, built on oracle.pipeline's stages):

  roi_align_model        torchvision.ops.roi_align on NHWC, each fp32 operation rounded once in the kernel's order
  roi_pool_model         torchvision.ops.roi_pool on NHWC
  roi_align_ref64        the exact (float64) weighted mean at the model's fp32 sample coordinates, and an error bound
  pool_stage             one of the two models as the pooling stage of the chains below
  test_image             oracle.pipeline.test_image with the pooling swapped in
  score_boxes            region_oracle.score_boxes (caller boxes as RoIs) with the pooling swapped in

Both models are vectorised over channels and over the RoIs that share a sample grid, so whole-network chains stay affordable.
`_bug` (tests only) switches in one plausible mistake, so a test can show that its comparator catches it.
"""
import numpy as np

from oracle import nets as N
from oracle import pipeline as P

F = np.float32
SCALE = F(1.0 / 16)
CHUNK = 1 << 22          # elements per vectorised step


def _image_index(rois, batch):
    return np.clip(np.trunc(rois[:, 0]).astype(np.int64), 0, batch - 1)


def _axis(v, dim, bug=None):
    """One axis of the bilinear sample: v fp32 -> (lo, hi, l, h, valid, v after the clamps).  A sample outside [-1, dim] is
    invalid; v is clamped at 0; at lo >= dim - 1 both neighbours become dim - 1 and v = dim - 1."""
    valid = ~((v <= -1) if bug == "le_minus_one" else (v < -1)) & ~(v > dim)
    v = np.where(valid, v, F(0)).astype(F)
    v = np.where(v <= 0, F(0), v).astype(F)
    lo = v.astype(np.int64)
    if bug == "no_top_clamp":
        hi = lo + 1                                  # neighbour past the map: read as zero padding
    else:
        edge = lo >= dim - 1
        lo = np.where(edge, dim - 1, lo)
        hi = np.where(edge, dim - 1, lo + 1)
        v = np.where(edge, F(dim - 1), v).astype(F)
    l = (v - lo.astype(F)).astype(F)
    return lo, hi, l, (F(1) - l).astype(F), valid, v


def _align_geometry(rois, pooled, sampling_ratio, aligned, scale, bug):
    r = np.asarray(rois, dtype=F)
    off = F(0.5) if aligned and bug != "no_offset" else F(0)
    sx, sy = (r[:, 1] * scale - off).astype(F), (r[:, 2] * scale - off).astype(F)
    ex, ey = (r[:, 3] * scale - off).astype(F), (r[:, 4] * scale - off).astype(F)
    rw, rh = (ex - sx).astype(F), (ey - sy).astype(F)
    if not aligned and bug != "no_min_size":
        rw, rh = np.where(rw < 1, F(1), rw).astype(F), np.where(rh < 1, F(1), rh).astype(F)
    bw, bh = (rw / F(pooled)).astype(F), (rh / F(pooled)).astype(F)
    if sampling_ratio > 0:
        gw = gh = np.full(r.shape[0], sampling_ratio, np.int64)
    else:
        gw, gh = np.ceil(bw).astype(np.int64), np.ceil(bh).astype(np.int64)
    count = gh * gw if bug == "no_min_count" else np.maximum(gh * gw, 1)
    return sx, sy, bw, bh, gw, gh, count


@np.errstate(invalid="ignore", divide="ignore", over="ignore")      # non-finite maps: IEEE results, as on the device
def _align(feat, rois, pooled, sampling_ratio, aligned, scale, bug, ref64):
    feat = np.asarray(feat, dtype=F)
    B, H, W, C = feat.shape
    R = rois.shape[0]
    sx, sy, bw, bh, gw, gh, count = _align_geometry(rois, pooled, sampling_ratio, aligned, scale, bug)
    bi = _image_index(np.asarray(rois, F), B)
    src = np.pad(feat, ((0, 0), (0, 2), (0, 2), (0, 0))) if bug == "no_top_clamp" else feat
    acc_t = np.float64 if ref64 else F
    out = np.zeros((R, pooled, pooled, C), acc_t)
    mag = np.zeros((R, pooled, pooled, C), np.float64)
    pidx = np.arange(pooled, dtype=F)
    keys = np.stack([gh, gw], axis=1)
    for g_h, g_w in {tuple(k) for k in keys.tolist()}:
        sel = np.where((keys[:, 0] == g_h) & (keys[:, 1] == g_w))[0]
        if g_h <= 0 or g_w <= 0:
            continue                                     # no sample: 0 / count
        step = max(1, CHUNK // (pooled * pooled * C))
        for s0 in range(0, sel.shape[0], step):
            ii = sel[s0:s0 + step]
            # sample coordinates [G, P, g]: (start + p * bin) + ((i + 0.5) * bin) / g, each op rounded in fp32
            iy = (np.arange(g_h, dtype=F) + F(0.5)).astype(F)
            ix = (np.arange(g_w, dtype=F) + F(0.5)).astype(F)
            y = ((sy[ii, None, None] + pidx[None, :, None] * bh[ii, None, None]).astype(F)
                 + ((iy[None, None, :] * bh[ii, None, None]).astype(F) / F(g_h)).astype(F)).astype(F)
            x = ((sx[ii, None, None] + pidx[None, :, None] * bw[ii, None, None]).astype(F)
                 + ((ix[None, None, :] * bw[ii, None, None]).astype(F) / F(g_w)).astype(F)).astype(F)
            ylo, yhi, ly, hy, yv, yc = _axis(y, H, bug)
            xlo, xhi, lx, hx, xv, xc = _axis(x, W, bug)
            if ref64:                                    # exact weights at the same fp32 (clamped) coordinates
                ly, lx = yc.astype(np.float64) - ylo, xc.astype(np.float64) - xlo
                hy, hx = 1.0 - ly, 1.0 - lx
            b = bi[ii][:, None, None]
            acc = np.zeros((ii.shape[0], pooled, pooled, C), acc_t)
            am = np.zeros(acc.shape, np.float64)
            for a in range(g_h):
                for c in range(g_w):
                    Yl, Yh, Xl, Xh = ylo[:, :, a, None], yhi[:, :, a, None], xlo[:, None, :, c], xhi[:, None, :, c]
                    hya, lya, hxc, lxc = hy[:, :, a, None], ly[:, :, a, None], hx[:, None, :, c], lx[:, None, :, c]
                    w1, w2, w3, w4 = hya * hxc, hya * lxc, lya * hxc, lya * lxc
                    v1, v2, v3, v4 = src[b, Yl, Xl], src[b, Yl, Xh], src[b, Yh, Xl], src[b, Yh, Xh]
                    t1, t2, t3, t4 = w1[..., None] * v1, w2[..., None] * v2, w3[..., None] * v3, w4[..., None] * v4
                    t = ((t1 + t2) + t3) + t4
                    ok = (yv[:, :, a, None] & xv[:, None, :, c])[..., None]
                    acc = np.where(ok, acc + t, acc)
                    if ref64:
                        am = np.where(ok, am + (np.abs(t1) + np.abs(t2) + np.abs(t3) + np.abs(t4)), am)
            out[ii] = acc
            mag[ii] = am
    cnt = count.astype(acc_t)[:, None, None, None]
    res = (out / cnt).astype(acc_t)
    if not ref64:
        return res
    n = np.maximum(gh * gw, 0).astype(np.float64)[:, None, None, None]
    return res, mag / cnt.astype(np.float64), n


def roi_align_model(feat, rois, pooled, sampling_ratio=0, aligned=False, scale=SCALE, _bug=None):
    """torchvision.ops.roi_align(NCHW(feat), rois, pooled, scale, sampling_ratio, aligned) on NHWC feat [B,H,W,C] fp32, rois
    [R,5] = (image index clamped to [0, B-1], x1, y1, x2, y2) -> [R, pooled, pooled, C] fp32.  Per output element:
    acc += ((w1*v1 + w2*v2) + w3*v3) + w4*v4 over the samples in (iy, ix) order, then acc / max(gh*gw, 1).  A sample outside
    [-1, dim] is skipped; torchvision adds 0 * feat[b, 0, 0] for it instead, which differs only where that cell is +-Inf or NaN."""
    return _align(feat, np.asarray(rois, F), pooled, sampling_ratio, aligned, F(scale), _bug, False).astype(F)


def roi_align_ref64(feat, rois, pooled, sampling_ratio=0, aligned=False, scale=SCALE):
    """-> (exact, bound): the float64 weighted mean at roi_align_model's fp32 sample coordinates (weights ly = y - y_low,
    hy = 1 - ly ... formed in float64), and a bound on |roi_align_model - exact|.

    Derivation, u = 2^-24, gamma_k = k u / (1 - k u), n = gh * gw samples: at the clamped fp32 coordinate y >= 0, ly = y - y_low
    is exact (y_low = floor(y), the difference is a multiple of ulp(y) below 1); hy = 1 - ly rounds once, and the product
    w = hy * hx rounds once more, so each fp32 weight is the exact one times (1 + t), |t| <= gamma_3.  The product w * v adds one
    rounding (gamma_4), the three additions of the four terms at most three more (gamma_7 on each term), the running sum over n
    samples at most n more (gamma_{n+7}), the division by the count one more.  Hence
        |model - exact| <= gamma_{n+8} * (sum over the samples of |w1 v1| + |w2 v2| + |w3 v3| + |w4 v4|) / count
    for results away from the subnormal range; 8 n 2^-149 / count covers the absolute error of subnormal products and sums."""
    res, mag, n = _align(feat, np.asarray(rois, F), pooled, sampling_ratio, aligned, F(scale), None, True)
    u = 2.0 ** -24
    k = n + 8
    cnt = np.maximum(n, 1)
    return res, (k * u / (1 - k * u)) * mag + 8 * n * 2.0 ** -149 / cnt


def _round_half_away(v):
    v = np.asarray(v, np.float64)
    return (np.sign(v) * np.floor(np.abs(v) + 0.5)).astype(np.int64)


def roi_pool_model(feat, rois, pooled, scale=SCALE, _bug=None):
    """torchvision.ops.roi_pool on NHWC: corners round(x * scale) half away from zero, rh = max(y2 - y1 + 1, 1), bin = rh / P
    in fp32, rows floor(p * bin) + y1 .. ceil((p+1) * bin) + y1 clamped to [0, H] (columns alike); the max by '>' from
    -FLT_MAX in (row, column) order, 0 for an empty bin."""
    feat = np.asarray(feat, dtype=F)
    rois = np.asarray(rois, F)
    B, H, W, C = feat.shape
    R = rois.shape[0]
    rnd = (lambda v: np.rint(np.asarray(v, np.float64)).astype(np.int64)) if _bug == "half_even" else _round_half_away
    xy = [rnd((rois[:, k] * F(scale)).astype(F)) for k in (1, 2, 3, 4)]
    sx, sy, ex, ey = xy
    bw = (np.maximum(ex - sx + 1, 1).astype(F) / F(pooled)).astype(F)
    bh = (np.maximum(ey - sy + 1, 1).astype(F) / F(pooled)).astype(F)
    bi = _image_index(rois, B)
    out = np.zeros((R, pooled, pooled, C), F)
    lowest = F(-np.finfo(F).max)
    for ph in range(pooled):
        h0 = np.clip(np.floor((F(ph) * bh).astype(F)).astype(np.int64) + sy, 0, H)
        h1 = np.clip(np.ceil((F(ph + 1) * bh).astype(F)).astype(np.int64) + sy, 0, H)
        for pw in range(pooled):
            w0 = np.clip(np.floor((F(pw) * bw).astype(F)).astype(np.int64) + sx, 0, W)
            w1 = np.clip(np.ceil((F(pw + 1) * bw).astype(F)).astype(np.int64) + sx, 0, W)
            empty = (h1 <= h0) | (w1 <= w0)
            m = np.full((R, C), lowest, F)
            for dy in range(int(max((h1 - h0).max(), 0))):
                y = h0 + dy
                for dx in range(int(max((w1 - w0).max(), 0))):
                    x = w0 + dx
                    ok = (y < h1) & (x < w1)
                    v = feat[bi, np.minimum(y, H - 1), np.minimum(x, W - 1)]
                    m = np.where(ok[:, None] & (v > m), v, m)
            out[:, ph, pw] = np.where(empty[:, None], F(0), m)
    return out


def edge_rois(h, w, rng, n_random=60):
    """Blob-pixel RoIs over an h x w map (x16): random boxes, many partly or wholly off the map, and the edge cases: boxes
    straddling each side, wholly outside, inverted, zero-size, sub-cell, whole-map, and samples exactly at -1."""
    H, W = 16.0 * h, 16.0 * w
    x1 = rng.uniform(-0.5 * W, 1.2 * W, n_random); y1 = rng.uniform(-0.5 * H, 1.2 * H, n_random)
    bw = rng.uniform(0, 1.5 * W, n_random); bh = rng.uniform(0, 1.5 * H, n_random)
    boxes = list(np.stack([x1, y1, x1 + bw, y1 + bh], 1))
    boxes += [
        [-40, 0.3 * H, 20, 0.6 * H], [0.8 * W, 0.2 * H, W + 50, 0.4 * H],          # straddle left / right
        [0.1 * W, -33, 0.4 * W, 9], [0.3 * W, 0.9 * H, 0.5 * W, H + 70],           # straddle top / bottom
        [-300, -300, -100, -100], [W + 20, H + 20, W + 400, H + 90],               # wholly outside
        [0.7 * W, 0.6 * H, 0.2 * W, 0.1 * H],                                      # inverted
        [0.5 * W, 0.5 * H, 0.5 * W, 0.5 * H],                                      # zero size
        [3.0, 5.0, 9.0, 11.0],                                                     # inside one cell
        [0, 0, W - 1, H - 1], [0, 0, W, H], [-W, -H, 2 * W, 2 * H],                # whole map, the caller-box bound
        [-32, -32, 0, 0], [-16, -24, 16, 8],                                       # samples exactly at -1
        [W - 8, H - 8, W + 8, H + 8], [16 * (w - 1), 16 * (h - 1), W, H],          # the last cell, y_low at H - 1
    ]
    r = np.asarray(boxes, np.float64).astype(F)
    return np.hstack([np.zeros((r.shape[0], 1), F), r]).astype(F)


def half_rois(rng, h, w, n=120):
    """Corners whose x / 16 lands exactly on +-k.5 (x = 16k + 8)."""
    k = rng.integers(-3, max(h, w) + 3, (n, 4))
    r = (16 * k + 8).astype(F)
    r[:, 2:] = np.maximum(r[:, 2:], r[:, :2] - 16)
    return np.hstack([np.zeros((n, 1), F), r]).astype(F)


def pool_stage(mode, pooled, sampling_ratio=0, aligned=False):
    """(feat [B,H,W,C], rois [R,5]) -> pool5 of POOLING_MODE `mode` ('align' | 'pool')."""
    if mode == "align":
        return lambda feat, rois: roi_align_model(feat, rois, pooled, sampling_ratio, aligned)
    assert mode == "pool"
    return lambda feat, rois: roi_pool_model(feat, rois, pooled)


def front(net, w, blob, im_info, o):
    """The stages ahead of the pooling (backbone, RPN, proposals): they do not depend on the pooling mode."""
    im_info = np.asarray(im_info, dtype=F)
    st = {}
    st["feat"] = N.image_to_head(net, w, blob)
    st["rpn"], st["rpn_cls_score"], st["rpn_bbox_pred"] = P.rpn_head(net, w, st["feat"])
    st["rpn_scores"], st["rpn_props"], st["anchors"] = P.rpn_decode(st["rpn_cls_score"], st["rpn_bbox_pred"], im_info, o)
    st["rois"], st["roi_scores"], st["roi_keep"] = P.proposals(st["rpn_scores"], st["rpn_props"], o)
    return st


def head(net, w, front_st, num_classes, o, pool):
    """front() followed by pool5 = pool(feat, rois), the head and the classifier."""
    st = dict(front_st)
    st["pool5"] = pool(st["feat"], st["rois"])
    st["fc7"] = N.head_to_tail(net, w, st["pool5"])
    st["cls_score"], st["cls_prob"], st["bbox_pred"] = P.region_classification(net, w, st["fc7"], num_classes, o)
    return st


def test_image(net, w, blob, im_info, num_classes, o, pool):
    """oracle.pipeline.test_image with pool5 = pool(feat, rois) (a pool_stage) in place of the crop."""
    return head(net, w, front(net, w, blob, im_info, o), num_classes, o, pool)


def score_boxes(net, w, blob, boxes, scale, orig_hw, o, pool):
    """Caller boxes [n,4] in original-image pixels, pooled by `pool` -> dict(rois, pool5, fc7, cls_score, cls_prob, bbox_pred,
    scores, pred_boxes)."""
    boxes = np.asarray(boxes, dtype=F).reshape(-1, 4)
    st = {"rois": np.hstack([np.zeros((boxes.shape[0], 1), F), (boxes * F(scale)).astype(F)]).astype(F)}
    st["pool5"] = pool(N.image_to_head(net, w, blob), st["rois"])
    st["fc7"] = N.head_to_tail(net, w, st["pool5"])
    num_classes = w[N.scope_of(net) + "/cls_score/weights"].shape[1]
    st["cls_score"], st["cls_prob"], st["bbox_pred"] = P.region_classification(net, w, st["fc7"], num_classes, o)
    st["scores"], st["pred_boxes"] = P.im_detect_post(st["rois"], st["cls_prob"], st["bbox_pred"], scale, orig_hw[0], orig_hw[1])
    return st
