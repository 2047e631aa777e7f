"""Float64 references, comparators and edge cases for the post-processing extensions (helper, CPU only):

  soft_nms64        Soft-NMS restated from the text of Detectron's cpu_soft_nms (utils/cython_nms.pyx) in float64, with a
                    running error bound per value and the margin of every decision the run takes
  check_soft64      an fp32 result (the C oracle, the numpy model or the device) against soft_nms64
  EDGES             edge-case generators, exact in fp32: integer coordinates and exactly representable thresholds
  features_ref      numpy gather of frcnn_detect_features
"""
import math

import numpy as np

F = np.float32
U = 2.0 ** -24                                   # unit roundoff of fp32 round-to-nearest
FMAX = float(np.finfo(F).max)


# ---- Soft-NMS in float64 ---------------------------------------------------------------------------------------------
# Error model.  Every value v of the float64 run carries e(v), a bound on |v32 - v| where v32 is what the fp32 definition
# computes (each operation one round-to-nearest, include/frcnn_b200.h).  For z = x op y with inputs carrying ex, ey:
#   +, -   e(z) = ex + ey + u|z|               *   e(z) = |y|ex + |x|ey + ex*ey + u|z|
#   /      e(z) = (ex + |z|ey) / (|y| - ey) + u|z|       min, max   e(z) = max(ex, ey)
# and e(z) = 0 when both inputs are exact and z is representable in fp32 (the rounding then returns z itself; for +, - and * of
# fp32 operands the float64 result is exact at the magnitudes used here, and a float64 quotient of fp32 operands that has 24
# significant bits is the exact quotient).  The gaussian weight is bounded by its interval: w32 lies between
# exp(-(q + e(q))) and exp(-(q - e(q))), each widened by the fp64 exp's two ulps and rounded to fp32 (rounding is monotone).
# So a score decayed k times carries e(s) <= |s| * sum_k (c_k + 1) u, c_k u the relative bound of the k-th weight: c = 0 for an exact weight (untouched, hard, or exact integer overlaps), and it
# grows as 1 - ov cancels for linear, or with q for gaussian.  The bound is first order plus the ex*ey terms: it is derived,
# not fitted, and the comparator applies it with no slack.
def _r(z, e):
    if not math.isfinite(z):
        return 0.0 if e == 0.0 else math.inf
    if abs(z) > FMAX:
        return math.inf
    if e == 0.0 and float(F(z)) == z:
        return 0.0
    return e + U * abs(z)


def _sub(x, ex, y, ey):
    z = x - y
    return z, _r(z, ex + ey)


def _add(x, ex, y, ey):
    z = x + y
    return z, _r(z, ex + ey)


def _mul(x, ex, y, ey):
    z = x * y
    if not math.isfinite(z) or not (math.isfinite(x) and math.isfinite(y)):
        return z, 0.0 if ex == 0.0 and ey == 0.0 else math.inf
    return z, _r(z, abs(y) * ex + abs(x) * ey + ex * ey)


def _div(x, ex, y, ey):
    z = x / y
    if ey >= abs(y):
        return z, math.inf
    return z, _r(z, (ex + abs(z) * ey) / (abs(y) - ey))


def _area(b):
    w, ew = _add(*_sub(b[2], 0.0, b[0], 0.0), 1.0, 0.0)
    h, eh = _add(*_sub(b[3], 0.0, b[1], 0.0), 1.0, 0.0)
    return _mul(w, ew, h, eh)


def _undecided(margin, err):
    """A decision is open when its margin is within the fp32 error of its inputs; an exact zero margin with exact inputs is
    decided (the fp32 run computes the same zero)."""
    if math.isnan(margin):
        return False
    return err > 0.0 and abs(margin) <= err


class Soft64:
    """Result of soft_nms64: rows [k,5] float64 (input boxes, decayed scores), keep [k], err [k] (score error bounds), decays
    [k] (decays applied to each kept score), settled (the leading selections every decision of which is decided), complete
    (all decisions decided: the kept count is determined too) and margins {argmax gap, ov - nt, score - thresh}: the smallest
    non-zero |margin| of each kind with its error bound, how close the run came to flipping a decision."""

    def __init__(self):
        self.rows, self.keep, self.err, self.decays = [], [], [], []
        self.settled, self.complete = 0, True
        self.margins = {"argmax": (math.inf, 0.0), "ov-nt": (math.inf, 0.0), "score-thresh": (math.inf, 0.0)}

    def note(self, kind, margin, err):
        if margin != 0.0 and not math.isnan(margin) and abs(margin) < self.margins[kind][0]:
            self.margins[kind] = (abs(margin), err)
        return _undecided(margin, err)


def soft_nms64(dets, method="linear", sigma=0.5, nt=0.3, score_thresh=0.001):
    """Detectron's cpu_soft_nms, restated: for each i, the scan maxscore < boxes[pos, 4] picks the selection (lowest position
    of the maximum; a NaN head stays); every later box that overlaps it ('+1' pixel IoU) is decayed, and pruned with the last
    box moved into its place when its score falls below the threshold.  Float64 throughout; parameters rounded to fp32 once,
    as the product does.  -> Soft64."""
    d = np.asarray(dets, dtype=F)[:, :5]
    # x1 y1 x2 y2 s | index, e(s), decays, input score, decay history (see the tie rule below)
    a = [[float(v) for v in row] + [k, 0.0, 0, float(row[4]), ()] for k, row in enumerate(d)]
    sigma, nt, thresh = float(F(sigma)), float(F(nt)), float(F(score_thresh))
    res = Soft64()
    settled = None
    N = len(a)
    i = 0
    while i < N:
        maxpos = i
        for pos in range(i + 1, N):
            if a[maxpos][4] < a[pos][4]:
                maxpos = pos
        a[i], a[maxpos] = a[maxpos], a[i]
        t = a[i]
        sm, em = t[4], t[6]
        if settled is None:
            for pos in range(i + 1, N):
                s, e = a[pos][4], a[pos][6]
                if math.isnan(s) or math.isnan(sm):
                    continue
                if s == sm:
                    # a tie is decided when both values are exact, or when both rows started from the same input score and
                    # met the same fp32 weights in the same order: their fp32 values are then equal too.  A weight is known
                    # to be the same fp32 value when its overlap was an exact quotient (inter and union exact: the fp32 ov is
                    # that quotient rounded once) of the same value, or when the same box was decayed by the same selection.
                    # Any other tie of inexact values may order either way in fp32.
                    if em + e > 0.0 and (a[pos][8] != t[8] or a[pos][9] != t[9]):
                        settled = i
                        break
                    continue
                margin, err = (sm - s, em + e) if math.isfinite(sm - s) else (math.inf, 0.0)
                if res.note("argmax", margin, err):
                    settled = i
                    break
        ta, eta = _area(t)
        open_decay = False
        pos = i + 1
        while pos < N:
            b = a[pos]
            iw, eiw = _add(*_sub(min(t[2], b[2]), 0.0, max(t[0], b[0]), 0.0), 1.0, 0.0)
            open_decay |= _undecided(iw, eiw)
            overlapped = False
            if iw > 0:
                ih, eih = _add(*_sub(min(t[3], b[3]), 0.0, max(t[1], b[1]), 0.0), 1.0, 0.0)
                open_decay |= _undecided(ih, eih)
                if ih > 0:
                    overlapped = True
                    inter, ein = _mul(iw, eiw, ih, eih)
                    ua, eua = _sub(*_add(ta, eta, *_area(b)), inter, ein)
                    ov, eov = _div(inter, ein, ua, eua)
                    if method == "gaussian":
                        q, eq = _div(*_mul(ov, eov, ov, eov), sigma, 0.0)
                        w = math.exp(-q)
                        lo, hi = math.exp(-(q + eq)), math.exp(-max(q - eq, 0.0))
                        # exp64 within an ulp or two, then one rounding to fp32 (monotone): w32 lies in this interval
                        ew = max(float(F(hi * (1 + 2.0 ** -51))) - w, w - float(F(lo * (1 - 2.0 ** -51))))
                    else:
                        open_decay |= res.note("ov-nt", ov - nt, eov)
                        if method == "linear":
                            w, ew = _sub(1.0, 0.0, ov, eov) if ov > nt else (1.0, 0.0)
                        else:
                            w, ew = (0.0, 0.0) if ov > nt else (1.0, 0.0)
                    if math.isinf(b[4]) and b[6] == 0.0:     # an exact infinity stays one while the fp32 weight is surely > 0
                        b[4], b[6] = w * b[4], (0.0 if ew == 0.0 or w - ew > 0.0 else math.inf)
                    else:
                        b[4], b[6] = _mul(w, ew, b[4], b[6])
                    b[7] += 1
                    if not (w == 1.0 and ew == 0.0):          # an exact weight 1 leaves the fp32 score as it was
                        b[9] += ((ov,) if ein == 0.0 and eua == 0.0 else (t[5], tuple(b[:4])),)
                    open_decay |= res.note("score-thresh", b[4] - thresh, b[6])
            if overlapped and b[4] < thresh:
                a[pos] = a[N - 1]
                N -= 1
            else:
                pos += 1
        if settled is None and open_decay:
            settled = i + 1
        i += 1
    res.rows = np.array([r[:5] for r in a[:N]], np.float64).reshape(-1, 5)
    res.keep = np.array([r[5] for r in a[:N]], np.int64)
    res.err = np.array([r[6] for r in a[:N]], np.float64)
    res.decays = np.array([r[7] for r in a[:N]], np.int64)
    res.complete = settled is None
    res.settled = N if settled is None else min(settled, N)
    return res


def check_soft64(rows, keep, dets, ref, what=""):
    """An fp32 Soft-NMS result (rows [k,5], keep [k]) of dets against soft_nms64's ref: the keep order identical over the
    settled selections (all of it, with the count, when every decision is decided), each box the input row bit for bit, and
    each kept score within its error bound of the float64 score (NaN where it is NaN, the same infinity where it is infinite).
    -> the largest |s32 - s64| / bound over scores with a non-zero bound."""
    rows, keep = np.asarray(rows), np.asarray(keep)
    k = ref.settled
    if ref.complete:
        assert keep.shape[0] == ref.keep.shape[0], "%s: %d kept, float64 keeps %d" % (what, keep.shape[0], ref.keep.shape[0])
    assert keep.shape[0] >= k, "%s: %d kept, float64 settles %d" % (what, keep.shape[0], k)
    bad = np.nonzero(keep[:k] != ref.keep[:k])[0]
    assert bad.size == 0, "%s: selection %d is row %d, float64 selects %d" % (what, bad[0], keep[bad[0]], ref.keep[bad[0]])
    d = np.asarray(dets, dtype=F)
    assert rows[:k, :4].tobytes() == d[keep[:k], :4].tobytes(), "%s: kept boxes are not the input rows" % what
    s32, s64, e = rows[:k, 4].astype(np.float64), ref.rows[:k, 4], ref.err[:k]
    nan = np.isnan(s64)
    assert np.array_equal(np.isnan(s32), nan), "%s: NaN scores differ" % what
    fin = np.isfinite(s64)
    assert np.array_equal(s32[~fin & ~nan], s64[~fin & ~nan]), "%s: infinite scores differ" % what
    diff = np.where(fin, np.abs(np.where(fin, s32, 0.0) - np.where(fin, s64, 0.0)), 0.0)
    over = fin & (diff > e)
    if over.any():
        j = int(np.argmax(over))
        raise AssertionError("%s: score %d is %r, float64 %r, bound %.3g (%d decays)" % (what, j, s32[j], s64[j], e[j], ref.decays[j]))
    pos = fin & (e > 0)
    return float((diff[pos] / e[pos]).max()) if pos.any() else 0.0


# ---- edge cases ----------------------------------------------------------------------------------------------------------
# Each generator (rng, n) -> (dets fp32 [n,5], (method, sigma, nt, score_thresh)).  Coordinates are integers and thresholds
# exactly representable, so every overlap below is computed exactly in fp32 and the decisions at the edge are exact.
def grid_box(k, w=20, h=20, cell=40):
    """A w x h box (inclusive corners, '+1' area w*h) in cell k of a 64-wide grid: boxes in different cells never overlap."""
    x, y = (k % 64) * cell, (k // 64) * cell
    return [x, y, x + w - 1, y + h - 1]


def quantised_scores(rng, n, lo=1, hi=4096):
    """Multiples of 2^-12: exact in fp32, with ties."""
    return rng.integers(lo, hi, n).astype(np.float64) / 4096.0


def clustered_int(rng, n, per=6):
    """Integer boxes around n // per centres in separate grid cells: overlapping groups, no overlap between groups."""
    g = max(n // per, 1)
    out = np.zeros((n, 4), np.float64)
    for k in range(n):
        x, y, _, _ = grid_box(int(rng.integers(0, g)), cell=80)
        j = rng.integers(0, 8, 4)
        out[k] = [x + j[0], y + j[1], x + 30 + j[2], y + 30 + j[3]]
    return out


def _rows(boxes, scores):
    return np.hstack([np.asarray(boxes, np.float64), np.asarray(scores, np.float64)[:, None]]).astype(F)


def iou_at_nt(rng, n):
    """Triples in their own cells: t (10 x 10), b1 inside t with IoU exactly 0.5 = nt (not decayed: '>' is strict) and b2 with
    IoU 0.6 (decayed)."""
    boxes, scores = [], []
    for k in range(n):
        x, y, _, _ = grid_box(k // 3)
        boxes.append([[x, y, x + 9, y + 9], [x, y, x + 9, y + 4], [x, y, x + 9, y + 5]][k % 3])
        scores.append([0.75, 0.5, 0.375][k % 3] + (k // 3 % 7) / 4096.0)
    return _rows(boxes, scores), ("linear", 0.5, 0.5, 0.001)


def decay_to_thresh(rng, n):
    """t (score 0.75), then b1 and b2 with IoU 0.5 against it (weight 1 - 0.5 = 0.5, exact): b1 decays from 0.25 to exactly
    the prune threshold 0.125 (kept: '<' is strict), b2 from one ulp below 0.25 to one ulp below it (pruned)."""
    below = float(np.nextafter(F(0.25), F(0)))
    boxes, scores = [], []
    for k in range(n):
        x, y, _, _ = grid_box(k // 3)
        boxes.append([[x, y, x + 9, y + 9], [x, y, x + 9, y + 4], [x, y, x + 9, y + 4]][k % 3])
        scores.append([0.75, 0.25, below][k % 3])
    return _rows(boxes, scores), ("linear", 0.5, 0.3, 0.125)


def all_pruned_first(rng, n):
    """n copies of one box: IoU 1, weight 0, every other candidate pruned at the first selection."""
    return _rows(np.tile([10, 10, 50, 50], (n, 1)), quantised_scores(rng, n)), ("linear", 0.5, 0.3, 0.001)


def hole_table(rng, n):
    """Row 0 the top box; rows 1 .. n/2 - 1 its copies (pruned at the first selection: the most holes the table can hold,
    cap/2 - 1 at n = cap); the upper half far-away boxes with tied scores that fill the holes in swap-with-last order."""
    h = max(n // 2, 1)
    boxes = [grid_box(0)] * h + [grid_box(1 + k) for k in range(n - h)]
    scores = [0.875] + [0.5] * (n - 1)
    return _rows(boxes, scores), ("linear", 0.5, 0.3, 0.001)


def no_overlap(rng, n):
    """Every box in its own cell: nothing is decayed, and scores under the prune threshold stay (they never overlap)."""
    s = quantised_scores(rng, n)
    s[::5] = 1.0 / 4096.0                        # below score_thresh 0.001 (= 4.1 / 4096)
    return _rows([grid_box(k) for k in range(n)], s), ("linear", 0.5, 0.3, 0.001)


def all_tied(rng, n):
    return _rows(clustered_int(rng, n), np.full(n, 0.5)), ("linear", 0.5, 0.3, 0.001)


def signed_zeros(rng, n):
    """Scores +0, -0, 0.25, 0.5: -0 and +0 tie (the lower position wins), overlapped zeros are pruned, lone ones stay."""
    s = np.array([0.0, -0.0, 0.25, 0.5])[rng.integers(0, 4, n)]
    return _rows(clustered_int(rng, n, per=3), s), ("gaussian", 0.5, 0.3, 0.001)


def sigma_tiny(rng, n):
    """sigma 1e-30: ov^2 / sigma is huge, the weight underflows to 0 and every overlapped box is pruned."""
    return _rows(clustered_int(rng, n), quantised_scores(rng, n)), ("gaussian", 1e-30, 0.3, 0.001)


def sigma_huge(rng, n):
    """sigma 1e30: the weight rounds to 1 and nothing changes."""
    return _rows(clustered_int(rng, n), quantised_scores(rng, n)), ("gaussian", 1e30, 0.3, 0.001)


def inf_scores(rng, n):
    """+Inf scores among overlapping boxes: linear keeps them infinite (weight > 0), the selections take them first."""
    s = quantised_scores(rng, n)
    s[rng.integers(0, n, max(n // 8, 1))] = np.inf
    return _rows(clustered_int(rng, n, per=4), s), ("linear", 0.5, 0.3, 0.001)


def inf_hard(rng, n):
    """+Inf scores under hard suppression: 0 * Inf is NaN mid-run, and a NaN is never pruned (NaN < thresh is false)."""
    s = quantised_scores(rng, n)
    s[rng.integers(0, n, max(n // 4, 1))] = np.inf
    return _rows(clustered_int(rng, n, per=4), s), ("hard", 0.5, 0.3, 0.001)


def nan_scores(rng, n):
    """NaN scores in the input: a NaN at the head position is selected at once, otherwise NaNs wait until only NaNs are left."""
    s = quantised_scores(rng, n)
    s[rng.integers(0, n, max(n // 6, 1))] = np.nan
    if n > 1:
        s[0] = np.nan
    return _rows(clustered_int(rng, n, per=4), s), ("linear", 0.5, 0.3, 0.001)


EDGES = {f.__name__: f for f in (iou_at_nt, decay_to_thresh, all_pruned_first, hole_table, no_overlap, all_tied, signed_zeros,
                                 sigma_tiny, sigma_huge, inf_scores, inf_hard, nan_scores)}
NONFINITE = ("inf_scores", "inf_hard", "nan_scores")

# The four rows of the NaN finding: no overlaps, so only the selection rule orders them.  The scan keeps the NaN head (row 0),
# then takes the largest number (row 3), then the remaining head (row 2, NaN), then row 1.
NAN_ROWS = np.array([[0, 0, 10, 10, np.nan], [100, 0, 110, 10, 0.5], [200, 0, 210, 10, np.nan], [300, 0, 310, 10, 0.9]], F)
NAN_KEEP = [0, 3, 2, 1]


# ---- per-detection features --------------------------------------------------------------------------------------------
def features_ref(keep, keep_cnt, fc7, max_det):
    """frcnn_detect_features in numpy: keep [B, C, r], keep_cnt [B, C], fc7 [B*r, F] -> (feat [B, max_det, F], roi int32
    [B, max_det]).  Slot k of image b is the k-th entry of the concatenation over classes c >= 1 of keep[b, c, :keep_cnt[b, c]];
    slots past the count hold -1 and zeros."""
    B, C, r = keep.shape
    fdim = fc7.shape[1]
    feat = np.zeros((B, max_det, fdim), F)
    roi = np.full((B, max_det), -1, np.int32)
    for b in range(B):
        ids = np.concatenate([keep[b, c, :keep_cnt[b, c]] for c in range(1, C)]).astype(np.int64)[:max_det]
        roi[b, :ids.shape[0]] = ids
        feat[b, :ids.shape[0]] = fc7[b * r + ids]
    return feat, roi


def features_model(keep, keep_cnt, fc7, max_det, inclusive=False):
    """detect_features_kernel's slot lookup in numpy: the exclusive prefix s_off of the counts of classes 1 .. C-1, then for
    each slot < min(max_det, total) the last class c with s_off[c] <= slot by binary search, and keep[c, slot - s_off[c]].
    inclusive=True is a deliberate mistake (slot <= total) that reads one entry past the last class's count."""
    B, C, r = keep.shape
    feat = np.zeros((B, max_det, fc7.shape[1]), F)
    roi = np.full((B, max_det), -1, np.int32)
    for b in range(B):
        cnt = np.where(np.arange(C) >= 1, keep_cnt[b], 0)
        off = np.concatenate([[0], np.cumsum(cnt)])
        for slot in range(max_det):
            if not (slot <= off[C] if inclusive else slot < off[C]):
                continue
            lo, hi = 1, C
            while hi - lo > 1:
                mid = (lo + hi) >> 1
                lo, hi = (mid, hi) if off[mid] <= slot else (lo, mid)
            roi[b, slot] = keep[b, lo, slot - off[lo]]
            feat[b, slot] = fc7[b * r + roi[b, slot]]
    return feat, roi


def features_case(rng, C, r=50, B=3):
    """keep int32 [B, C, r] (every entry a valid RoI row, also past the counts, so that reading past a count shows), keep_cnt
    int32 [B, C] with class 0 holding a count it never emits.  C > 2: image 0 has 0..3 per class (about 1.5 C in all, above
    every max_det) with class 1 empty; image 1 totals 12 over classes 2, C/2 - 1 and C - 1, with C/2 empty; image 2 totals 5
    over classes 1 and 3C/5, with C - 1 empty.  C = 2: totals 0, 5 and 12.  Totals 5 and 12 end inside an 8-slot block and
    inside (0, max_det) for max_det 7 / 8 / 9 / 100."""
    keep = np.stack([np.stack([rng.permutation(r) for _ in range(C)]) for _ in range(B)]).astype(np.int32)
    cnt = np.zeros((B, C), np.int32)
    if C > 2:
        cnt[0] = rng.integers(0, 4, C)
        cnt[0, 1] = 0
        cnt[1, [2, C // 2 - 1, C - 1]] = [4, 1, 7]
        cnt[2, [1, 3 * C // 5]] = [2, 3]
    else:
        cnt[:, 1] = [0, 5, 12]
    cnt[:, 0] = 5
    return keep, cnt
