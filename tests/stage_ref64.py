"""float64 references, per-element bounds, comparators and edge-case generators for the detection-tail stage tests
(`test_stage_edges_gpu.py`, `test_stages_gpu.py`; their teeth are shown on the CPU by `test_stage_ref64.py`).

Stages whose kernel claims the oracle's fp32 op order (box decodes, de-normalised deltas, crop_and_resize, the per-class NMS
records) are compared value for value (`check_exact`: +0 == -0, NaN == NaN).  The softmaxes and the spatial mean use `expf`
or a different summation order than numpy, so they are held to a per-element bound around a float64 truth, derived below.
u = 2^-24 is the fp32 unit roundoff; 2^-149 the smallest fp32 subnormal."""
import numpy as np
import torch

F = np.float32
U = 2.0 ** -24
TINY = 2.0 ** -149


def gamma(k):
    """Classical bound of k rounded operations: |fl - exact| <= gamma_k * (sum of |terms|), gamma_k = k u / (1 - k u)."""
    return k * U / (1 - k * U)


# ---- guard-banded device outputs ------------------------------------------------------------------------------------
GUARD = 64
SENTINEL = np.int32(0x7fa5a5a5)


def guarded_out(shape, fill=float("nan")):
    """(buf, out): `out` is a `fill`-prefilled fp32 view of `shape` between GUARD sentinel words on each side."""
    numel = int(np.prod(shape))
    buf = torch.full((numel + 2 * GUARD,), int(SENTINEL), dtype=torch.int32, device="cuda")
    out = buf.view(torch.float32)[GUARD:GUARD + numel].view(shape)
    out.fill_(fill)
    return buf, out


def check_guarded(buf, numel, what="output"):
    b = buf.cpu().numpy()
    assert (b[:GUARD] == SENTINEL).all() and (b[GUARD + numel:] == SENTINEL).all(), "store outside the %s" % what


# ---- comparators ----------------------------------------------------------------------------------------------------
def check_exact(got, want, what=""):
    """Same value in every element (+0 == -0 and NaN == NaN count as equal)."""
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape, "%s: shape %s, want %s" % (what, got.shape, want.shape)
    bad = ~((got == want) | (np.isnan(got) & np.isnan(want)))
    if bad.any():
        i = np.unravel_index(np.argmax(bad), bad.shape)
        raise AssertionError("%s: %d of %d elements differ, first at %s: got %r, want %r"
                             % (what, int(bad.sum()), bad.size, i, got[i], want[i]))


def check_boxes_exact(got, want, what=""):
    """Box coordinates [..., 4k], value for value, except the boxes whose reference holds a NaN (an inf - inf in the decode:
    numpy propagates it, the kernels' fminf / fmaxf clip return the bound; DESIGN §2).  Returns the excluded-box mask."""
    g = np.asarray(got).reshape(-1, 4)
    w = np.asarray(want).reshape(-1, 4)
    nan = np.isnan(w).any(axis=1)
    check_exact(g[~nan], w[~nan], what)
    return nan


def check_bounded(got, want64, bound, what=""):
    """|got - want64| <= bound in every element (a non-finite output fails); returns max err / bound."""
    got64 = np.asarray(got, dtype=np.float64)
    assert got64.shape == want64.shape, "%s: shape %s, want %s" % (what, got64.shape, want64.shape)
    assert np.isfinite(got64).all(), "%s: non-finite output" % what
    err = np.abs(got64 - want64)
    ratio = err / bound
    if not (err <= bound).all():
        i = np.unravel_index(np.argmax(ratio), ratio.shape)
        raise AssertionError("%s: max err/bound %.3g at %s: got %r, want %r, bound %.3g"
                             % (what, ratio[i], i, got64[i], want64[i], bound[i]))
    return float(ratio.max())


# ---- softmax ----------------------------------------------------------------------------------------------------------
def cls_depth(C):
    """Additions on the longest path of cls_finish's sum: ceil(C/32) per lane (strided over the row), then 5 xor shuffles."""
    return -(-C // 32) + 5


RPN_DEPTH = 1          # rpn_decode's 2-way softmax: e_bg + e_fg


def softmax_ref(x, depth):
    """float64 softmax over the last axis of fp32 logits `x`, and the per-element bound of a kernel that evaluates
        d_j = fl(x_j - m)  (m = max_j x_j, exact),  e_j = expf(d_j),  s = sum_j e_j  (a tree of depth `depth`),  p_i = fl(e_i / s)

    Bound.  With d_j = x_j - m exact and K_i = |d_i| + max_j|d_j| + 4 + 4 + depth + 1:
      * the rounded subtraction d^_j = d_j (1 + δ), |δ| <= u, changes exp(d_j) by the factor exp(d_j δ): |d_j| u relative;
      * expf is within 2 ulp (CUDA programming guide, no fast-math), and 1 ulp <= 2u |y| for a normal y: 4u relative;
      * so every e_j is exp(d_j) within |d_j| u + 4u (numerator: |d_i| + 4; summands: at most max_j|d_j| + 4);
      * a sum of positive terms along a tree of depth `depth` is within gamma_depth ~ depth u relative;
      * the division adds u.
    These compose to |p - p64| <= p64 (exp(K u) - 1) <= p64 K u (1 + 2 K u) for K u <= 2^-11 (asserted).  Subnormal results:
    an expf below 2^-126 is off by up to 2 * 2^-149 absolute, which stays <= 2 * 2^-149 after the division by s >= 1
    (s holds exp(0) = 1 for the maximum), and a subnormal quotient rounds by up to 0.5 * 2^-149; so the floor is
    2.5 * 2^-149 (subnormal summands move s relatively by < C 2^-148, far inside the (1 + 2 K u) slack).  In full:
        |p - p64| <= p64 K u (1 + 2 K u) + 2.5 * 2^-149
    Returns (p64, bound)."""
    x64 = np.asarray(x, dtype=np.float64)
    d = x64 - x64.max(axis=-1, keepdims=True)
    e = np.exp(d)
    p64 = e / e.sum(axis=-1, keepdims=True)
    ad = np.abs(d)
    ku = (ad + ad.max(axis=-1, keepdims=True) + 4 + 4 + depth + 1) * U
    assert ku.max() <= 2.0 ** -11, "logit spread outside the bound's first-order regime"
    return p64, p64 * ku * (1 + 2 * ku) + 2.5 * TINY


def rpn_fg_ref(bg, fg):
    """float64 fg probability of the pair (bg, fg) and its bound (softmax_ref with depth 1)."""
    p64, bound = softmax_ref(np.stack([np.asarray(bg, F), np.asarray(fg, F)], axis=-1), RPN_DEPTH)
    return p64[..., 1], bound[..., 1]


# ---- spatial mean -----------------------------------------------------------------------------------------------------
def spatial_mean_ref(x):
    """x fp32 [r, h, w, c] -> (float64 mean over h*w, bound) for a kernel that adds the hw = h*w values one by one from 0
    (hw - 1 rounded adds; the first is exact) and divides once by hw.

    Bound.  The sum is within gamma_{hw-1} sum|x| of the exact one; dividing by hw (exact in fp32) and rounding adds
    u |s / hw| <= u |mean64| + u gamma_{hw-1} sum|x| / hw, and gamma_{hw-1} (1 + u) <= gamma_hw, so
        |mean - mean64| <= gamma_hw * sum|x| / hw + u |mean64|."""
    r, h, w, c = x.shape
    hw = h * w
    x64 = np.asarray(x, dtype=np.float64).reshape(r, hw, c)
    m64 = x64.sum(axis=1) / hw
    return m64, gamma(hw) * np.abs(x64).sum(axis=1) / hw + U * np.abs(m64)


# ---- logit rows -------------------------------------------------------------------------------------------------------
ROW_KINDS = ("equal", "spike100", "offset+1e4", "offset-1e4", "sigma3", "sigma30")


def logit_rows(rng, r, C, kinds=ROW_KINDS):
    """fp32 [r, C] logits, row i of kind kinds[i % len(kinds)] -> (x, kind index per row).
      equal       every logit the same value: p = 1/C
      spike100    N(0, 0.5^2) and one class 100 above the row's maximum: the others land near 1e-44 (fp32 subnormals)
      offset±1e4  ±1e4 + N(0, 1): the logits carry 2^-10 quantisation, the differences stay exact
      sigma3/30   N(0, 3^2) and N(0, 30^2): probabilities from 1e-6 down to underflow"""
    x = np.empty((r, C), np.float64)
    kind = np.arange(r) % len(kinds)
    for k, name in enumerate(kinds):
        rows = np.flatnonzero(kind == k)
        n = rows.shape[0]
        if name == "equal":
            v = np.repeat(rng.standard_normal((n, 1)) * 5, C, axis=1)
        elif name == "spike100":
            v = rng.standard_normal((n, C)) * 0.5
            v[np.arange(n), rng.integers(0, C, n)] = v.max(axis=1) + 100
        elif name.startswith("offset"):
            v = float(name[6:]) + rng.standard_normal((n, C))
        elif name.startswith("sigma"):
            v = rng.standard_normal((n, C)) * float(name[5:])
        else:
            raise ValueError(name)
        x[rows] = v
    return x.astype(F), kind


# ---- de-normalised deltas ---------------------------------------------------------------------------------------------
BBOX_STDS = (0.1, 0.13, 0.2, 0.27)          # four distinct values: an x/y or w/h swap changes the output
BBOX_MEANS = (0.011, -0.023, 0.031, -0.047)  # four distinct non-zero values: a wrong or missing mean changes the output


def denorm_ref(deltas, stds, means):
    """network.py:431-432 on a fp32 tensor: fl(fl(d * std) + mean), std / mean tiled over the classes."""
    C = deltas.shape[1] // 4
    s = np.tile(np.asarray(stds, F), C)
    m = np.tile(np.asarray(means, F), C)
    return ((deltas * s).astype(F) + m).astype(F)


# ---- box deltas at the edges ------------------------------------------------------------------------------------------
EDGE_DWH = (-104.0, -20.0, 20.0, 88.7, 89.0)    # exp -> 0 (below half the smallest subnormal), tiny, large, finite max, inf
EDGE_DXY = (1e30, -1e30)                          # centre far off either side: x1 > W - 1 or x2 < 0 after the decode


def edge_deltas(rng, n, K, p_edge=0.35, sigma=0.5):
    """fp32 [n, 4K] deltas: N(0, sigma^2), each coordinate replaced by an edge value with probability p_edge; the first rows
    hold every edge value in the (dx, dw) and (dy, dh) slots of class 0 so that each is present at any n >= 7."""
    d = rng.standard_normal((n, K, 4)) * sigma
    m = rng.random((n, K, 4)) < p_edge
    xy = rng.choice(EDGE_DXY, (n, K, 4))
    wh = rng.choice(EDGE_DWH, (n, K, 4))
    d[..., :2] = np.where(m[..., :2], xy[..., :2], d[..., :2])
    d[..., 2:] = np.where(m[..., 2:], wh[..., 2:], d[..., 2:])
    for j, v in enumerate(EDGE_DWH[:min(n, 5)]):
        d[j, 0, 2:] = v
    for j, v in enumerate(EDGE_DXY[:max(min(n - 5, 2), 0)]):
        d[5 + j, 0, :2] = v
    return d.reshape(n, 4 * K).astype(F)


def nan_deltas(n, K):
    """fp32 [n, 4K] deltas whose decode hits inf - inf: dx, dy = ±3e38 (pcx = ±inf for w >= 2) with dw, dh = 89
    (pw = inf).  Row 2i: x1 = inf - inf = NaN, x2 = +inf; row 2i+1: x1 = -inf, x2 = -inf + inf = NaN."""
    d = np.zeros((n, K, 4), F)
    d[:, :, :2] = np.where((np.arange(n) % 2 == 0)[:, None, None], F(3e38), F(-3e38))
    d[:, :, 2:] = 89.0
    return d.reshape(n, 4 * K)


# ---- crop boxes -------------------------------------------------------------------------------------------------------
def crop_last_sample(c1, c2, dim, crop):
    """The fp32 sample coordinates of crop_and_resize (network.py's normalisation, then TF's un-normalisation) for a box
    edge pair (c1, c2) in blob pixels on a map of `dim` cells: -> (first, last) sample."""
    n = (F(dim) - F(1)) * F(16)
    a, b = F(c1) / n, F(c2) / n
    step = (b - a) * F(dim - 1) / F(crop - 1)
    return a * F(dim - 1), a * F(dim - 1) + F(crop - 1) * step


def boundary_edge(dim, crop):
    """A blob coordinate c2 >= 0 such that the box edge pair (0, c2) puts its last sample exactly on dim - 1 (the largest
    in-map coordinate, where floor == ceil == dim - 1)."""
    up = down = F((dim - 1) * 16)
    for _ in range(1024):
        for v in (up, down):
            if crop_last_sample(0, v, dim, crop)[1] == F(dim - 1):
                return F(v)
        up, down = np.nextafter(up, F(np.inf)), np.nextafter(down, F(0))
    raise AssertionError("no boundary edge for dim %d crop %d" % (dim, crop))


def crop_boxes(rng, fh, fw, n, crop):
    """fp32 [n, 4] RoI boxes (x1, y1, x2, y2) in blob pixels for a fh x fw map (extent X = (fw-1)*16, Y = (fh-1)*16):
    a fixed head of edge boxes, then random boxes inside and around the map.  The head: straddling and fully outside each
    of the four sides, inverted in x, y and both, zero-size (inside and outside), the full map, and boxes whose last
    sample lands exactly on fw - 1 / fh - 1 for this crop size."""
    X, Y = float((fw - 1) * 16), float((fh - 1) * 16)
    xb, yb = float(boundary_edge(fw, crop)), float(boundary_edge(fh, crop))
    head = [
        [-0.4 * X, 0.2 * Y, 0.5 * X, 0.7 * Y], [0.5 * X, 0.2 * Y, 1.4 * X, 0.7 * Y],         # straddle left / right
        [0.2 * X, -0.4 * Y, 0.7 * X, 0.5 * Y], [0.2 * X, 0.5 * Y, 0.7 * X, 1.4 * Y],         # straddle top / bottom
        [-3 * X, 0.1 * Y, -0.5 * X, 0.9 * Y], [1.2 * X, 0.1 * Y, 4 * X, 0.9 * Y],            # fully left / right
        [0.1 * X, -3 * Y, 0.9 * X, -0.2 * Y], [0.1 * X, 1.1 * Y, 0.9 * X, 3 * Y],            # fully above / below
        [-2 * X, -2 * Y, 3 * X, 3 * Y],                                                      # around the whole map
        [0.8 * X, 0.1 * Y, 0.2 * X, 0.9 * Y], [0.1 * X, 0.8 * Y, 0.9 * X, 0.2 * Y],          # inverted in x / y
        [0.9 * X, 0.9 * Y, -0.3 * X, -0.3 * Y],                                              # inverted in both, leaving the map
        [0.3 * X, 0.6 * Y, 0.3 * X, 0.6 * Y], [1.5 * X, -0.5 * Y, 1.5 * X, -0.5 * Y],        # zero-size inside / outside
        [0, 0, X, Y], [0, 0, xb, yb], [0, 0.3 * Y, xb, 0.6 * Y], [0.3 * X, 0, 0.6 * X, yb],  # full map; last sample on the edge
    ]
    head = np.asarray(head, np.float64)[:n]
    m = n - head.shape[0]
    xy = rng.uniform(-0.5, 1.5, (m, 2)) * (X, Y)
    wh = rng.uniform(-0.3, 1.2, (m, 2)) * (X, Y)
    rest = np.hstack([xy, xy + wh])
    return np.vstack([head, rest]).astype(F)


# ---- per-class NMS + cap ---------------------------------------------------------------------------------------------
QUANT_LEVELS = (0.0, 0.05, 0.125, 0.25, 0.5, 0.75)
SPARSE_TOP = (0.5, 0.2, 0.15, 0.1, 0.04, 0.01)     # level weights that keep the top levels rare (a few hundred records)


def quantised_probs(rng, R, C, levels=QUANT_LEVELS, weights=None):
    """fp32 [R, C] table whose entries take a few values: per-class and cross-class score ties everywhere."""
    return rng.choice(np.asarray(levels, F), size=(R, C), p=weights)


def clustered_pred(rng, R, C, size=500.0):
    """fp32 [R, 4C] integer boxes around R // 8 centres (jitter ±15 px): overlapping sets, so a tie decides who survives."""
    k = max(R // 8, 1)
    xy = rng.uniform(0, size, (k, 2))
    wh = rng.uniform(20, 200, (k, 2))
    centres = np.hstack([xy, xy + wh])[rng.integers(0, k, R)]
    pred = centres[:, None, :] + rng.uniform(-15, 15, (R, C, 4))
    return np.round(pred.reshape(R, 4 * C)).astype(F)


def grid_pred(R, C):
    """fp32 [R, 4C]: RoI i owns a 20 x 20 box in its own 30-px grid cell, the same for every class -- no two RoIs overlap,
    so every candidate survives its class NMS and the cap alone decides what is kept."""
    i = np.arange(R)
    x, y = (i % 64) * 30.0, (i // 64) * 30.0
    b = np.stack([x, y, x + 19, y + 19], axis=1)
    return np.tile(b, (1, C)).astype(F)


def cap_tie_probs(rng, R, C, n_above, n_tied, hi=0.875, tie=0.5):
    """fp32 [R, C]: n_above (RoI, fg class) cells at `hi`, n_tied cells at `tie`, every other cell 0 (never a candidate)."""
    p = np.zeros((R, C), F)
    cells = rng.choice(R * (C - 1), n_above + n_tied, replace=False)
    r, c = cells // (C - 1), 1 + cells % (C - 1)
    p[r[:n_above], c[:n_above]] = hi
    p[r[n_above:], c[n_above:]] = tie
    return p


def flat_records(per_class):
    """test_net_post's per-class lists -> [n, 6] rows (x1, y1, x2, y2, score, class) in class order: the device record."""
    rows = [np.hstack([d, np.full((d.shape[0], 1), j, F)]) for j, d in enumerate(per_class) if d.shape[0]]
    return np.vstack(rows).astype(F) if rows else np.zeros((0, 6), F)


def check_records(det, nd, cnt, per_class, max_det, what=""):
    """Device records against the oracle's per-class lists: the TRUE count, the first min(count, max_det) rows value for
    value (boxes, scores, classes and order) and the per-class kept counts."""
    want = flat_records(per_class)
    assert nd == want.shape[0], "%s: %d records, want %d" % (what, nd, want.shape[0])
    k = min(nd, max_det)
    check_exact(np.asarray(det)[:k], want[:k], what + " records")
    if cnt is not None:
        assert [int(c) for c in cnt] == [d.shape[0] for d in per_class], "%s: per-class counts differ" % what
