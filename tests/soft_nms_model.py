"""Vectorised numpy model of the Soft-NMS kernel's parallel formulation (block_soft_nms in csrc/nms.cu): per selection, the
decay of every later candidate at once, the prune count, the closed-form hole filling (the k-th pruned position below the new
end receives the k-th survivor at or above it, in descending position order) and the lowest-position argmax.  Every fp32
operation is a separate round-to-nearest numpy op; the gaussian weight is exp in fp64 rounded once."""
import numpy as np

F = np.float32
METHODS = ("linear", "gaussian", "hard")


def scan_argmax(s):
    """Offset of the definition's selection in s: m = 0, then m = p wherever s[m] < s[p].  A NaN head is selected; otherwise
    the first maximum of the non-NaN scores (np.argmax alone would take the first NaN anywhere)."""
    if np.isnan(s[0]):
        return 0
    return int(np.argmax(np.where(np.isnan(s), -np.inf, s)))


def soft_nms_model(dets, method="linear", sigma=0.5, nt=0.3, score_thresh=0.001):
    """dets [n,>=5] -> (rows [k,5] fp32 in selection order with decayed scores, keep [k] int32 rows of dets)."""
    assert method in METHODS
    d = np.asarray(dets, dtype=F)
    x1, y1, x2, y2, s = (d[:, c].copy() for c in range(5))
    idx = np.arange(d.shape[0], dtype=np.int32)
    cols = (x1, y1, x2, y2, s, idx)
    sigma, nt, thr = F(sigma), F(nt), F(score_thresh)
    one = F(1)
    N, i = d.shape[0], 0
    while i < N:
        m = i + scan_argmax(s[i:N])
        for c in cols:
            c[i], c[m] = c[m], c[i]
        L = i + 1
        seg = slice(L, N)
        iw = (np.fmin(x2[i], x2[seg]) - np.fmax(x1[i], x1[seg])) + one
        ih = (np.fmin(y2[i], y2[seg]) - np.fmax(y1[i], y1[seg])) + one
        ovl = (iw > 0) & (ih > 0)
        with np.errstate(all="ignore"):
            inter = iw * ih
            ta = ((x2[i] - x1[i]) + one) * ((y2[i] - y1[i]) + one)
            ua = (ta + ((x2[seg] - x1[seg]) + one) * ((y2[seg] - y1[seg]) + one)) - inter
            ov = inter / ua
            if method == "gaussian":
                w = np.exp(-((ov * ov) / sigma).astype(np.float64)).astype(F)
            elif method == "linear":
                w = np.where(ov > nt, one - ov, one).astype(F)
            else:
                w = np.where(ov > nt, F(0), one).astype(F)
            ns = np.where(ovl, w * s[seg], s[seg]).astype(F)
        dead = ovl & (ns < thr)
        s[seg] = ns
        B = N - int(dead.sum())
        pos = np.arange(L, N)
        holes = pos[dead & (pos < B)]                # ascending
        movers = pos[~dead & (pos >= B)][::-1]       # descending
        assert holes.shape == movers.shape
        for c in cols:
            c[holes] = c[movers]
        N = B
        i += 1
    return np.stack([x1[:N], y1[:N], x2[:N], y2[:N], s[:N]], axis=1).astype(F), idx[:N].copy()
