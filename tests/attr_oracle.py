"""float64 restatement of the attribute head on the bottom-up regions (include/frcnn_b200.h, frcnn_regions_attr_embed), its
per-element bounds and comparators.  Per region with fc7 row x, class logits z (C columns, background included):
  1. c = argmax_rule(z)                                  numpy's argmax: the first NaN, else the first maximal column
  2. e = cls_embedding[c]
  3. h = relu([x ; e] . W_fc_attr + b_fc_attr)          fc7 first
  4. s = h . W_attr_score + b_attr_score, attr_prob = softmax(s)
  5. attributes = 1 + argmax_rule(attr_prob[1:]), attr_conf = attr_prob[attributes]
The keyword knobs of `head64` exist for the mutant tests (tests/test_attributes.py): each names one plausible mistake."""
import numpy as np

import conv_split_model as M
import stage_ref64 as S

F = np.float32
U = 2.0 ** -24
ALPHA = 8.0            # the conv tests' fp32-grade factor (tests/test_conv_gpu.py (b))
TINY16 = 2.0 ** -14    # below it the F16X3 activation split keeps fewer than 22 bits


def argmax_rule(row):
    """np.argmax of one row, restated: the index of the first NaN if the row holds one, else of the first maximal value."""
    row = np.asarray(row)
    nan = np.flatnonzero(np.isnan(row))
    if nan.size:
        return int(nan[0])
    return int(np.flatnonzero(row == row.max())[0])


def argmax_last(row):
    """Mutant of argmax_rule: ties go to the last maximal column."""
    row = np.asarray(row)
    nan = np.flatnonzero(np.isnan(row))
    if nan.size:
        return int(nan[0])
    return int(np.flatnonzero(row == row.max())[-1])


def embed(cls_score, table, argmax=argmax_rule, first=0):
    """Steps 1-2 on the rows of cls_score [n, C]: (classes [n] int, embedding rows [n, E] fp32).  first=1 is the
    foreground-only mutant."""
    c = np.array([first + argmax(r[first:]) for r in np.asarray(cls_score)], dtype=np.int64).reshape(-1)
    return c, np.asarray(table)[c]


def fc64(x, w, b, relu):
    """One FC on the conv kernel against float64: x [n, K] fp32 (the device's own inputs), w [K, N], b [N] ->
    (y64 [n, N], bound [n, N]).  The bound is the conv tests' F16X3 / TF32X3 one for a layer with a bias and no scale:
        ALPHA u S + 2u (|a| + 2|a + b|),  S = |x| . |w|,
    plus ALPHA times the split's own loss on activations below 2^-14 (conv_split_model.activation_error), as net_ref64 does."""
    x64 = np.asarray(x, np.float64)
    w64 = np.asarray(w, np.float64)
    a = x64 @ w64
    y = a + np.asarray(b, np.float64)
    bound = ALPHA * U * (np.abs(x64) @ np.abs(w64)) + 2 * U * (np.abs(a) + 2 * np.abs(y))
    small = (np.abs(x64) < TINY16) & (x64 != 0)
    if small.any():
        e = np.where(small, M.activation_error(np.asarray(x, F), M.F16X3) * np.abs(x64), 0.0)
        bound += ALPHA * (np.nan_to_num(e) @ np.abs(w64))
    return (np.maximum(y, 0.0) if relu else y), bound


def softmax64(score, A):
    """attr_prob of the fp32 logits score[:, :A]: (p64, bound), frcnn_attr_finish's arithmetic is cls_finish's
    (stage_ref64.softmax_ref at cls_depth(A))."""
    return S.softmax_ref(np.asarray(score, F)[:, :A], S.cls_depth(A))


def pick(prob, argmax=argmax_rule, first=1):
    """Step 5 on the rows of prob [n, A]: (attributes [n] int, attr_conf [n] of prob's dtype).  first=0 is the mutant that
    counts attributes from column 0."""
    prob = np.asarray(prob)
    a = np.array([first + argmax(r[first:]) for r in prob], dtype=np.int64).reshape(-1)
    return a, prob[np.arange(prob.shape[0]), a]


def head64(fc7, cls_score, w, scope, argmax=argmax_rule, fg_only=False, emb_first=False, relu=True, attr_first=1):
    """Steps 1-5 in float64 from fp32 inputs: fc7 [n, F], cls_score [n, C], w the TF-named variables.  -> dict(classes, emb,
    hidden, score, attr_prob, attributes, attr_conf), every layer on the float64 output of the one before."""
    classes, emb = embed(cls_score, w[scope + "/cls_embedding/weights"], argmax, 1 if fg_only else 0)
    x = np.concatenate([emb, fc7] if emb_first else [fc7, emb], axis=1).astype(np.float64)
    w1 = np.asarray(w[scope + "/fc_attr/weights"], np.float64)
    h = x @ w1 + np.asarray(w[scope + "/fc_attr/biases"], np.float64)
    if relu:
        h = np.maximum(h, 0.0)
    s = h @ np.asarray(w[scope + "/attr_score/weights"], np.float64) + np.asarray(w[scope + "/attr_score/biases"], np.float64)
    e = np.exp(s - s.max(axis=1, keepdims=True))
    p = e / e.sum(axis=1, keepdims=True)
    attributes, conf = pick(p, argmax, attr_first)
    return dict(classes=classes, emb=emb, hidden=h, score=s, attr_prob=p, attributes=attributes, attr_conf=conf)


def check_attributes(got_prob, got_attr, got_conf, p64, bound, what=""):
    """attr_prob within `bound` of p64; attributes equal to the float64 choice wherever its best probability beats every other
    column of attr_prob[1:] by more than both bounds; and exactly the rule on the device's own probabilities, attr_conf their
    value at that column.  Returns (max err/bound, rows whose choice was decided by the margin)."""
    ratio = S.check_bounded(got_prob, p64, bound, what + " attr_prob")
    want_attr, _ = pick(p64)
    rows = np.arange(p64.shape[0])
    q = p64[:, 1:].copy()
    qb = bound[:, 1:]
    top = want_attr - 1
    q_top, b_top = q[rows, top], qb[rows, top]
    q[rows, top] = -np.inf
    clear = (q_top - b_top > (q + qb).max(axis=1)) if q.shape[1] > 1 else np.ones(len(rows), bool)
    bad = clear & (np.asarray(got_attr) != want_attr)
    assert not bad.any(), "%s attributes: %d rows differ where the margin exceeds the bound, first %d: got %d, want %d" % (
        what, int(bad.sum()), int(np.argmax(bad)), int(np.asarray(got_attr)[np.argmax(bad)]), int(want_attr[np.argmax(bad)]))
    own_attr, own_conf = pick(np.asarray(got_prob, F))
    S.check_exact(np.asarray(got_attr), own_attr, what + " attributes (the rule on the device's own attr_prob)")
    S.check_exact(np.asarray(got_conf), own_conf, what + " attr_conf")
    return ratio, int(clear.sum())
