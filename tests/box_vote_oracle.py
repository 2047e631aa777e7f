"""Box-voting oracle for the tests (test infrastructure, built on oracle.pipeline's conventions):

  box_vote_c          the plain-C restatement of include/frcnn_b200.h's definition (tests/box_vote_c.c), compiled on first use
                      with -ffp-contract=off
  test_net_post_vote  lib/model/test.py:162-180 with greedy NMS or Soft-NMS, then box voting, the stable re-sort of score-changing
                      methods and the max_per_image cap, returning RoI indices too
"""
import ctypes
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from oracle import nms as ONMS
import soft_nms_oracle as SO

F = np.float32
METHODS = {"ID": 0, "AVG": 1, "IOU_AVG": 2, "GENERALIZED_AVG": 3, "QUASI_SUM": 4, "TEMP_AVG": 5}
STRICT, NO_PLUS_ONE, FP32_SUMS = 1, 2, 4          # oracle variants: deliberate mistakes the comparators must catch
_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "box_vote_c.c")
_LIB = None


def lib():
    """Compiled into the temporary directory (keyed by the source's hash), so it also works from a read-only tree."""
    global _LIB
    if _LIB is None:
        src = open(_SRC, "rb").read()
        path = os.path.join(tempfile.gettempdir(), "frcnn_box_vote_oracle_%d_%s.so" % (os.getuid(), hashlib.sha1(src).hexdigest()[:12]))
        if not os.path.exists(path):
            tmp = path + ".%d.tmp" % os.getpid()
            subprocess.check_call(["gcc", "-O2", "-std=c99", "-fPIC", "-shared", "-ffp-contract=off", "-o", tmp, _SRC, "-lm"])
            os.replace(tmp, path)
        L = ctypes.CDLL(path)
        fp = ctypes.POINTER(ctypes.c_float)
        ci, cf = ctypes.c_int, ctypes.c_float
        L.oracle_box_vote.argtypes = [fp, ci, fp, ci, cf, ci, cf, ci, fp]
        L.oracle_box_vote.restype = None
        _LIB = L
    return _LIB


def _rows(d):
    d = np.asarray(d, dtype=F)
    return np.ascontiguousarray(d[:, :5]) if d.size else np.zeros((0, 5), F)


def box_vote_c(top,all_dets, thresh=0.8, method="ID", beta=1.0, variant=0):
    """top [n,>=5], all_dets [m,>=5] -> fp32 [n,5] voted rows in top's order.  thresh and beta are rounded to fp32 once, as the
    product does."""
    fp = ctypes.POINTER(ctypes.c_float)
    t, a = _rows(top), _rows(all_dets)
    out = np.zeros((max(t.shape[0], 1), 5), F)
    lib().oracle_box_vote(t.ctypes.data_as(fp), t.shape[0], a.ctypes.data_as(fp), a.shape[0], float(F(thresh)), METHODS[method],
                          float(F(beta)), int(variant), out.ctypes.data_as(fp))
    return out[:t.shape[0]].copy()


def stable_resort(rows):
    """Order of a score-changing method's class list: descending voted score, ties in NMS order."""
    return np.argsort(-rows[:, 4].astype(np.float64), kind="stable")


def test_net_post_vote(scores, boxes, vote, nt=0.3, max_per_image=100, thresh=0.0, soft=None, use_gpu_nms=True, variant=0,
                       weights="original", resort=stable_resort, vote_fn=box_vote_c):
    """Per class j >= 1: the candidates (rows with scores[:, j] > thresh, ascending RoI order), greedy NMS (nt, the gpu_nms or
    cpu_nms predicate) or Soft-NMS(soft = (method, sigma, prune)), box voting(vote = (VOTE_TH, SCORING_METHOD, BETA)) of the
    kept rows against the candidates, for a score-changing method the stable re-sort, then the max_per_image cap ->
    (list over classes of fp32 [k,5], list over classes of int64 [k] RoI indices).  weights='decayed' votes against the
    Soft-NMS output instead of the candidates (a deliberate mistake for the tests); resort / vote_fn replace the re-sort and
    the vote (vote_fn(top, all, thresh, method, beta, variant) -> [n,5]) for the tests' restatements."""
    vth, method, beta = vote
    C = scores.shape[1]
    out, idx = [np.zeros((0, 5), F)], [np.zeros(0, np.int64)]
    for j in range(1, C):
        inds = np.where(scores[:, j] > F(thresh))[0]
        dets = np.hstack([boxes[inds, 4 * j:4 * j + 4], scores[inds, j][:, None]]).astype(F)
        if soft is None:
            keep = ONMS.nms_plus1_c(dets, nt, inclusive=not use_gpu_nms)
            rows = dets[keep]
        else:
            rows, keep = SO.soft_nms_c(dets, soft[0], soft[1], nt, soft[2])
        voters = rows if weights == "decayed" else dets
        rows = vote_fn(rows, voters, vth, method, beta, variant)
        ri = inds[keep].astype(np.int64)
        if method != "ID":
            o = resort(rows)
            rows, ri = rows[o], ri[o]
        out.append(rows)
        idx.append(ri)
    if max_per_image > 0:
        allsc = np.hstack([d[:, 4] for d in out[1:]]) if C > 1 else np.zeros(0, F)
        if allsc.shape[0] > max_per_image:
            th = np.sort(allsc)[-max_per_image]
            sel = [d[:, 4] >= th for d in out[1:]]
            out = [out[0]] + [d[s] for d, s in zip(out[1:], sel)]
            idx = [idx[0]] + [i[s] for i, s in zip(idx[1:], sel)]
    return out, idx
