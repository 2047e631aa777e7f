"""Soft-NMS oracle for the tests (test infrastructure, built on oracle.pipeline's conventions):

  soft_nms_c          the plain-C sequential restatement (tests/soft_nms_c.c), compiled on first use with -ffp-contract=off
  test_net_post_soft  lib/model/test.py:162-180 with Soft-NMS as the per-class stage, returning RoI indices too
"""
import ctypes
import hashlib
import os
import subprocess
import tempfile

import numpy as np

F = np.float32
METHODS = {"linear": 0, "gaussian": 1, "hard": 2}
_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "soft_nms_c.c")
_LIB = None


def lib():
    """The oracle is compiled into the temporary directory (keyed by the source's hash), so it also works from a read-only tree."""
    global _LIB
    if _LIB is None:
        src = open(_SRC, "rb").read()
        path = os.path.join(tempfile.gettempdir(), "frcnn_soft_nms_oracle_%d_%s.so" % (os.getuid(), hashlib.sha1(src).hexdigest()[:12]))
        if not os.path.exists(path):
            tmp = path + ".%d.tmp" % os.getpid()
            subprocess.check_call(["gcc", "-O2", "-std=c99", "-fPIC", "-shared", "-ffp-contract=off", "-o", tmp, _SRC, "-lm"])
            os.replace(tmp, path)
        L = ctypes.CDLL(path)
        fp, ip = ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_int)
        L.oracle_soft_nms.argtypes = [fp, ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_float, ctypes.c_float, fp, ip]
        L.oracle_soft_nms.restype = ctypes.c_int
        L.oracle_soft_nms_variant.argtypes = L.oracle_soft_nms.argtypes + [ctypes.c_int]
        L.oracle_soft_nms_variant.restype = ctypes.c_int
        _LIB = L
    return _LIB


# oracle variants: deliberate mistakes that the float64 comparator of post_ref64.py must catch
GE_NT, NO_PLUS_ONE, PRUNE_UNTOUCHED, TIES_HIGH, STABLE_COMPACT, GAUSS_NO_SQUARE = 1, 2, 4, 8, 16, 32


def soft_nms_c(dets, method="linear", sigma=0.5, nt=0.3, score_thresh=0.001, variant=0):
    """dets [n,>=5] -> (rows [k,5] fp32 in selection order with decayed scores, keep [k] int32 rows of dets).  Parameters are
    rounded to fp32 once, as the product does."""
    d = np.ascontiguousarray(np.asarray(dets, dtype=F)[:, :5])
    n = d.shape[0]
    out = np.zeros((max(n, 1), 5), F)
    keep = np.zeros(max(n, 1), np.int32)
    k = lib().oracle_soft_nms_variant(d.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), n, METHODS[method], float(F(sigma)),
                                      float(F(nt)), float(F(score_thresh)), out.ctypes.data_as(ctypes.POINTER(ctypes.c_float)),
                                      keep.ctypes.data_as(ctypes.POINTER(ctypes.c_int)), int(variant))
    return out[:k].copy(), keep[:k].copy()


def test_net_post_soft(scores, boxes, soft, nt=0.3, max_per_image=100, thresh=0.0):
    """Per class j >= 1: the rows with scores[:, j] > thresh in ascending RoI order, Soft-NMS(soft = (method, sigma,
    score_thresh), overlap threshold nt), then the max_per_image cap -> (list over classes of fp32 [k,5], list over classes of
    int64 [k] RoI indices)."""
    method, sigma, prune = soft
    C = scores.shape[1]
    out, idx = [np.zeros((0, 5), F)], [np.zeros(0, np.int64)]
    for j in range(1, C):
        inds = np.where(scores[:, j] > F(thresh))[0]
        dets = np.hstack([boxes[inds, 4 * j:4 * j + 4], scores[inds, j][:, None]]).astype(F)
        rows, keep = soft_nms_c(dets, method, sigma, nt, prune)
        out.append(rows)
        idx.append(inds[keep].astype(np.int64))
    if max_per_image > 0:
        allsc = np.hstack([d[:, 4] for d in out[1:]]) if C > 1 else np.zeros(0, F)
        if allsc.shape[0] > max_per_image:
            th = np.sort(allsc)[-max_per_image]
            sel = [d[:, 4] >= th for d in out[1:]]
            out = [out[0]] + [d[s] for d, s in zip(out[1:], sel)]
            idx = [idx[0]] + [i[s] for i, s in zip(idx[1:], sel)]
    return out, idx
