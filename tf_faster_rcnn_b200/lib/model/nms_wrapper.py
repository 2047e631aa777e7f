"""`nms(dets, thresh, force_cpu=False)` with the reference's contract (lib/model/nms_wrapper.py:15-23):
empty input -> []; otherwise indices into the UNSORTED `dets`, in descending-score order.

Both of the reference's predicates run on the GPU here (there is no CPU implementation):
  cfg.USE_GPU_NMS and not force_cpu -> gpu_nms semantics ('+1' areas, suppress when IoU >  thresh)
  otherwise                         -> cpu_nms semantics ('+1' areas, suppress when ovr >= thresh)
The host argsort mirrors gpu_nms.pyx:25-28 / cpu_nms.pyx:25 but is stable (ties: lower index first).

`soft_nms(...)` is an extension beyond the reference with Detectron's contract (Soft-NMS, Bodla et al. 2017), also on the GPU, and
so is `box_voting(...)` (Detectron's TEST.BBOX_VOTE)."""
import numpy as np

from model.config import cfg
from tf_faster_rcnn_b200 import engine, ops


def nms(dets, thresh, force_cpu=False):
    if dets.shape[0] == 0:
        return []
    dets = np.ascontiguousarray(dets, dtype=np.float32)
    order = np.argsort(-dets[:, 4], kind="stable")
    t32, flags = engine.nms_threshold(thresh, bool(cfg.USE_GPU_NMS) and not force_cpu)
    keep = ops.nms_host(dets[order], t32, flags, device_id=-1)   # the process's current device (rank-local under torchrun)
    return list(order[keep])


def soft_nms(dets, sigma=0.5, overlap_thresh=0.3, score_thresh=0.001, method="linear"):
    """Soft-NMS of dets [n, 5] (x1, y1, x2, y2, score), taken in row order, semantics of include/frcnn_b200.h
    (frcnn_soft_nms_host).  method: 'linear' | 'gaussian' | 'hard'; every parameter is used as fp32.
    -> (dets_out [k, 5] fp32 in selection order with the decayed scores, keep [k] indices into dets).  Empty input ->
    (zeros((0, 5)), [])."""
    code, sigma32, thresh32 = engine.soft_nms_args(method, sigma, score_thresh)
    if dets.shape[0] == 0:
        return np.zeros((0, 5), np.float32), []
    return ops.soft_nms_host(dets, code, sigma32, float(np.float32(overlap_thresh)), thresh32, device_id=-1)


def box_voting(top_dets, all_dets, thresh, scoring_method="ID", beta=1.0):
    """Detectron's box voting on the GPU (frcnn_box_vote_host, semantics of include/frcnn_b200.h): each row of top_dets [n, 5]
    (x1, y1, x2, y2, score) gets the score-weighted mean box of the rows of all_dets [m, 5] that overlap it by >= thresh, and
    with a scoring_method other than 'ID' ('AVG', 'IOU_AVG', 'GENERALIZED_AVG', 'QUASI_SUM', 'TEMP_AVG') a new score.
    thresh and beta are used as fp32.  -> fp32 [n, 5] in top_dets' row order (a row with no voter keeps its values)."""
    t32, code, b32 = engine.box_vote_args(thresh, scoring_method, beta)
    if top_dets.shape[0] == 0:
        return np.zeros((0, 5), np.float32)
    return ops.box_vote_host(top_dets, all_dets, t32, code, b32, device_id=-1)
