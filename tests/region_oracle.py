"""Oracle additions for the region-feature tests (test infrastructure, built on oracle.pipeline's stages):

  test_net_post_indexed  oracle.pipeline.test_net_post that also returns the RoI index of every kept row
  score_boxes            Fast R-CNN scoring of caller boxes (TEST.HAS_RPN = False): crop_pool, head_to_tail,
                         region_classification and im_detect_post on rois = fp32(box * fp32(scale))
"""
import numpy as np

from oracle import nets as N
from oracle import nms as NMS
from oracle import pipeline as P

F = np.float32


def test_net_post_indexed(scores, boxes, o=None, thresh=0.0):
    """lib/model/test.py:162-180 -> (list over classes of fp32 [k,5], list over classes of int64 [k] RoI indices = rows of
    scores / boxes).  Rows equal oracle.pipeline.test_net_post's."""
    o = o or P.opts()
    C = scores.shape[1]
    out, idx = [np.zeros((0, 5), F)], [np.zeros(0, np.int64)]
    for j in range(1, C):
        inds = np.where(scores[:, j] > thresh)[0]
        dets = np.hstack([boxes[inds, 4 * j:4 * j + 4], scores[inds, j][:, None]]).astype(F)
        keep = NMS.nms_plus1_c(dets, o["nms_thresh"], inclusive=not o["use_gpu_nms"])
        out.append(dets[keep])
        idx.append(inds[keep].astype(np.int64))
    mpi = o["max_per_image"]
    if mpi > 0:
        allsc = np.hstack([d[:, 4] for d in out[1:]]) if C > 1 else np.zeros(0, F)
        if allsc.shape[0] > mpi:
            th = np.sort(allsc)[-mpi]
            sel = [d[:, 4] >= th for d in out[1:]]
            out = [out[0]] + [d[s] for d, s in zip(out[1:], sel)]
            idx = [idx[0]] + [i[s] for i, s in zip(idx[1:], sel)]
    return out, idx


def score_boxes(net, w, blob, boxes, scale, orig_hw, o=None):
    """Caller boxes [n,4] in original-image pixels -> dict(rois, fc7, cls_score, cls_prob, bbox_pred, scores, pred_boxes)."""
    o = o or P.opts()
    boxes = np.asarray(boxes, dtype=F).reshape(-1, 4)
    st = {"rois": np.hstack([np.zeros((boxes.shape[0], 1), F), (boxes * F(scale)).astype(F)]).astype(F)}
    feat = N.image_to_head(net, w, blob)
    st["fc7"] = N.head_to_tail(net, w, P.crop_pool(net, feat, st["rois"], o))
    num_classes = w[N.scope_of(net) + "/cls_score/weights"].shape[1]
    st["cls_score"], st["cls_prob"], st["bbox_pred"] = P.region_classification(net, w, st["fc7"], num_classes, o)
    st["scores"], st["pred_boxes"] = P.im_detect_post(st["rois"], st["cls_prob"], st["bbox_pred"], scale, orig_hw[0], orig_hw[1])
    return st
