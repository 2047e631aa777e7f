"""Test-time augmentation oracle (test infrastructure, composed from oracle.pipeline): Detectron's im_detect_bbox_aug in union
mode, restated for this project's views.

  views          the view list (target short side, max size, flip) in union order: flipped base, then each extra scale followed
                 by its flip, the base view last
  unflip         a mirrored view's boxes back to original pixels in fp32: x1 = (W - x2') - 1, x2 = (W - x1') - 1
  union          vstack of the views' (scores, boxes), mirrored views un-flipped
  union_model    numpy model of frcnn_aug_union's layout: [B, R_union] rows, valid rows of each view in order, zero tail
  im_detect_aug  the oracle alone: get_image_blob on im or im[:, ::-1] at each view's scale, test_image, im_detect_post, union
  post           test_net_post, or the Soft-NMS oracle, on a union
"""
import os
import sys

import numpy as np

from oracle import pipeline as P

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import soft_nms_oracle as SO  # noqa: E402

F = np.float32


def views(h_flip, scales, max_size, base=(600, 1000)):
    out = [tuple(base) + (True,)] if h_flip else []
    for s in scales:
        out.append((s, max_size, False))
        if h_flip:
            out.append((s, max_size, True))
    return out + [tuple(base) + (False,)]


def unflip(boxes, orig_w):
    """boxes [n, 4C] fp32 of a mirrored view -> original pixels; every operation one fp32 rounding."""
    b = np.array(boxes, dtype=F).reshape(boxes.shape[0], boxes.shape[1] // 4, 4)
    w = F(orig_w)
    x1 = (w - b[..., 2]) - F(1.0)
    x2 = (w - b[..., 0]) - F(1.0)
    b[..., 0], b[..., 2] = x1, x2
    return b.reshape(boxes.shape)


def union(scores, boxes, flips, orig_w):
    """per view scores [n_v, C], boxes [n_v, 4C] (valid rows only) -> the union in view order."""
    bx = [unflip(b, orig_w) if f else np.asarray(b, F) for b, f in zip(boxes, flips)]
    return np.vstack(scores).astype(F), np.vstack(bx).astype(F)


def union_model(probs, boxes, counts, flips, orig_w):
    """frcnn_aug_union's outputs.  probs[v] [B, R_v, C], boxes[v] [B, R_v, 4C], counts[v] [B] (clamped to [0, R_v]),
    orig_w [B] -> (cls_prob [B, R_union, C], pred_boxes [B, R_union, 4C], num_rois int32 [B])."""
    B, C = probs[0].shape[0], probs[0].shape[2]
    ru = sum(p.shape[1] for p in probs)
    up, ub, num = np.zeros((B, ru, C), F), np.zeros((B, ru, 4 * C), F), np.zeros(B, np.int32)
    for b in range(B):
        n = [int(min(max(c[b], 0), p.shape[1])) for c, p in zip(counts, probs)]
        s, x = union([p[b, :k] for p, k in zip(probs, n)], [q[b, :k] for q, k in zip(boxes, n)], flips, orig_w[b])
        up[b, :s.shape[0]], ub[b, :s.shape[0]], num[b] = s, x, s.shape[0]
    return up, ub, num


def im_detect_aug(net, w, im, num_classes, o, view_list):
    """The oracle alone on one uint8 BGR image: -> (scores [R_union, C], boxes [R_union, 4C]) in original pixels."""
    sc, bx = [], []
    for target, max_size, flip in view_list:
        src = np.ascontiguousarray(im[:, ::-1]) if flip else im
        blob, s = P.get_image_blob(src, dict(o, test_scale=target, test_max_size=max_size))
        st = P.test_image(net, w, blob, np.array([blob.shape[1], blob.shape[2], s], F), num_classes, o)
        scores, boxes = P.im_detect_post(st["rois"], st["cls_prob"], st["bbox_pred"], s, im.shape[0], im.shape[1])
        sc.append(scores)
        bx.append(boxes)
    return union(sc, bx, [v[2] for v in view_list], im.shape[1])


def post(scores, boxes, o, soft=None, thresh=0.0):
    """test.py:162-180 on a union: greedy (o's predicate) or Soft-NMS (soft = (method, sigma, prune)) -> list over classes."""
    if soft is None:
        return P.test_net_post(scores, boxes, o, thresh)
    return SO.test_net_post_soft(scores, boxes, soft, o["nms_thresh"], o["max_per_image"], thresh)[0]
