"""Inference driver with the reference's entry points (lib/model/test.py): _get_image_blob :26-58,
im_detect :86-107, apply_nms :109-136, test_net :138-192.

im_detect keeps the reference data flow (host blob -> net.test_image -> decode -> clip) but the decode/clip
run in a device kernel right behind the CUDA graph (frcnn_bbox_decode) instead of NumPy.  test_net by default
also keeps the per-class NMS + max_per_image cap on the device (frcnn_detect_post); setting
`FUSED_POST = False` runs the reference's Python loop over `nms()` instead (same results).

Under torchrun (torch.distributed initialised, world size W > 1) test_net shards the imdb -- image i on rank i mod W --
and all-gathers each step's fixed-size detection records straight from the buffers the last kernel wrote
(tf_faster_rcnn_b200/parallel.py); rank 0 assembles all_boxes, writes detections.pkl and evaluates."""
import os
import pickle

import cv2
import numpy as np
import torch

from model.config import cfg, get_output_dir
from model.nms_wrapper import box_voting, nms, soft_nms
from tf_faster_rcnn_b200 import engine
from utils.blob import im_list_to_blob
from utils.timer import Timer

FUSED_POST = True
# Images per device launch in test_net's single-process loop (consecutive images with equal blob shapes are grouped).  1 = the
# reference's data flow; tools/test_net.py --batch N raises it (throughput mode, SURVEY 8(f) rank 4).
BATCH_SIZE = 1
# Opt-in (SURVEY 8(f) rank 2): build the blob on the device from the uint8 image (mean subtraction + the cv2.resize
# INTER_LINEAR arithmetic restated in a kernel, <= 1e-4 from OpenCV) instead of on the host.  Off by default so that the
# default data flow is the reference's (host OpenCV blob).
DEVICE_PREPROCESS = False


def _get_image_blob(im):
    """BGR uint8 image -> ([1,H,W,3] fp32 blob, scale factors): mean-subtract, resize so the short side is
    TEST.SCALES[i] unless that would push the long side over TEST.MAX_SIZE."""
    pixels = im.astype(np.float32, copy=True)
    pixels -= cfg.PIXEL_MEANS
    resized, factors = [], []
    for target in cfg.TEST.SCALES:
        r, f = _resize(pixels, target, cfg.TEST.MAX_SIZE)
        resized.append(r)
        factors.append(f)
    return im_list_to_blob(resized), np.array(factors)


def _scale_factor(im_shape, target, max_size):
    """short side -> target unless the long side would exceed max_size"""
    short_side, long_side = min(im_shape[:2]), max(im_shape[:2])
    f = float(target) / float(short_side)
    if np.round(f * long_side) > max_size:
        f = float(max_size) / float(long_side)
    return f


def _resize(pixels, target, max_size):
    f = _scale_factor(pixels.shape, target, max_size)
    return cv2.resize(pixels, None, None, fx=f, fy=f, interpolation=cv2.INTER_LINEAR), f


def blob_geometry(im_shape, target=None, max_size=None):
    """(H, W, scale) of the blob _get_image_blob would build for an image of this shape (first TEST scale, or `target` short
    side capped by `max_size`)."""
    f = _scale_factor(im_shape, cfg.TEST.SCALES[0] if target is None else target, cfg.TEST.MAX_SIZE if max_size is None else max_size)
    # cv2.resize with fx/fy: dsize = cvRound(size * f) (round half to even)
    return int(np.rint(im_shape[0] * f)), int(np.rint(im_shape[1] * f)), f


# ---- test-time augmentation (TEST.BBOX_AUG; Detectron's im_detect_bbox_aug in union mode) ---------------------------------------
# A view is (scale, flip): the base view (TEST.SCALES[0], TEST.MAX_SIZE), one view per BBOX_AUG.SCALES entry (that short side,
# the long side capped by BBOX_AUG.MAX_SIZE) and, with H_FLIP, the mirrored twin of each.  A mirrored view is resize(im[:, ::-1]):
# mirrored first, then resized, so un-flipping its boxes (x1 = (W - x2') - 1, x2 = (W - x1') - 1 in fp32, W the original width)
# is exact in original pixels.  The union of an image takes the valid RoI rows of each view in Detectron's order: the flipped
# base view, then every extra scale followed by its flip, the base view last.  The order decides only ties and Soft-NMS's
# candidate order.  The per-class NMS (greedy or Soft-NMS), the max_per_image cap and the records then run unchanged on the union.

def aug_views(im_shape):
    """The views of an image of this shape in union order: [(target, max_size, flip), ...]."""
    flip, scales, max_size = engine.bbox_aug_option(cfg.TEST.BBOX_AUG, cfg.TEST.BBOX_REG)
    base = (cfg.TEST.SCALES[0], cfg.TEST.MAX_SIZE)
    views = [base + (True,)] if flip else []
    for s in scales:
        views.append((s, max_size, False))
        if flip:
            views.append((s, max_size, True))
    return views + [base + (False,)]


def aug_view_blob(im, target, max_size, flip):
    """One view's host blob ([1,H,W,3] fp32, scale factor): _get_image_blob's arithmetic on im, or on im[:, ::-1] when flipped."""
    pixels = (im[:, ::-1] if flip else im).astype(np.float32, copy=True)
    pixels -= cfg.PIXEL_MEANS
    r, f = _resize(pixels, target, max_size)
    return im_list_to_blob([r]), f


def _run_aug(net, ims, detect, double_buffer=False, device_preprocess=False):
    """ims: images whose views have the same blob shapes -> the AugPlan after one launch (records when `detect`, else the union
    left in its cls_prob / pred_boxes / num_rois).  Every check raises before device work."""
    views = aug_views(ims[0].shape)
    hws = [im.shape[:2] for im in ims]
    if device_preprocess:
        geo = [blob_geometry(ims[0].shape, t, m) for t, m, _ in views]
        aug = net.aug_plan([(g[0], g[1], fl) for g, (_, _, fl) in zip(geo, views)], len(ims))
        means = np.asarray(cfg.PIXEL_MEANS, dtype=np.float64).ravel()
        from tf_faster_rcnn_b200 import ops
        for b, im in enumerate(ims):
            img = torch.from_numpy(np.ascontiguousarray(im)).cuda(non_blocking=True)
            for v, (_, _, fl) in enumerate(views):
                ops.preprocess(img, means, geo[v][2], geo[v][2], aug.view_image(v)[b:b + 1], hflip=fl)
        scales = [[g[2]] * len(ims) for g in geo]
    else:
        per_view = [[aug_view_blob(im, *view) for im in ims] for view in views]
        aug = net.aug_plan([(pv[0][0].shape[1], pv[0][0].shape[2], fl) for pv, (_, _, fl) in zip(per_view, views)], len(ims))
        for v, pv in enumerate(per_view):
            aug.view_image(v).copy_(torch.from_numpy(np.concatenate([x[0] for x in pv], axis=0)), non_blocking=True)
        scales = [[x[1] for x in pv] for pv in per_view]
    aug.double_buffer = double_buffer
    aug.launch(scales, hws, detect=detect)
    return aug


def _aug_key(im):
    """The tuple of view blob shapes of an image: images with equal keys share one augmented launch."""
    return tuple(blob_geometry(im.shape, t, m)[:2] + (fl,) for t, m, fl in aug_views(im.shape))


def _run_device_preprocess(net, im, post, detect, boxes=None):
    """uint8 image -> H2D (0.5 MB instead of the 5.8 MB fp32 blob) -> preprocess kernel -> graph.  boxes: caller RoIs
    (fp32 [n,4], original-image pixels) instead of the RPN's."""
    from tf_faster_rcnn_b200 import ops, engine
    H, W, f = blob_geometry(im.shape)
    if boxes is not None:
        engine.check_pool_boxes(net.options["pooling_mode"], [boxes], [f], (H, W))
    plan = net.plan_for(H, W) if boxes is None else net.plan_for(H, W, cap=engine.box_capacity(boxes.shape[0]))
    img = torch.from_numpy(np.ascontiguousarray(im)).cuda(non_blocking=True)
    ops.preprocess(img, np.asarray(cfg.PIXEL_MEANS, dtype=np.float64).ravel(), f, f, plan.image)
    if boxes is not None:
        plan.set_boxes([boxes])
    plan.launch(f, im.shape[0], im.shape[1], post=post, detect=detect)
    return plan, f


def _get_blobs(im):
    data, factors = _get_image_blob(im)
    return {'data': data}, factors


def im_detect(sess, net, im, boxes=None):
    """-> scores [R, C] fp32, pred_boxes [R, 4C] fp32 in ORIGINAL-image pixels.  boxes: [n, 4] boxes (x1,y1,x2,y2,
    original-image pixels) scored instead of the RPN's proposals (Fast R-CNN, TEST.HAS_RPN = False): then R = n, in the
    given order.  With TEST.BBOX_AUG.ENABLED: the union of the views (R = its row count, see aug_views)."""
    if cfg.TEST.BBOX_AUG.ENABLED:
        if boxes is not None:
            raise ValueError("TEST.BBOX_AUG (test-time augmentation) does not apply to caller boxes: disable it for this call")
        aug = _run_aug(net, [im], detect=False, device_preprocess=DEVICE_PREPROCESS)
        torch.cuda.current_stream().synchronize()
        r = int(aug.num_rois[0].item())
        return aug.cls_prob[:r].cpu().numpy(), aug.pred_boxes[:r].cpu().numpy()
    if boxes is not None:
        from tf_faster_rcnn_b200 import engine
        boxes = engine.check_boxes([np.asarray(boxes, dtype=np.float32)], 1)[0]
    if DEVICE_PREPROCESS:
        plan, f = _run_device_preprocess(net, im, post=True, detect=False, boxes=boxes)
        im_scales = np.array([f])
    else:
        blobs, im_scales = _get_blobs(im)
        assert len(im_scales) == 1, "Only single-image batch implemented"
        blob = blobs['data']
        blobs['im_info'] = np.array([blob.shape[1], blob.shape[2], im_scales[0]], dtype=np.float32)
        if boxes is None:
            plan = net._run(blob, blobs['im_info'], post=True, detect=False, orig_hw=im.shape[:2])
        else:
            plan = net._run_boxes(blob, [im_scales[0]], [im.shape[:2]], [boxes])
    torch.cuda.current_stream().synchronize()
    r = int(plan.num_rois[0].item())
    scores = plan.cls_prob[:r].cpu().numpy()
    if cfg.TEST.BBOX_REG:
        pred_boxes = plan.pred_boxes[:r].cpu().numpy()
    else:
        boxes = plan.rois[:r, 1:5].cpu().numpy() / np.float32(im_scales[0])
        pred_boxes = np.tile(boxes, (1, scores.shape[1]))
    return scores, pred_boxes


def apply_nms(all_boxes, thresh):
    """NMS over already-collected detections all_boxes[cls][image] (used by tools/reval.py)."""
    out = [[[] for _ in range(len(all_boxes[0]))] for _ in range(len(all_boxes))]
    for c, per_image in enumerate(all_boxes):
        for i, dets in enumerate(per_image):
            if len(dets) == 0:
                continue
            ok = np.where((dets[:, 2] > dets[:, 0]) & (dets[:, 3] > dets[:, 1]))[0]
            dets = dets[ok, :]
            if len(dets) == 0:
                continue
            keep = nms(dets, thresh)
            if len(keep):
                out[c][i] = dets[keep, :].copy()
    return out


def _detections_python_loop(scores, boxes, num_classes, thresh, max_per_image):
    """test.py:162-180 verbatim flow over the (GPU) nms(), or soft_nms() per class when TEST.SOFT_NMS.ENABLED; with
    TEST.BBOX_VOTE.ENABLED each class's kept rows are then voted against its candidates (box_voting) and, for a score-changing
    method, re-sorted stably by descending voted score, as the fused post does."""
    per_class = [np.zeros((0, 5), np.float32)]
    bv = cfg.TEST.BBOX_VOTE
    for j in range(1, num_classes):
        inds = np.where(scores[:, j] > thresh)[0]
        cls_dets = np.hstack((boxes[inds, j * 4:(j + 1) * 4], scores[inds, j][:, np.newaxis])).astype(np.float32, copy=False)
        if cfg.TEST.SOFT_NMS.ENABLED:
            sn = cfg.TEST.SOFT_NMS
            kept, _ = soft_nms(cls_dets, sn.SIGMA, cfg.TEST.NMS, sn.SCORE_THRESH, sn.METHOD)
        else:
            kept = cls_dets[nms(cls_dets, cfg.TEST.NMS), :]
        if bv.ENABLED:
            kept = box_voting(kept, cls_dets, bv.VOTE_TH, bv.SCORING_METHOD, bv.SCORING_METHOD_BETA)
            if bv.SCORING_METHOD != "ID":
                kept = kept[np.argsort(-kept[:, 4], kind="stable")]
        per_class.append(kept)
    if max_per_image > 0:
        image_scores = np.hstack([d[:, -1] for d in per_class[1:]])
        if len(image_scores) > max_per_image:
            image_thresh = np.sort(image_scores)[-max_per_image]
            per_class = [per_class[0]] + [d[d[:, -1] >= image_thresh, :] for d in per_class[1:]]
    return per_class


def detect_image(net, im, thresh=0., max_per_image=100):
    """One image through the fused device path -> list over classes of fp32 [k,5] (x1,y1,x2,y2,score)."""
    _set_post_options(net, thresh, max_per_image)
    if cfg.TEST.BBOX_AUG.ENABLED:
        det = _run_aug(net, [im], detect=True).records()[0]
    else:
        blobs, im_scales = _get_blobs(im)
        blob = blobs['data']
        im_info = np.array([blob.shape[1], blob.shape[2], im_scales[0]], dtype=np.float32)
        det, _ = net.detect(blob, im_info, im.shape[:2])
    C = net.num_classes
    cls = det[:, 5].astype(np.int64)
    return [det[cls == j, :5] for j in range(C)]


def _set_post_options(net, thresh, max_per_image):
    net.options["score_thresh"], net.options["max_per_image"] = float(thresh), int(max_per_image)
    net.options["nms_thresh"] = cfg.TEST.NMS
    net.options["soft_nms"] = engine.soft_nms_option(cfg.TEST.SOFT_NMS)
    net.options["box_vote"] = engine.box_vote_option(cfg.TEST.BBOX_VOTE)


def _detect_record(net, im, thresh, max_per_image):
    """Fused path for one image, result left on the device: the plan's record buffer of this launch
    ([REC_HEADER + max_det*6] fp32, int32 count in word 0), stream-ordered.  Consecutive launches of a plan alternate between
    two record buffers, so the record stays valid while the NEXT image runs (the sharded loop gathers it meanwhile); so do the
    augmented launches of TEST.BBOX_AUG."""
    if cfg.TEST.BBOX_AUG.ENABLED:
        _set_post_options(net, thresh, max_per_image)
        return _run_aug(net, [im], detect=True, double_buffer=True).rec[0]
    blobs, im_scales = _get_blobs(im)
    blob = blobs['data']
    im_info = np.array([blob.shape[1], blob.shape[2], im_scales[0]], dtype=np.float32)
    _set_post_options(net, thresh, max_per_image)
    plan = net.plan_for(blob.shape[1], blob.shape[2])
    plan.double_buffer = True
    plan = net._run(blob, im_info, post=True, detect=True, orig_hw=im.shape[:2])
    return plan.rec[0]


def detect_images(net, ims, thresh=0., max_per_image=100, batch_size=None):
    """Several images through the fused device path, grouping CONSECUTIVE images whose blobs have the same shape into batches
    of up to `batch_size` (default BATCH_SIZE).  -> per image a list over classes of fp32 [k,5].  Batch 1 is the reference's
    data flow; larger batches are the throughput extension (same per-image arithmetic, M = batch * pixels per layer)."""
    bs = int(batch_size or BATCH_SIZE)
    _set_post_options(net, thresh, max_per_image)
    C = net.num_classes
    if cfg.TEST.BBOX_AUG.ENABLED:      # groups: consecutive images whose whole tuple of view blob shapes matches
        out, i = [], 0
        keys = [_aug_key(im) for im in ims]
        while i < len(ims):
            j = i + 1
            while j < len(ims) and j - i < bs and keys[j] == keys[i]:
                j += 1
            for det in _run_aug(net, ims[i:j], detect=True).records():
                cls = det[:, 5].astype(np.int64)
                out.append([det[cls == c, :5] for c in range(C)])
            i = j
        return out
    prepared = []
    for im in ims:
        blobs, im_scales = _get_blobs(im)
        prepared.append((blobs['data'], float(im_scales[0]), im.shape[:2]))
    out = [None] * len(ims)
    i = 0
    while i < len(prepared):
        j = i + 1
        while j < len(prepared) and j - i < bs and prepared[j][0].shape == prepared[i][0].shape:
            j += 1
        group = prepared[i:j]
        if len(group) == 1:
            b0, s0, hw0 = group[0]
            dets = [net.detect(b0, np.array([b0.shape[1], b0.shape[2], s0], np.float32), hw0)[0]]
        else:
            dets, _ = net.detect_batch(np.concatenate([g[0] for g in group], axis=0), [g[1] for g in group], [g[2] for g in group])
        for k, det in enumerate(dets):
            cls = det[:, 5].astype(np.int64)
            out[i + k] = [det[cls == c, :5] for c in range(C)]
        i = j
    return out


def _test_net_sharded(imdb, detect_record, verbose=True):
    """Lock-step loop over ceil(N / W) steps; every rank returns the complete all_boxes[cls][image].
    detect_record(image index) -> record tensor [REC_HEADER + max_det*6] fp32 (int32 count in word 0) on the collective's
    device, valid until two more records have been produced.  ONE all-gather per step, issued asynchronously: while it is in
    flight the rank already runs its next image, and the previous step's gathered records are scattered on the host."""
    import torch.distributed as dist
    from tf_faster_rcnn_b200 import parallel
    rank, world = dist.get_rank(), dist.get_world_size()
    num_images = len(imdb.image_index)
    all_boxes = [[[] for _ in range(num_images)] for _ in range(imdb.num_classes)]
    mine = parallel.shard_indices(num_images, rank, world)
    device = torch.device("cuda", torch.cuda.current_device()) if dist.get_backend() == "nccl" else torch.device("cpu")
    gather = idle = None
    timer = Timer()
    nsteps = parallel.steps_for(num_images, world)
    for step in range(nsteps):
        timer.tic()
        slot = step & 1
        if gather is not None:
            gather.before_overwrite(slot)              # the gather of step-2 has read the record buffer about to be reused
        rec = detect_record(mine[step]) if step < len(mine) else None
        if gather is None:
            # ranks without an image (N < W) learn the record size from the others: one extra tiny collective, once
            cap = torch.tensor([rec.numel() if rec is not None else 0], dtype=torch.int64, device=device)
            dist.all_reduce(cap, op=dist.ReduceOp.MAX)
            if device.type == "cuda":
                from tf_faster_rcnn_b200 import ops
                idle = ops.zeros(int(cap.item()))
            else:
                idle = torch.zeros(int(cap.item()), dtype=torch.float32)
            gather = parallel.RecordGather(idle, world)
        gather.issue(slot, rec if rec is not None else idle)
        if step > 0:
            parallel.records_to_all_boxes(all_boxes, step - 1, world, gather.result(slot ^ 1), num_images)
        timer.toc()
        if verbose and rank == 0:
            print('im_detect: {:d}/{:d} {:.3f}s per step of {:d} images'.format(
                min((step + 1) * world, num_images), num_images, timer.average_time, world))
    if nsteps > 0:
        parallel.records_to_all_boxes(all_boxes, nsteps - 1, world, gather.result((nsteps - 1) & 1), num_images)
    return all_boxes


def test_net(sess, net, imdb, weights_filename, max_per_image=100, thresh=0.):
    """Run the detector over imdb; all_boxes[cls][image] = [k,5]; pickles detections.pkl and evaluates."""
    np.random.seed(cfg.RNG_SEED)
    num_images = len(imdb.image_index)
    output_dir = get_output_dir(imdb, weights_filename)
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        assert FUSED_POST and cfg.TEST.BBOX_REG, "sharded test_net gathers the fused path's device records"
        all_boxes = _test_net_sharded(
            imdb, lambda i: _detect_record(net, cv2.imread(imdb.image_path_at(i)), thresh, max_per_image))
        if dist.get_rank() == 0:
            with open(os.path.join(output_dir, 'detections.pkl'), 'wb') as f:
                pickle.dump(all_boxes, f, pickle.HIGHEST_PROTOCOL)
            print('Evaluating detections')
            imdb.evaluate_detections(all_boxes, output_dir)
        dist.barrier()
        return all_boxes
    all_boxes = [[[] for _ in range(num_images)] for _ in range(imdb.num_classes)]
    _t = {'im_detect': Timer(), 'misc': Timer()}
    if FUSED_POST and cfg.TEST.BBOX_REG and BATCH_SIZE > 1:
        for i0 in range(0, num_images, BATCH_SIZE):
            ims = [cv2.imread(imdb.image_path_at(i)) for i in range(i0, min(i0 + BATCH_SIZE, num_images))]
            _t['im_detect'].tic()
            results = detect_images(net, ims, thresh, max_per_image)
            _t['im_detect'].toc()
            for k, per_class in enumerate(results):
                for j in range(1, imdb.num_classes):
                    all_boxes[j][i0 + k] = per_class[j]
            print('im_detect: {:d}/{:d} {:.3f}s per batch of {:d}'.format(min(i0 + BATCH_SIZE, num_images), num_images,
                                                                          _t['im_detect'].average_time, BATCH_SIZE))
    else:
        for i in range(num_images):
            im = cv2.imread(imdb.image_path_at(i))
            if FUSED_POST and cfg.TEST.BBOX_REG:
                _t['im_detect'].tic()
                per_class = detect_image(net, im, thresh, max_per_image)
                _t['im_detect'].toc()
                _t['misc'].tic()
            else:
                _t['im_detect'].tic()
                scores, boxes = im_detect(sess, net, im)
                _t['im_detect'].toc()
                _t['misc'].tic()
                per_class = _detections_python_loop(scores, boxes, imdb.num_classes, thresh, max_per_image)
            for j in range(1, imdb.num_classes):
                all_boxes[j][i] = per_class[j]
            _t['misc'].toc()
            print('im_detect: {:d}/{:d} {:.3f}s {:.3f}s'.format(i + 1, num_images, _t['im_detect'].average_time, _t['misc'].average_time))
    with open(os.path.join(output_dir, 'detections.pkl'), 'wb') as f:
        pickle.dump(all_boxes, f, pickle.HIGHEST_PROTOCOL)
    print('Evaluating detections')
    imdb.evaluate_detections(all_boxes, output_dir)
    return all_boxes
