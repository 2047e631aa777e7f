"""`Network` base class with the reference's call surface (lib/nets/network.py):
create_architecture :386-454, test_image :470-479, extract_head :464-467; subclasses implement
_image_to_head / _head_to_tail (:380-384).  Instead of building a TF graph, create_architecture records
the options; the first test_image for a blob shape builds a ShapePlan (device buffers, TMA-backed conv
plans, CUDA graph) and later calls replay it.  `sess` arguments are accepted and ignored.
"""
import os

import numpy as np
import torch

from model.config import cfg
from layer_utils.generate_anchors import generate_anchors
from tf_faster_rcnn_b200 import engine, _native

_REGISTRY = []   # networks created in this process (the tensorflow shim's Saver.restore walks it)


def _no_bbox_aug(what):
    if cfg.TEST.BBOX_AUG.ENABLED:
        raise ValueError("TEST.BBOX_AUG (test-time augmentation) does not apply to %s: disable it for this call" % what)


class Network(object):
    def __init__(self):
        self._feat_stride = [16, ]
        self._predictions = {}
        self._layers = {}
        self._scope = None
        self.weights = None
        self._plans = {}
        self._aug_plans = {}   # test-time augmentation: (views, batch) -> engine.AugPlan over plans of _plans
        self.use_cuda_graph = True
        _REGISTRY.append(self)

    # ---- reference surface ---------------------------------------------------------------------------
    def create_architecture(self, mode, num_classes, tag=None, anchor_scales=(8, 16, 32), anchor_ratios=(0.5, 1, 2)):
        assert tag is not None
        if mode != "TEST":
            raise NotImplementedError("only the TEST-mode (inference) graph exists in this build")
        num_classes = engine.check_num_classes(num_classes)
        self._mode, self._tag = mode, tag
        self._num_classes = num_classes
        self._anchor_scales, self._anchor_ratios = tuple(anchor_scales), tuple(anchor_ratios)
        self._num_scales, self._num_ratios = len(anchor_scales), len(anchor_ratios)
        self._num_anchors = self._num_scales * self._num_ratios
        self.base_anchors = generate_anchors(ratios=np.array(self._anchor_ratios), scales=np.array(self._anchor_scales)).astype(np.float32)
        self.anchor_key = "%s|%s" % (self._anchor_scales, self._anchor_ratios)
        # POOLING_MODE 'crop' (the reference's), 'align' (RoIAlign, with cfg.ROI_ALIGN) or 'pool' (RoIPool); read at plan build
        roi_align = engine.roi_align_option(cfg.POOLING_MODE, cfg.POOLING_SIZE, cfg.ROI_ALIGN)
        engine.check_rpn_channels(cfg.RPN_CHANNELS)
        attributes = engine.attributes_option(cfg.ATTRIBUTES)
        self.options = dict(
            pooling_mode=cfg.POOLING_MODE, roi_align=roi_align,
            test_mode=cfg.TEST.MODE, use_e2e_tf=bool(cfg.USE_E2E_TF), use_gpu_nms=bool(cfg.USE_GPU_NMS),
            rpn_nms_thresh=cfg.TEST.RPN_NMS_THRESH, rpn_pre_nms_top_n=cfg.TEST.RPN_PRE_NMS_TOP_N,
            rpn_post_nms_top_n=cfg.TEST.RPN_POST_NMS_TOP_N, rpn_top_n=cfg.TEST.RPN_TOP_N,
            pooling_size=cfg.POOLING_SIZE, resnet_max_pool=bool(cfg.RESNET.MAX_POOL),
            bbox_stds=tuple(cfg.TRAIN.BBOX_NORMALIZE_STDS), bbox_means=tuple(cfg.TRAIN.BBOX_NORMALIZE_MEANS),
            nms_thresh=cfg.TEST.NMS, max_per_image=100, score_thresh=0.0, rpn_channels=cfg.RPN_CHANNELS,
            soft_nms=engine.soft_nms_option(cfg.TEST.SOFT_NMS), box_vote=engine.box_vote_option(cfg.TEST.BBOX_VOTE),
            attributes=attributes,
        )
        if self.options["test_mode"] not in ("nms", "top"):
            raise NotImplementedError
        self._plans = {}
        self._aug_plans = {}
        return {"rois": None}

    def test_image(self, sess, image, im_info):
        """-> (cls_score, cls_prob, bbox_pred, rois) host fp32 arrays, rois in blob-scale pixels."""
        plan = self._run(image, im_info)
        torch.cuda.current_stream().synchronize()
        r = int(plan.num_rois[0].item())
        out = (plan.cls_score[:r].cpu().numpy(), plan.cls_prob[:r].cpu().numpy(), plan.bbox_pred[:r].cpu().numpy(),
               plan.rois[:r].cpu().numpy())
        return out

    def extract_head(self, sess, image):
        plan = self._run(image, np.array([image.shape[1], image.shape[2], 1.0], np.float32))
        torch.cuda.current_stream().synchronize()
        return plan.feat.cpu().numpy()

    def _image_to_head(self, tape, image):
        raise NotImplementedError

    def _head_to_tail(self, tape, pool5):
        raise NotImplementedError

    # ---- device side -------------------------------------------------------------------------------------
    @property
    def num_anchors(self):
        return self._num_anchors

    @property
    def num_classes(self):
        return self._num_classes

    @property
    def scope(self):
        return self._scope

    def crop_pre_pool(self):
        """14x14 crop + 2x2 max pool (network.py:154-157) unless a subclass crops 7x7 directly."""
        return True

    def arch_name(self):
        """'vgg16' | 'res50' | 'res101' | 'res152' | 'mobile' (the --net names of tools/test_net.py:92-103)."""
        return {"vgg_16": "vgg16", "MobilenetV1": "mobile"}.get(self._scope) or "res%d" % self._num_layers

    def check_variables(self, tensors):
        """What tf.train.Saver.restore would reject: TEST-graph variables missing from `tensors` or of another shape
        (class count, anchor set, backbone).  Needs create_architecture() first.  -> list of messages."""
        from tf_faster_rcnn_b200 import synth
        return synth.check(self.arch_name(), tensors, self._num_classes, self._num_anchors,
                           rpn_channels=int(cfg.RPN_CHANNELS), pooling_size=int(cfg.POOLING_SIZE),
                           depth_multiplier=float(getattr(self, "_depth_multiplier", 1.0)), attributes=self.options["attributes"])

    def load_weights(self, tensors, strict=False):
        """tensors: dict TF-variable-name -> numpy array (HWIO convs, [in,out] FCs, BatchNorm stats).
        strict: verify names and shapes against the architecture first (checkpoint restores) and raise ValueError."""
        if strict:
            problems = self.check_variables(tensors)
            if problems:
                raise ValueError("checkpoint does not match the %s TEST graph (%d classes, %d anchors):\n  %s"
                                 % (self.arch_name(), self._num_classes, self._num_anchors, "\n  ".join(problems)))
        self.weights = engine.Weights(dict(tensors))
        self._plans = {}
        self._aug_plans = {}

    MAX_PLANS = int(os.environ.get("FRCNN_MAX_PLANS", "6"))

    def plan_for(self, h, w, batch=1, cap=None):
        """ShapePlan of blob shape (h, w) x batch.  A plan owns every layer's activation buffer, the TMA descriptors and the CUDA
        graphs of that shape (0.6-1.3 GB per image at 600x800..1000), so the cache is a small LRU: a dataset with hundreds of
        distinct shapes recycles plans instead of growing without bound (evicted buffers return to the caching allocator).
        cap: a caller-box plan (RoIs = up to `cap` given boxes per image, no RPN), cached beside the RPN plans."""
        if self.weights is None:
            raise RuntimeError("no weights loaded: call load_weights() / Saver.restore() before test_image")
        key = (int(h), int(w), int(batch)) if cap is None else (int(h), int(w), int(batch), "boxes", int(cap))
        plan = self._plans.pop(key, None)
        if plan is None:
            dev = torch.cuda.current_device() if torch.cuda.is_available() else 0
            _native.check(_native.lib().frcnn_check_device(dev), "check_device")   # fails loudly: no CPU fallback exists
            while len(self._plans) >= max(1, self.MAX_PLANS):
                old_key = next(iter(self._plans))
                old = self._plans.pop(old_key)
                torch.cuda.current_stream().synchronize()   # nothing of the evicted plan is still in flight
                old.release()
            plan = engine.ShapePlan(self, key[0], key[1], key[2], use_graph=self.use_cuda_graph,
                                    rois_source="rpn" if cap is None else "boxes", cap=cap)
        self._plans[key] = plan                             # most recently used last
        return plan

    def aug_plan(self, views, batch):
        """AugPlan of test-time augmentation for `batch` images with views ((h, w, flip), ...) in union order; its sub-plans come
        from plan_for.  Raises ValueError (too many views, union rows or blob shapes) before any device work."""
        views = tuple((int(h), int(w), bool(f)) for h, w, f in views)
        engine.check_aug_views(views, engine.aug_rois_per_view(self.options), max(1, self.MAX_PLANS))
        key = (views, int(batch))
        aug = self._aug_plans.pop(key, None)
        if aug is None:
            while len(self._aug_plans) >= max(1, self.MAX_PLANS):
                self._aug_plans.pop(next(iter(self._aug_plans)))
            aug = engine.AugPlan(self, views, int(batch))
        else:
            aug.bind()
        self._aug_plans[key] = aug                          # most recently used last
        return aug

    def detect_aug(self, blobs, im_scales, orig_hws, flips):
        """Test-time augmentation (TEST.BBOX_AUG) through the fused device path: per view v a blob blobs[v] [B, H_v, W_v, 3]
        (numpy or torch; a mirrored view is the blob of the mirrored image), im_scales[v] its B scale factors and flips[v];
        orig_hws: per image the original (h, w).  The views' detections are merged in the given order ahead of the per-class
        NMS and the max_per_image cap.  -> (list of B det arrays [n,6], aug plan)."""
        b = int(blobs[0].shape[0])
        assert len(blobs) == len(im_scales) == len(flips) and len(orig_hws) == b
        aug = self.aug_plan([(x.shape[1], x.shape[2], f) for x, f in zip(blobs, flips)], b)
        for v, x in enumerate(blobs):
            assert x.shape[0] == b and x.shape[3] == 3
            src = x if isinstance(x, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32))
            aug.view_image(v).copy_(src, non_blocking=True)
        aug.launch(im_scales, orig_hws, detect=True)
        return aug.records(), aug

    def _batch_plan(self, images, im_scales, orig_hws, cap=None):
        """A batch call's arguments checked (images [B, H, W, 3], B scale factors, B original (h, w)) -> (plan_for that shape,
        batch and cap; the B per-image (scale, orig_h, orig_w) meta rows)."""
        assert images.shape[3] == 3 and len(im_scales) == len(orig_hws) == images.shape[0]
        meta = [(float(s), int(hw[0]), int(hw[1])) for s, hw in zip(im_scales, orig_hws)]
        return self.plan_for(images.shape[1], images.shape[2], len(meta), cap=cap), meta

    def _copy_in(self, plan, image):
        if isinstance(image, torch.Tensor):
            plan.image.copy_(image, non_blocking=True)
        else:
            plan.image.copy_(torch.from_numpy(np.ascontiguousarray(image, dtype=np.float32)), non_blocking=True)

    def _run(self, image, im_info, post=False, detect=False, orig_hw=None):
        assert image.shape[0] == 1 and image.shape[3] == 3, "test_image / im_detect take ONE image (use detect_batch for more)"
        plan = self.plan_for(image.shape[1], image.shape[2])
        self._copy_in(plan, image)
        oh, ow = orig_hw if orig_hw is not None else (None, None)
        plan.launch(float(im_info[2]), oh, ow, post=post, detect=detect)
        return plan

    def detect(self, image, im_info, orig_hw):
        """Fused device path for im_detect + test_net's per-class NMS + max_per_image cap.
        Returns (det [n,6] = x1,y1,x2,y2,score,class; plan) after one stream sync (one D2H copy of the record)."""
        plan = self._run(image, im_info, post=True, detect=True, orig_hw=orig_hw)
        return plan.records()[0], plan

    def detect_batch(self, images, im_scales, orig_hws):
        """Throughput path: `images` [B,H,W,3] blobs of ONE shape (numpy or a pinned torch tensor), per-image scale factors and
        original (h, w).  -> (list of B det arrays [n,6], plan).  The reference is batch 1; this is SURVEY 8(f) rank 4."""
        plan, meta = self._batch_plan(images, im_scales, orig_hws)
        self._copy_in(plan, images)
        plan.launch(post=True, detect=True, meta=meta)
        return plan.records(), plan

    # ---- region features: per-detection head features, and scoring of caller-supplied boxes ---------------------------------
    def detect_features(self, images, im_scales, orig_hws):
        """detect_batch plus, for every detection, the head's per-RoI feature vector (fc7: 2048-d ResNet, 4096-d VGG16, 1024-d
        MobileNet) and the index of the RoI it came from, gathered on the device in the same graph replay.
        -> (list over images of (det [n,6], feats [n,F] fp32, roi_index [n] int32), plan); det equals detect_batch's records.
        Needs options['max_per_image'] > 0."""
        _no_bbox_aug("per-detection features (detect_features)")
        engine.check_feature_mode(int(self.options["max_per_image"]))
        plan, meta = self._batch_plan(images, im_scales, orig_hws)
        self._copy_in(plan, images)
        plan.launch(post=True, features=True, meta=meta)
        dets = plan.records()
        feats, rois = plan.feat_out.cpu(), plan.roi_out.cpu()
        return [(d, feats[i, :d.shape[0]].numpy().copy(), rois[i, :d.shape[0]].numpy().copy()) for i, d in enumerate(dets)], plan

    def detect_regions(self, images, im_scales, orig_hws, conf_thresh=0.2, min_boxes=10, max_boxes=100):
        """Bottom-up regions (Anderson et al. 2018, bottom-up-attention's generate_tsv.py): per image the distinct RoIs ranked by
        their best class confidence after per-class NMS over all RoIs (TEST.NMS, USE_GPU_NMS's predicate), the RoIs with
        confidence >= conf_thresh in ascending RoI order when there are min_boxes to max_boxes of them, else the top
        min(max(count, min_boxes), max_boxes) by confidence.  One graph replay after the network outputs; the definition is
        frcnn_detect_regions' (include/frcnn_b200.h).  TEST.SOFT_NMS, TEST.BBOX_VOTE and max_per_image do not apply.
        -> (list over images of dict(boxes [n,4] fp32 unregressed RoI boxes in image pixels, features [n,F] fp32, conf [n] fp32,
        classes [n] int32, roi_index [n] int32), plan).  With the attribute head on (cfg.ATTRIBUTES.NUM_CLASSES = A > 0) each dict
        also holds attr_prob [n, A] fp32, attributes [n] int32 (1 + the argmax of attr_prob[:, 1:]) and attr_conf [n] fp32, computed
        on the device in the same replay (frcnn_regions_attr_embed / frcnn_attr_finish).  ValueError before any device work for a conf_thresh outside [0, 1], counts
        that are not integers with 0 <= min_boxes <= max_boxes, max_boxes >= 1, and with TEST.BBOX_AUG enabled."""
        _no_bbox_aug("bottom-up regions (detect_regions)")
        args = engine.region_args(conf_thresh, min_boxes, max_boxes)
        plan, meta = self._batch_plan(images, im_scales, orig_hws)
        self._copy_in(plan, images)
        plan.launch(meta=meta, regions=args)
        return plan.regions(), plan

    def _run_boxes(self, images, im_scales, orig_hws, boxes):
        """Enqueue `images` [B,H,W,3] with caller boxes as the RoIs on a caller-box plan (no sync) -> plan."""
        _no_bbox_aug("caller boxes (score_boxes / im_detect(boxes=))")
        boxes = engine.check_boxes(boxes, int(images.shape[0]))
        engine.check_pool_boxes(self.options["pooling_mode"], boxes, im_scales, images.shape[1:3])
        plan, meta = self._batch_plan(images, im_scales, orig_hws, cap=engine.box_capacity(max(a.shape[0] for a in boxes)))
        self._copy_in(plan, images)
        plan.set_boxes(boxes)
        plan.launch(post=True, meta=meta)
        return plan

    def score_boxes(self, images, im_scales, orig_hws, boxes):
        """The Fast R-CNN mode: classify and regress caller boxes instead of RPN proposals.  boxes: per image an fp32 [n_i, 4]
        array (x1, y1, x2, y2 in original-image pixels, n_i <= 1024).  -> (list over images of (scores [n_i, C],
        pred_boxes [n_i, 4C], feats [n_i, F]), plan): im_detect's outputs for those boxes, plus the head features.
        With POOLING_MODE 'align' or 'pool', a non-finite box or one that leaves [-W, 2W] x [-H, 2H] of the blob once scaled raises
        ValueError before any device work."""
        plan = self._run_boxes(images, im_scales, orig_hws, boxes)
        out = []
        for i, a in enumerate(boxes):
            rows = slice(i * plan.R, i * plan.R + a.shape[0])
            out.append((plan.cls_prob[rows].cpu().numpy(), plan.pred_boxes[rows].cpu().numpy(), plan.fc7[rows].cpu().numpy()))
        return out, plan

    # ---- pipelined throughput API: overlap the next batch's host->device copy with the current batch's compute ---------------
    def submit_batch(self, images, im_scales, orig_hws):
        """Enqueue one batch without waiting for it: the H2D copy of `images` (a PINNED torch tensor or a numpy array, [B,H,W,3])
        runs on a copy stream into one of two staging buffers, the compute stream picks it up behind an event, replays the graph
        and copies the records into one of two pinned host buffers.  -> ticket for collect_batch().  At most TWO tickets may be
        outstanding (submit i+1, collect i, submit i+2, ...): that is what keeps the copy of batch i+1 under the compute of
        batch i.  Results are identical to detect_batch()."""
        plan, meta = self._batch_plan(images, im_scales, orig_hws)
        pipe = plan.__dict__.setdefault("_pipe", None)
        if pipe is None:
            pipe = plan._pipe = dict(copy_stream=torch.cuda.Stream(), stage=[torch.empty_like(plan.image) for _ in range(2)],
                                     staged=[torch.cuda.Event() for _ in range(2)], consumed=[torch.cuda.Event() for _ in range(2)],
                                     done=[torch.cuda.Event() for _ in range(2)], host=[None, None], turn=0, used=[False, False])
        k = pipe["turn"] & 1
        pipe["turn"] += 1
        src = images if isinstance(images, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(images, dtype=np.float32))
        main = torch.cuda.current_stream()
        with torch.cuda.stream(pipe["copy_stream"]):
            if pipe["used"][k]:
                pipe["copy_stream"].wait_event(pipe["consumed"][k])     # the compute stream has taken the previous content of stage k
            pipe["stage"][k].copy_(src, non_blocking=True)
            pipe["staged"][k].record(pipe["copy_stream"])
        main.wait_event(pipe["staged"][k])
        plan.image.copy_(pipe["stage"][k], non_blocking=True)             # device-to-device: ~microseconds, keeps the graph's input address fixed
        pipe["consumed"][k].record(main)
        pipe["used"][k] = True
        plan.launch(post=True, detect=True, meta=meta)
        if pipe["host"][k] is None or pipe["host"][k].shape != plan.rec.shape:
            pipe["host"][k] = torch.empty(plan.rec.shape, dtype=torch.float32).pin_memory()
        pipe["host"][k].copy_(plan.rec, non_blocking=True)
        pipe["done"][k].record(main)
        return (plan, k, plan.max_det)

    def collect_batch(self, ticket):
        """Wait for a submitted batch -> list of B det arrays [n,6]."""
        plan, k, max_det = ticket
        pipe = plan._pipe
        pipe["done"][k].synchronize()
        return engine.split_host_records(pipe["host"][k], max_det)
