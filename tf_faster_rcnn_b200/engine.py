"""Host-side executor of the TEST-mode graph on one GPU.

A `Tape` records, for one input shape, the ordered list of kernel launches (closures over
pre-built conv plans / static device buffers).  `Tape.run()` enqueues them on the current CUDA
stream; `ShapePlan` wraps a tape in a CUDA graph so that one image = one graph launch
(no tracing compiler: the graph is a recording of the explicit launches below).

Layer semantics follow lib/nets/network.py:233-262 (graph order), :323-378 (heads); the three
backbones emit their layers through the Tape from lib/nets/{vgg16,resnet_v1,mobilenet_v1}.py's
counterparts in tf_faster_rcnn_b200/lib/nets/.
"""
import collections
import ctypes
import os

import numpy as np
import torch

from . import _native as N
from . import ops

F = np.float32
C_void = ctypes.c_void_p


def bn_fold(gamma, beta, mean, var, eps):
    """tf.nn.batch_normalization (inference): y = x*inv + (beta - mean*inv), inv = gamma*rsqrt(var+eps)."""
    inv = (gamma.astype(F) * (F(1.0) / np.sqrt(var.astype(F) + F(eps)))).astype(F)
    return inv, (beta.astype(F) - mean.astype(F) * inv).astype(F)


def concat_layers(weights, names, bn_eps):
    """(w, scale, shift) of Weights.packed_concat on the host: W' = [W_1 diag(s_1) ; ...] in fp32, packed as w = W' / sigma
    with scale = sigma, the power of two per output channel that puts the column's largest |w| in [1, 2)
    (ops.column_scales); shift = the shifts added in order in fp32.

    Folding the BatchNorm scales moves them from the epilogue into the weights, so without sigma a channel whose scales
    are both small would sit far below the matrix's largest weight and lose the fp32 grade of the f16 split (it keeps 27
    binades below the layer's largest weight, ops.weight_exponent).  w * sigma == W' bit for bit (up to weights more than
    126 binades below their column's largest, whose quotient is subnormal and which the split drops anyway), and the
    epilogue's scale sigma * out_mult is a power of two, so the device multiplies by it exactly."""
    ss = [weights.scale_shift(nm, bn_eps) for nm in names]
    w = ops.concat_scaled_weights([weights[nm + "/weights"] for nm in names], [s for s, _ in ss])
    sigma = ops.column_scales(w)
    shift = ss[0][1]
    for _, sh in ss[1:]:
        shift = (shift + sh).astype(F)
    return (w / sigma).astype(F), sigma, shift


class Weights:
    """TF-variable-name -> numpy store plus a cache of device-packed layers (packed once per network)."""

    def __init__(self, tensors):
        self.t = tensors
        self._packed = {}
        self._dev = {}

    def __getitem__(self, k):
        return self.t[k]

    def __contains__(self, k):
        return k in self.t

    def dev(self, key, arr_fn):
        if key not in self._dev:
            self._dev[key] = torch.from_numpy(np.ascontiguousarray(arr_fn(), dtype=F)).cuda()
        return self._dev[key]

    def scale_shift(self, name, bn_eps):
        """epilogue vectors of layer `name`: BatchNorm fold when bn_eps is given, else (None, biases|None)."""
        if bn_eps is not None:
            p = name + "/BatchNorm/"
            return bn_fold(self.t[p + "gamma"], self.t[p + "beta"], self.t[p + "moving_mean"], self.t[p + "moving_variance"], bn_eps)
        b = self.t.get(name + "/biases")
        return None, (None if b is None else b.astype(F))

    def packed_conv(self, name, bn_eps=None, w_key="/weights"):
        if name not in self._packed:
            sc, sh = self.scale_shift(name, bn_eps)
            self._packed[name] = ops.PackedConv(self.t[name + w_key], sc, sh)
        return self._packed[name]

    def packed_concat(self, names, bn_eps):
        """One 1x1 layer computing the sum of the BatchNorm'd 1x1 layers `names` over their concatenated inputs:
        weights [W_1 diag(s_1) ; W_2 diag(s_2) ; ...] (scales folded in fp32, each output column normalised by a power of
        two that returns as its epilogue scale: concat_layers) and shift = the sum of the shifts in fp32."""
        key = "+".join(names)
        if key not in self._packed:
            self._packed[key] = ops.PackedConv(*concat_layers(self, names, bn_eps))
        return self._packed[key]

    def packed_custom(self, key, build):
        """build() -> (w_hwio, scale, shift) for fused layers (RPN heads, cls+bbox)."""
        if key not in self._packed:
            w, sc, sh = build()
            self._packed[key] = ops.PackedConv(w, sc, sh)
        return self._packed[key]


class LaunchGraph:
    """A recorded launch sequence as an executable CUDA graph, captured and replayed through the C ABI (frcnn_graph_*): plain
    cudaStreamBeginCapture / cudaGraphLaunch on the stream the stages were enqueued on -- no framework graph object, no
    generator-state fill kernels per replay.  FRCNN_TORCH_GRAPH=1 selects torch.cuda.CUDAGraph instead (A/B, debugging)."""

    def __init__(self, fns):
        self._h = ctypes.c_void_p()
        self._torch = None
        if os.environ.get("FRCNN_TORCH_GRAPH") == "1":
            self._torch = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self._torch):
                for fn in fns:
                    fn()
            return
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            N.check(N.lib().frcnn_graph_begin(C_void(side.cuda_stream)), "graph_begin")
            try:
                for fn in fns:
                    fn()
            finally:
                rc = N.lib().frcnn_graph_end(C_void(side.cuda_stream), ctypes.byref(self._h))
            N.check(rc, "graph_end")
        torch.cuda.current_stream().wait_stream(side)

    def replay(self):
        if self._torch is not None:
            self._torch.replay()
        else:
            N.check(N.lib().frcnn_graph_launch(self._h, ops._stream()), "graph_launch")

    def __del__(self):
        try:
            if self._h:
                N.lib().frcnn_graph_destroy(self._h)
                self._h = ctypes.c_void_p()
        except Exception:
            pass


class Tape:
    def __init__(self, weights):
        self.w = weights
        self.steps = []        # (label, callable)
        self.flops = 0.0       # algorithmic 2*MAC of every conv/FC layer recorded
        self.conv_flops = 0.0  # ... of the wgmma implicit-GEMM launches only
        self.bufs = []
        self.conv_plans = []   # ops.ConvPlan objects, in launch order

    def new(self, *shape, dtype=torch.float32):
        t = torch.empty(shape, dtype=dtype, device="cuda")
        self.bufs.append(t)
        return t

    def add(self, label, fn):
        self.steps.append((label, fn))

    def run(self):
        for _, fn in self.steps:
            fn()

    # ---- dense layers -------------------------------------------------------------------------------
    def conv(self, x, name, stride=1, mode="SAME", act=N.ACT_RELU, bn_eps=None, residual=None, packed=None, x2=None, mean=False):
        """x2: second input of a pointwise layer whose packed weights cover both inputs' channels (Weights.packed_concat).
        mean: return [n, cout], each image's spatial mean of the activated output (the output map is never stored)."""
        pc = packed if packed is not None else self.w.packed_conv(name, bn_eps)
        n, h, w, _ = x.shape
        ho, wo, pt, pl = ops.conv_out_hw(h, w, pc.kh, stride, mode)
        out = self.new(n, pc.cout) if mean else self.new(n, ho, wo, pc.cout)
        plan = ops.ConvPlan(x, pc, out, stride, pt, pl, act, residual, x2=x2, mean=mean)
        self.conv_plans.append(plan)
        self.add("conv:" + name, plan.run)
        fl = 2.0 * n * ho * wo * pc.cout * pc.kh * pc.kw * pc.cin
        self.flops += fl
        self.conv_flops += fl
        return out

    def fc(self, x2d, name, act=N.ACT_NONE, packed=None):
        r, k = x2d.shape
        out = self.conv(x2d.view(1, 1, r, k), name, 1, "SAME", act, None, None, packed)
        return out.view(r, -1)

    def conv_first(self, x, name, k, stride, mode, act, bn_eps=None):
        sc, sh = self.w.scale_shift(name, bn_eps)
        wd = self.w.dev(name + "/weights", lambda: self.w[name + "/weights"])
        scd = None if sc is None else self.w.dev(name + "/scale", lambda: sc)
        shd = None if sh is None else self.w.dev(name + "/shift", lambda: sh)
        n, h, w, _ = x.shape
        ho, wo, pt, pl = ops.conv_out_hw(h, w, k, stride, mode)
        cout = int(self.w[name + "/weights"].shape[3])
        out = self.new(n, ho, wo, cout)
        self.add("conv_first:" + name, lambda: ops.conv_first(x, wd, scd, shd, out, k, stride, pt, pl, act))
        self.flops += 2.0 * n * ho * wo * cout * k * k * 3
        return out

    def depthwise(self, x, name, stride, act, bn_eps):
        sc, sh = self.w.scale_shift(name, bn_eps)
        c = x.shape[3]
        wd = self.w.dev(name + "/dw", lambda: self.w[name + "/depthwise_weights"].reshape(3, 3, c))
        scd = self.w.dev(name + "/scale", lambda: sc)
        shd = self.w.dev(name + "/shift", lambda: sh)
        n, h, w, _ = x.shape
        ho, wo, pt, pl = ops.conv_out_hw(h, w, 3, stride, "SAME" if stride == 1 else "EXPLICIT")
        out = self.new(n, ho, wo, c)
        self.add("depthwise:" + name, lambda: ops.depthwise3x3(x, wd, scd, shd, out, stride, pt, pl, act))
        return out

    def max_pool(self, x, k, stride, mode):
        """mode 'SAME' (TF: padded cells never win) | 'ZEROPAD1' (tf.pad 1 + VALID) | 'VALID'."""
        n, h, w, c = x.shape
        if mode == "SAME":
            ho, wo = -(-h // stride), -(-w // stride)
            pt, _ = ops.same_pads(h, k, stride); pl, _ = ops.same_pads(w, k, stride)
            neg = True
        elif mode == "ZEROPAD1":
            ho, wo, pt, pl, neg = (h + 2 - k) // stride + 1, (w + 2 - k) // stride + 1, 1, 1, False
        else:
            ho, wo, pt, pl, neg = (h - k) // stride + 1, (w - k) // stride + 1, 0, 0, True
        out = self.new(n, ho, wo, c)
        self.add("max_pool", lambda: ops.max_pool(x, out, k, stride, pt, pl, neg))
        return out

    def spatial_mean(self, x):
        out = self.new(x.shape[0], x.shape[3])
        self.add("spatial_mean", lambda: ops.spatial_mean(x, out))
        return out


REC_HEADER = 8     # 4-byte words in front of every image's detection rows: word 0 = int32 detection count

# the options the post step is built for; a change rebuilds it (PostStage._ensure_post).  soft_nms: soft_nms_args() or None;
# box_vote: box_vote_args() or None
PostKey = collections.namedtuple("PostKey", "score_thresh nms_thresh use_gpu_nms max_per_image soft_nms box_vote", defaults=(None,))
# the options the bottom-up regions step is built for (PostStage._ensure_regions); conf_thresh is the fp32 threshold of region_args
RegionKey = collections.namedtuple("RegionKey", "conf_thresh min_boxes max_boxes nms_thresh use_gpu_nms")
REGION_FIELDS = ("boxes", "features", "conf", "classes", "roi_index")
ATTR_FIELDS = ("attr_prob", "attributes", "attr_conf")     # the attribute head's region fields (options['attributes'] on)


class PostStage:
    """The test_net tail of a plan whose im_detect outputs are `cls_prob`, `pred_boxes` and `num_rois` (`batch` images of `R`
    rows): the per-class NMS or Soft-NMS into `keep` / `keep_cnt` / `keep_score` (`post_ws`: the greedy NMS's workspace), with
    the box_vote option the voting into `vote_box`, the max_per_image cap and the detection records, built on first use for the
    options in force; in feature mode also the
    per-detection gather of `fc7`; in region mode the bottom-up regions step over `cls_prob`, `rois`, `num_rois`, `im_meta` and
    `fc7`.  The subclass allocates those buffers.  Two record buffers: with `double_buffer`,
    consecutive detect launches alternate between them.  Also the plan's CUDA-graph cache."""

    def __init__(self, net, batch, use_graph):
        self.net, self.batch = net, batch
        self.post_key = None
        self.regions_key = self.regions_step = None                 # region mode (_ensure_regions)
        self.reg_box = self.reg_key = self.reg_out = self.reg_ws = None
        self.attr_steps, self.attr_bufs = [], None                  # the attribute head on the regions (_build_attributes)
        self.recs = [None, None]
        self.rec = self.ndet = None    # views of the buffer the LAST detect launch wrote
        self.post_steps = [None, None]
        self.feat_out = self.roi_out = self.features_step = None   # feature mode (_ensure_post(features=True))
        self.vote_box = None                                        # box voting (_build_post)
        self.double_buffer = False
        self.slot = 0
        self.max_det = 0
        self.graphs = {}
        self.use_graph = use_graph

    def _ensure_post(self, features=False):
        """(Re)build the detection-record buffers and the post step for the current score / NMS thresholds, cap, Soft-NMS and
        box-voting settings; with `features`, also the per-detection feature buffers and their gather step."""
        o = self.net.options
        soft, vote = o.get("soft_nms"), o.get("box_vote")
        key = PostKey(float(o["score_thresh"]), float(o["nms_thresh"]), bool(o["use_gpu_nms"]), int(o["max_per_image"]),
                      None if soft is None else soft_nms_args(*soft), None if vote is None else box_vote_args(*vote))
        if key != self.post_key:
            self._build_post(key)
        if features and self.features_step is None:
            check_feature_mode(key.max_per_image)
            C, B, fdim = self.net.num_classes, self.batch, int(self.fc7.shape[1])
            # feat_out [B, max_det, F]: row k of image b = fc7 row of record row k; roi_out [B, max_det] int32 (-1 past the count)
            self.feat_out = ops.zeros((B, self.max_det, fdim))
            self.roi_out = ops.zeros((B, self.max_det), dtype=torch.int32)
            self.features_step = lambda: ops.detect_features(self.keep, self.keep_cnt, self.fc7, C, self.feat_out, self.roi_out)

    def _build_post(self, key):
        C, R, B = self.net.num_classes, self.R, self.batch
        mpi, soft = key.max_per_image, key.soft_nms
        # records: max_per_image survivors + head-room for ties at the threshold score; no cap -> every (roi, class) pair.
        # A record set that still does not fit is reported through ndet > max_det and raised on the host (never truncated).
        self.max_det = max_det = 2 * mpi + 56 if mpi > 0 else R * (C - 1)
        thr, flags = nms_threshold(key.nms_thresh, key.use_gpu_nms)
        # box voting: the voted boxes [B, C, R] float4 the records read (allocated only with the option on)
        self.vote_box = None if key.box_vote is None else ops.zeros((B, C, R, 4))
        vote = None if key.box_vote is None else (*key.box_vote, self.vote_box)

        def make_post(rec):
            # as_strided: view() repacks a size-1 batch dimension, which would drop the record stride at batch 1
            det, ndet = rec.as_strided((B, max_det, 6), (rec.stride(0), 6, 1), REC_HEADER), rec.view(torch.int32)[:, 0]
            if soft is not None:
                return lambda: ops.detect_post_soft(self.cls_prob, self.pred_boxes, self.num_rois, C, key.score_thresh, soft[0], soft[1],
                                                    float(F(key.nms_thresh)), soft[2], mpi, det, ndet, self.keep, self.keep_cnt,
                                                    self.keep_score, batch=B, vote=vote)
            return lambda: ops.detect_post(self.cls_prob, self.pred_boxes, self.num_rois, C, key.score_thresh, thr, flags, mpi, det, ndet,
                                           self.keep, self.keep_cnt, self.keep_score, self.post_ws, batch=B, vote=vote)
        self.recs = [ops.zeros((B, REC_HEADER + max_det * 6)) for _ in range(2)]
        self.post_steps = [make_post(r) for r in self.recs]
        self.post_key = key
        self._select(0)
        self.graphs.pop(("detect", 0), None); self.graphs.pop(("detect", 1), None)
        self.feat_out = self.roi_out = self.features_step = None
        self.graphs.pop(("features", 0), None)

    def _ensure_regions(self, conf_thresh, min_boxes, max_boxes):
        """(Re)build the bottom-up regions step for region_args' (fp32 conf_thresh, min_boxes, max_boxes) and the NMS options in
        force.  Its buffers are allocated on first use: the RoI boxes (broadcast over the classes up to
        ops.REGIONS_CLASS_NMS_MAX classes, one per row above), the per-RoI keys and min(max_boxes, R) output rows per image.  Up to
        REGIONS_CLASS_NMS_MAX classes the per-class NMS reuses keep / keep_cnt / keep_score / post_ws; above, the step needs only its
        own workspace (the per-image overlap masks)."""
        o = self.net.options
        key = RegionKey(float(conf_thresh), int(min_boxes), int(max_boxes), float(o["nms_thresh"]), bool(o["use_gpu_nms"]))
        if key == self.regions_key:
            return
        C, R, B = self.net.num_classes, self.R, self.batch
        per_class = C <= ops.REGIONS_CLASS_NMS_MAX
        if self.reg_box is None:
            self.reg_box = ops.zeros(ops.regions_box_shape(B * R, C))
            self.reg_key = ops.zeros((B * R,), dtype=torch.int64)
            self.reg_ws = self.post_ws if per_class else ops.detect_regions_workspace(R, C, B)
        M = min(key.max_boxes, R)
        if self.reg_out is None or self.reg_out["conf"].shape[1] != M:
            fdim = int(self.fc7.shape[1])
            self.reg_out = dict(boxes=ops.zeros((B, M, 4)), features=ops.zeros((B, M, fdim)), conf=ops.zeros((B, M)),
                                classes=ops.zeros((B, M), dtype=torch.int32), roi_index=ops.zeros((B, M), dtype=torch.int32),
                                count=ops.zeros((B,), dtype=torch.int32))
            self._build_attributes(M)
        thr, flags = nms_threshold(key.nms_thresh, key.use_gpu_nms)
        out = self.reg_out
        keep = (self.keep, self.keep_cnt, self.keep_score) if per_class else (None, None, None)
        self.regions_step = lambda: ops.detect_regions(self.cls_prob, self.rois, self.num_rois, self.im_meta, self.fc7, C, thr, flags,
                                                       key.conf_thresh, key.min_boxes, key.max_boxes, *keep, self.reg_ws, self.reg_box,
                                                       self.reg_key, out, batch=B)
        for g in [g for g in self.graphs if isinstance(g, tuple) and g[0] == "regions"]:
            del self.graphs[g]
        self.regions_key = key

    def _build_attributes(self, M):
        """The attribute head on reg_out's M rows per image when options['attributes'] = (A, E, H) is on (include/frcnn_b200.h,
        frcnn_regions_attr_embed): its outputs join reg_out (attr_prob [B, M, A], attributes int32 [B, M], attr_conf [B, M]),
        and its scratch is emb [B*M, E], hidden [B*M, H] and score [B*M, ld] (A zero-padded to a multiple of 4 columns, as the
        cls|bbox head).  fc_attr reads the region features and emb as its two A sources, so the conv plans hold these buffers'
        addresses and are rebuilt with them whenever M changes."""
        attrs = self.net.options.get("attributes")
        if attrs is None:
            self.attr_steps, self.attr_bufs = [], None
            return
        A, E, H = attrs
        wts, sc, B, C = self.net.weights, self.net.scope, self.batch, self.net.num_classes
        rows, lda = B * M, (A + 3) // 4 * 4
        out = self.reg_out
        out["attr_prob"] = ops.zeros((B, M, A)); out["attributes"] = ops.zeros((B, M), dtype=torch.int32); out["attr_conf"] = ops.zeros((B, M))
        emb, hidden, score = ops.zeros((rows, E)), ops.zeros((rows, H)), ops.zeros((rows, lda))
        table = wts.dev(sc + "/cls_embedding", lambda: wts[sc + "/cls_embedding/weights"])

        def padded_score():
            w = np.zeros((1, 1, H, lda), F); b = np.zeros(lda, F)
            w[0, 0, :, :A] = wts[sc + "/attr_score/weights"]; b[:A] = wts[sc + "/attr_score/biases"]
            return w, None, b
        fc_attr = ops.ConvPlan(out["features"].view(1, 1, rows, -1), wts.packed_conv(sc + "/fc_attr"), hidden.view(1, 1, rows, H),
                               act=N.ACT_RELU, x2=emb.view(1, 1, rows, E))
        attr_score = ops.ConvPlan(hidden.view(1, 1, rows, H), wts.packed_custom(sc + "/attr_score", padded_score), score.view(1, 1, rows, lda))
        self.attr_bufs = dict(emb=emb, hidden=hidden, score=score, plans=(fc_attr, attr_score))
        self.attr_steps = [lambda: ops.regions_attr_embed(self.cls_score, C, out["roi_index"], out["count"], table, emb),
                           fc_attr.run, attr_score.run,
                           lambda: ops.attr_finish(score, A, out["count"], out["attr_prob"], out["attributes"], out["attr_conf"])]

    def regions(self):
        """Host copy of the bottom-up regions of the batch after a 'regions' launch: per image a dict of boxes [n,4] fp32,
        features [n,F] fp32, conf [n] fp32, classes [n] int32, roi_index [n] int32, and with the attribute head attr_prob [n,A]
        fp32, attributes [n] int32, attr_conf [n] fp32."""
        host = {k: v.cpu() for k, v in self.reg_out.items()}
        counts = host["count"].numpy()
        fields = REGION_FIELDS + (ATTR_FIELDS if self.attr_bufs is not None else ())
        return [{k: host[k][b, :int(counts[b])].numpy().copy() for k in fields} for b in range(self.batch)]

    def _select(self, slot):
        self.slot = slot
        self.rec = self.recs[slot]
        self.ndet = self.rec.view(torch.int32)[:, 0]

    def _begin_post(self, features=False):
        """Build the post step if the options changed and pick this launch's record buffer: the other one with `double_buffer`,
        else buffer 0 (always 0 in feature mode, which does not double-buffer)."""
        self._ensure_post(features)
        self._select(self.slot ^ 1 if self.double_buffer and not features else 0)

    def _replay(self, gkey, fns):
        """Run the launch list fns: as the CUDA graph cached under gkey (captured on first use, after one eager warm-up pass
        for function attributes and lazy allocations), or eagerly without graphs."""
        if not self.use_graph:
            for fn in fns:
                fn()
            return
        g = self.graphs.get(gkey)
        if g is None:
            for fn in fns:
                fn()
            torch.cuda.current_stream().synchronize()
            g = self.graphs[gkey] = LaunchGraph(fns)
        g.replay()

    def records(self):
        """Host copy of the detection records of the batch after a 'detect' launch: list of [n,6] arrays (one D2H copy)."""
        return split_host_records(self.rec.cpu(), self.max_det)


class ShapePlan(PostStage):
    """Everything needed to run `batch` images of one blob shape: static input/output buffers, the tape, its CUDA graphs.

    The reference graph is batch 1 (lib/nets/network.py:388); batch > 1 is the throughput mode (SURVEY 8(f) rank 4): the
    backbone sees M = batch * H * W output pixels per layer (the 38x50 ResNet maps fill the 132 SMs without split-K), the
    per-RoI head sees batch * R RoIs, and the single-CTA proposal / NMS kernels run one CTA per image side by side.
    One image (or batch) = ONE graph replay: the im_detect / test_net tail is part of the graph, its per-image scalars
    (scale, original size) are read from `im_meta` on the device.

    rois_source="boxes" (the Fast R-CNN mode, TEST.HAS_RPN = False): the RoIs are `cap` caller boxes per image staged by
    set_boxes() instead of the RPN's proposals; the RPN is not built and the head / im_detect tail are the same steps."""

    def __init__(self, net, h, w, batch=1, use_graph=True, rois_source="rpn", cap=None):
        super().__init__(net, batch, use_graph)
        self.h, self.w = h, w
        cfgd = net.options
        wts = net.weights
        t = Tape(wts)
        self.tape = t
        B = batch
        self.image = t.new(B, h, w, 3)
        self.im_info = np.zeros(3, F)
        C = net.num_classes
        sc = net.scope
        # per-image (scale, orig_h, orig_w), read by bbox_decode (and boxes_to_rois).  Pinned staging for the meta rows: a ring,
        # because the H2D copies are asynchronous and the host may already be preparing the launch after next (submit_batch
        # keeps two batches in flight)
        self.im_meta = t.new(B, 3)
        self.im_meta_ring = [torch.empty((B, 3), dtype=torch.float32).pin_memory() for _ in range(4)]
        self.im_meta_turn = 0
        self.im_meta_ring[0][:] = torch.tensor([1.0, float(h), float(w)])
        self.im_meta.copy_(self.im_meta_ring[0])
        # ---- backbone -----------------------------------------------------------------------------------
        feat = net._image_to_head(t, self.image)
        self.feat = feat
        _, fh, fw, cb = feat.shape
        assert fh == -(-h // 16) and fw == -(-w // 16), "feature map %dx%d does not match ceil(H/16) x ceil(W/16)" % (fh, fw)
        if rois_source == "boxes":
            self._caller_rois(t, cap)
        else:
            self._rpn_rois(t, feat)
        R = self.R
        # ---- RoI pooling (network.py:141-157 / resnet_v1.py:55-76) ---------------------------------------
        P = cfgd["pooling_size"]
        self.pool5 = t.new(B * R, P, P, cb)
        mode = cfgd["pooling_mode"]
        if mode == "align":        # extensions: P x P straight from the map, no 2P crop + 2x2 max
            sr, aligned = cfgd["roi_align"]
            t.add("roi_align", lambda: ops.roi_align(feat, self.rois, P, SPATIAL_SCALE, sr, aligned, self.pool5))
        elif mode == "pool":
            t.add("roi_pool", lambda: ops.roi_pool(feat, self.rois, P, SPATIAL_SCALE, self.pool5))
        else:
            pre_pool = net.crop_pre_pool()
            t.add("crop_pool", lambda: ops.crop_pool(feat, self.rois, P, pre_pool, self.pool5))
        # ---- per-RoI head + fused cls_score|bbox_pred FC (network.py:361-378) ------------------------------
        fc7 = net._head_to_tail(t, self.pool5)
        self.fc7 = fc7

        ld_head = (5 * C + 3) // 4 * 4            # zero-padded to a multiple of 4 columns: vector stores + split-K apply

        def fused_cls():
            wc, wb = wts[sc + "/cls_score/weights"], wts[sc + "/bbox_pred/weights"]
            wf = np.zeros((1, 1, wc.shape[0], ld_head), F); bf = np.zeros(ld_head, F)
            wf[0, 0, :, :C] = wc; wf[0, 0, :, C:5 * C] = wb
            bf[:C] = wts[sc + "/cls_score/biases"]; bf[C:5 * C] = wts[sc + "/bbox_pred/biases"]
            return wf, None, bf
        self.head_out = t.fc(fc7, sc + "/cls_bbox", N.ACT_NONE, packed=wts.packed_custom(sc + "/cls_bbox", fused_cls))
        self.cls_score = t.new(B * R, C); self.cls_prob = t.new(B * R, C); self.bbox_pred = t.new(B * R, 4 * C)
        stds, means = cfgd["bbox_stds"], cfgd["bbox_means"]
        t.add("cls_finish", lambda: ops.cls_finish(self.head_out, C, stds, means, self.cls_score, self.cls_prob, self.bbox_pred))
        self.n_test_image_steps = len(t.steps)
        # ---- im_detect tail on the device (test.py:95-107): per-image (scale, orig_h, orig_w) live in im_meta --------------
        self.pred_boxes = t.new(B * R, 4 * C)
        t.add("bbox_decode", lambda: ops.bbox_decode(self.rois, self.bbox_pred, C, self.im_meta, self.pred_boxes))
        self.n_im_detect_steps = len(t.steps)
        # ---- test_net tail (test.py:162-180): built on first use for the options in force (_ensure_post) ---------------------
        self.keep = t.new(B, C, R, dtype=torch.int32); self.keep_cnt = t.new(B, C, dtype=torch.int32)
        self.keep_score = t.new(B, C, R)
        self.post_ws = ops.detect_post_workspace(R, C, B); t.bufs.append(self.post_ws)

    def _caller_rois(self, t, cap):
        """RoIs from caller boxes: [batch, cap, 4] boxes + int32 counts staged through a pinned ring (set_boxes)."""
        B = self.batch
        self.R = cap
        self.rpn_out = self.rpn_dcol = self.roi_scores = self.roi_keep = None
        self.boxes = t.new(B, cap, 4); self.box_counts = t.new(B, dtype=torch.int32)
        self.box_ring = [(torch.zeros((B, cap, 4), dtype=torch.float32).pin_memory(), torch.zeros(B, dtype=torch.int32).pin_memory())
                         for _ in range(4)]
        self.box_turn = 0
        self.box_counts.zero_()
        self.rois = t.new(B * cap, 5); self.num_rois = t.new(B, dtype=torch.int32)
        t.add("boxes_to_rois", lambda: ops.boxes_to_rois(self.boxes, self.box_counts, self.im_meta, self.rois, self.num_rois))

    def set_boxes(self, boxes):
        """boxes: per image an fp32 [n_i, 4] array (original-image pixels, n_i <= cap); staged in pinned memory and copied on
        the launching stream, like set_meta."""
        self.box_turn = (self.box_turn + 1) & 3
        hb, hc = self.box_ring[self.box_turn]
        for b, a in enumerate(boxes):
            n = a.shape[0]
            hc[b] = n
            if n:
                hb[b, :n] = torch.from_numpy(a)
        self.boxes.copy_(hb, non_blocking=True)
        self.box_counts.copy_(hc, non_blocking=True)

    def _rpn_rois(self, t, feat):
        """RoIs from the RPN: 3x3 conv, fused cls|bbox 1x1, decode, sort, proposal NMS."""
        net, B, h, w = self.net, self.batch, self.h, self.w
        cfgd, wts, sc, A = net.options, net.weights, net.scope, net.num_anchors
        _, fh, fw, _ = feat.shape
        # ---- RPN (network.py:323-359): 3x3 conv + ONE fused 1x1 for cls(2A) | pad | bbox(4A) ---------------
        rpn = t.conv(feat, sc + "/rpn_conv/3x3", 1, "SAME", N.ACT_RELU)
        dcol = (2 * A + 3) // 4 * 4
        ld = (dcol + 4 * A + 3) // 4 * 4

        def fused_rpn():
            cin = int(wts[sc + "/rpn_cls_score/weights"].shape[2])
            wf = np.zeros((1, 1, cin, ld), F); bf = np.zeros(ld, F)
            wf[..., :2 * A] = wts[sc + "/rpn_cls_score/weights"]; bf[:2 * A] = wts[sc + "/rpn_cls_score/biases"]
            wf[..., dcol:dcol + 4 * A] = wts[sc + "/rpn_bbox_pred/weights"]; bf[dcol:dcol + 4 * A] = wts[sc + "/rpn_bbox_pred/biases"]
            return wf, None, bf
        rpn_out = t.conv(rpn, sc + "/rpn_heads", 1, "SAME", N.ACT_NONE, packed=wts.packed_custom(sc + "/rpn_heads", fused_rpn))
        self.rpn_out, self.rpn_dcol = rpn_out, dcol
        nanch = fh * fw * A
        self.nanch = nanch
        self.rpn_scores = t.new(B * nanch); self.rpn_props = t.new(B * nanch, 4)
        base = wts.dev("base_anchors/%s" % (net.anchor_key,), lambda: net.base_anchors)
        im_hw = (float(h), float(w))
        t.add("rpn_decode", lambda: ops.rpn_decode(rpn_out.view(B * fh * fw, ld), dcol, base, A, fh, fw, im_hw[0], im_hw[1],
                                                   self.rpn_scores, self.rpn_props, batch=B))
        self.order = t.new(B * nanch, dtype=torch.int32); self.sorted_scores = t.new(B * nanch)
        t.add("sort_desc", lambda: ops.sort_desc(self.rpn_scores, self.order, self.sorted_scores, None, batch=B))
        # ---- proposals (proposal_layer_tf | proposal_layer | proposal_top_layer) ---------------------------
        if cfgd["test_mode"] == "top":
            R, pre, thr, flags = cfgd["rpn_top_n"], 0, -1.0, 0
        elif cfgd["use_e2e_tf"]:
            R, pre, thr, flags = cfgd["rpn_post_nms_top_n"], 0, float(F(cfgd["rpn_nms_thresh"])), N.NMS_MODE_TF
        else:
            R, pre = cfgd["rpn_post_nms_top_n"], cfgd["rpn_pre_nms_top_n"]
            thr, flags = nms_threshold(cfgd["rpn_nms_thresh"], cfgd["use_gpu_nms"])
        self.R = R
        self.rois = t.new(B * R, 5); self.roi_scores = t.new(B * R)
        self.roi_keep = t.new(B * R, dtype=torch.int32); self.num_rois = t.new(B, dtype=torch.int32)
        t.add("proposals", lambda: ops.proposals(self.rpn_props, self.rpn_scores, self.order, pre, R, thr, flags, self.rois,
                                                 self.roi_scores, self.roi_keep, self.num_rois, batch=B))

    def nbytes(self):
        return sum(b.numel() * b.element_size() for b in self.tape.bufs)

    def release(self):
        """Drop graphs, conv plans (TMA descriptors, split-K workspaces) and activation buffers (LRU eviction)."""
        self.graphs.clear()
        self.tape.steps = []
        self.tape.conv_plans = []
        self.tape.bufs = []
        self.post_steps = [None, None]
        self.recs = [None, None]
        self.rec = self.ndet = None
        self.feat_out = self.roi_out = self.features_step = None
        self.regions_key = self.regions_step = None
        self.reg_box = self.reg_key = self.reg_out = self.reg_ws = None
        self.attr_steps, self.attr_bufs = [], None

    def steps_for(self, mode):
        """mode: 'test_image' (network outputs), 'im_detect' (+ decoded boxes), 'detect' (+ per-class NMS, cap, records),
        'features' (+ the head feature and RoI index of every record row); the last two after _begin_post.  'regions': the
        network outputs + the bottom-up regions step (no box decode, no records) + the attribute head when it is on, after
        _ensure_regions."""
        if mode in ("test_image", "regions"):
            fns = [fn for _, fn in self.tape.steps[:self.n_test_image_steps]]
            return fns + [self.regions_step] + self.attr_steps if mode == "regions" else fns
        fns = [fn for _, fn in self.tape.steps[:self.n_im_detect_steps]]
        if mode in ("detect", "features"):
            fns.append(self.post_steps[self.slot])
        if mode == "features":
            fns.append(self.features_step)
        return fns

    def set_meta(self, rows):
        """rows: per image (im_scale, orig_h, orig_w); staged in pinned memory, copied on the launching stream."""
        self.im_meta_turn = (self.im_meta_turn + 1) & 3
        host = self.im_meta_ring[self.im_meta_turn]
        for b, (s, oh, ow) in enumerate(rows):
            host[b, 0] = float(F(s)); host[b, 1] = float(oh); host[b, 2] = float(ow)
        self.im_meta.copy_(host, non_blocking=True)

    def launch(self, im_scale=1.0, orig_h=None, orig_w=None, post=False, detect=False, meta=None, features=False, regions=None):
        """Enqueue one batch (inputs already in self.image) on the current stream.  meta: per-image (scale, orig_h, orig_w)
        rows; the scalar arguments describe every image of the batch when meta is None.  features: detect + the feature
        gather into feat_out / roi_out (always record buffer 0: feature mode does not double-buffer).  regions: region_args'
        (conf_thresh, min_boxes, max_boxes) -> the network outputs + the bottom-up regions into reg_out (see regions())."""
        mode = "regions" if regions is not None else "features" if features else "detect" if detect else ("im_detect" if post else "test_image")
        if mode != "test_image":
            if meta is None:
                meta = [(im_scale, orig_h if orig_h is not None else self.h, orig_w if orig_w is not None else self.w)] * self.batch
            self.set_meta(meta)
        gkey = mode
        if mode in ("detect", "features"):
            self._begin_post(features)
            gkey = (mode, self.slot)
        elif mode == "regions":
            self._ensure_regions(*regions)
            gkey = ("regions", self.regions_key)
        self._replay(gkey, self.steps_for(mode))


AUG_MAX_ROIS = 8192    # RoI rows per image that the post step (ops.detect_post / _soft) takes: the cap of the union


class AugPlan(PostStage):
    """Test-time augmentation (TEST.BBOX_AUG) for `batch` images whose views have the blob shapes `views` = ((h, w, flip), ...),
    in union order.  Views of one blob shape share one ShapePlan at batch k*batch from the network's plan cache: unflipped views
    take the first slots, so an identity view and its flip are slots [0, B) and [B, 2B) of a batch-2B plan.  One call replays
    the sub-plans' im_detect graphs, then frcnn_aug_union merges the views' rows into the union buffers and the post step runs
    on them.  The union, the post step and its two alternating record buffers are this object's; the post step is the same
    PostStage as a ShapePlan's, run on R = the sum of the views' rows."""

    def __init__(self, net, views, batch):
        super().__init__(net, int(batch), net.use_cuda_graph)
        self.views = tuple(views)
        B, C = self.batch, net.num_classes
        self.shapes, self.view_slot, counts = aug_groups(self.views)
        self.group_batch = {hw: k * B for hw, k in counts.items()}
        self.subs = {}
        self.bind()
        self.rows = [self.subs[(h, w)].R for h, w, _ in self.views]
        R = self.R = sum(self.rows)
        self.cls_prob = ops.zeros((B * R, C)); self.pred_boxes = ops.zeros((B * R, 4 * C))
        self.num_rois = ops.zeros((B,), dtype=torch.int32)
        self.keep = ops.zeros((B, C, R), dtype=torch.int32); self.keep_cnt = ops.zeros((B, C), dtype=torch.int32)
        self.keep_score = ops.zeros((B, C, R))
        self.post_ws = ops.detect_post_workspace(R, C, B)

    def bind(self):
        """Fetch the sub-plans from the network's plan cache (marking them recently used).  A plan evicted by the LRU and rebuilt
        is a new object with new buffers: then the union's pointer table is rebuilt and the captured union / post graphs are
        dropped."""
        changed = False
        for hw in self.shapes:
            p = self.net.plan_for(hw[0], hw[1], self.group_batch[hw])
            if self.subs.get(hw) is not p:
                self.subs[hw] = p
                changed = True
        if changed:
            B, C = self.batch, self.net.num_classes
            table = []
            for v, (h, w, flip) in enumerate(self.views):
                p, k = self.subs[(h, w)], self.view_slot[v] * B
                table.append((p.cls_prob.data_ptr() + 4 * k * p.R * C, p.pred_boxes.data_ptr() + 16 * k * p.R * C,
                              p.num_rois.data_ptr() + 4 * k, p.R, flip))
            p0 = self.subs[self.views[0][:2]]
            self.table, self.meta_ptr = table, p0.im_meta.data_ptr() + 12 * self.view_slot[0] * B
            self.graphs.clear()

    def view_image(self, v):
        """View v's input slice [batch, h, w, 3] of its sub-plan's image buffer (fill it, then launch)."""
        B, k = self.batch, self.view_slot[v]
        return self.subs[self.views[v][:2]].image[k * B:(k + 1) * B]

    def _union(self):
        ops.aug_union(self.table, self.net.num_classes, self.meta_ptr, self.cls_prob, self.pred_boxes, self.num_rois)

    def launch(self, scales, orig_hws, detect=True):
        """Enqueue one call (inputs already in view_image(v)).  scales[v][b]: view v's scale factor of image b; orig_hws: per
        image (h, w).  detect=False stops after the union (im_detect's outputs in cls_prob / pred_boxes / num_rois)."""
        B = self.batch
        metas = {hw: [None] * p.batch for hw, p in self.subs.items()}
        for v, (h, w, _) in enumerate(self.views):
            k = self.view_slot[v] * B
            for b in range(B):
                metas[(h, w)][k + b] = (float(scales[v][b]), int(orig_hws[b][0]), int(orig_hws[b][1]))
        for hw, p in self.subs.items():
            p.launch(post=True, meta=metas[hw])
        if not detect:
            self._union()
            return
        self._begin_post()
        self._replay(("detect", self.slot), [self._union, self.post_steps[self.slot]])


def aug_groups(views):
    """views ((h, w, flip), ...) -> (distinct (h, w) in first-use order, slot of each view within its shape's plan, views per
    shape).  Unflipped views take the lower slots, then flipped ones, each in view order."""
    shapes, counts, slot = [], {}, [0] * len(views)
    for h, w, _ in views:
        if (h, w) not in shapes:
            shapes.append((h, w))
    for v in sorted(range(len(views)), key=lambda v: (bool(views[v][2]), v)):
        hw = tuple(views[v][:2])
        slot[v] = counts.get(hw, 0)
        counts[hw] = slot[v] + 1
    return shapes, slot, counts


def aug_rois_per_view(options):
    """RoI rows per image of one view: what ShapePlan._rpn_rois allots (RPN_TOP_N in 'top' mode, else RPN_POST_NMS_TOP_N)."""
    return int(options["rpn_top_n"] if options["test_mode"] == "top" else options["rpn_post_nms_top_n"])


def check_aug_views(views, rois_per_view, max_plans):
    """views: ((h, w, flip), ...) of one call; raises ValueError before any device work."""
    nv = len(views)
    if not 0 < nv <= N.AUG_MAX_VIEWS:
        raise ValueError("test-time augmentation with %d views: 1 to %d are supported" % (nv, N.AUG_MAX_VIEWS))
    if nv * rois_per_view > AUG_MAX_ROIS:
        raise ValueError("test-time augmentation: %d views x %d RoIs = %d union rows per image, more than the %d the per-class NMS "
                         "takes (fewer views, or fewer RoIs per view)" % (nv, rois_per_view, nv * rois_per_view, AUG_MAX_ROIS))
    shapes = len(set((int(h), int(w)) for h, w, _ in views))
    if shapes > max_plans:
        raise ValueError("test-time augmentation: the views have %d distinct blob shapes but the plan cache holds %d "
                         "(Network.MAX_PLANS); the plans of one call would evict each other" % (shapes, max_plans))


def bbox_aug_option(node, bbox_reg=True):
    """cfg.TEST.BBOX_AUG -> None when disabled, else the checked (H_FLIP, SCALES, MAX_SIZE); raises ValueError before any device
    work.  The view count is (1 + len(SCALES)) * (2 if H_FLIP else 1)."""
    if not node["ENABLED"]:
        return None
    if not bbox_reg:
        raise ValueError("TEST.BBOX_AUG needs TEST.BBOX_REG = True: the union merges the views' regressed boxes")
    scales = tuple(node["SCALES"])
    for s in scales:
        if not s > 0:
            raise ValueError("TEST.BBOX_AUG.SCALES must be positive short sides, got %r" % (scales,))
    if not node["MAX_SIZE"] > 0:
        raise ValueError("TEST.BBOX_AUG.MAX_SIZE must be positive, got %r" % (node["MAX_SIZE"],))
    nv = (1 + len(scales)) * (2 if node["H_FLIP"] else 1)
    if nv > N.AUG_MAX_VIEWS:
        raise ValueError("TEST.BBOX_AUG gives %d views: at most %d are supported" % (nv, N.AUG_MAX_VIEWS))
    return bool(node["H_FLIP"]), scales, node["MAX_SIZE"]


def split_host_records(host, max_det):
    """host: CPU float32 tensor [B, REC_HEADER + max_det*6] -> list of [n,6] numpy arrays; raises when a record set did not fit."""
    counts = host.view(torch.int32)[:, 0].numpy()
    out = []
    for b in range(host.shape[0]):
        n = int(counts[b])
        if n > max_det:
            raise RuntimeError("image %d of the batch produced %d detections but the record buffer holds %d "
                               "(score ties beyond the max_per_image head-room)" % (b, n, max_det))
        out.append(host[b, REC_HEADER:REC_HEADER + n * 6].view(n, 6).numpy().copy())
    return out


BOX_CAPACITIES = (64, 128, 256, 512, 1024)   # caller-box plans are built per (shape, batch, capacity): few distinct graphs


def box_capacity(n):
    """Smallest capacity in BOX_CAPACITIES that holds n caller boxes per image."""
    for cap in BOX_CAPACITIES:
        if n <= cap:
            return cap
    raise ValueError("%d boxes for one image: at most %d per call, split them over several calls" % (n, BOX_CAPACITIES[-1]))


def check_boxes(boxes, batch):
    """Caller boxes: a list of `batch` fp32 [n_i, 4] arrays (x1, y1, x2, y2 in original-image pixels) -> contiguous copies."""
    if len(boxes) != batch:
        raise ValueError("%d box arrays for %d images" % (len(boxes), batch))
    out = []
    for i, b in enumerate(boxes):
        a = b.numpy() if isinstance(b, torch.Tensor) else np.asarray(b)
        if a.ndim != 2 or a.shape[1] != 4:
            raise ValueError("boxes[%d] has shape %s, expected [n, 4]" % (i, tuple(a.shape)))
        if a.dtype != np.float32:
            raise TypeError("boxes[%d] has dtype %s, expected float32" % (i, a.dtype))
        out.append(np.ascontiguousarray(a))
    return out


POOLING_MODES = ("crop", "align", "pool")
SPATIAL_SCALE = 1.0 / 16     # the stride-16 feature map of every backbone


def roi_align_option(pooling_mode, pooling_size, node):
    """cfg.POOLING_MODE / POOLING_SIZE / ROI_ALIGN -> the network option: None outside 'align' mode, else the checked
    (SAMPLING_RATIO, ALIGNED).  An unknown mode raises NotImplementedError, an invalid value ValueError, before any device work."""
    if pooling_mode not in POOLING_MODES:
        raise NotImplementedError("POOLING_MODE %r: expected one of %s" % (pooling_mode, ", ".join(POOLING_MODES)))
    if pooling_mode == "crop":
        # crop_and_resize to P x P (or 2P x 2P before the 2x2 max pool) divides by P - 1: frcnn_crop_pool takes 2 <= P <= 16
        if type(pooling_size) is not int or not 2 <= pooling_size <= N.ROI_MAX_POOLED:
            raise ValueError("POOLING_SIZE must be an int in [2, %d] in 'crop' mode, got %r" % (N.ROI_MAX_POOLED, pooling_size))
        return None
    if type(pooling_size) is not int or not 1 <= pooling_size <= N.ROI_MAX_POOLED:
        raise ValueError("POOLING_SIZE must be an int in [1, %d] in %r mode, got %r" % (N.ROI_MAX_POOLED, pooling_mode, pooling_size))
    if pooling_mode == "pool":
        return None
    sr, aligned = node["SAMPLING_RATIO"], node["ALIGNED"]
    if type(sr) is not int or not 0 <= sr <= N.ROI_ALIGN_MAX_SAMPLING:
        raise ValueError("ROI_ALIGN.SAMPLING_RATIO must be an int in [0, %d] (0 = adaptive), got %r" % (N.ROI_ALIGN_MAX_SAMPLING, sr))
    if type(aligned) is not bool:
        raise ValueError("ROI_ALIGN.ALIGNED must be a bool, got %r" % (aligned,))
    return (sr, aligned)


def check_rpn_channels(n):
    """cfg.RPN_CHANNELS: the fused RPN heads take it as K, which the conv kernel walks in 32-channel k-blocks."""
    if not _is_int(n) or n <= 0 or n % 32:
        raise ValueError("RPN_CHANNELS must be a positive multiple of 32, got %r" % (n,))


def attributes_option(node):
    """cfg.ATTRIBUTES -> the network option: None when NUM_CLASSES is 0, else (NUM_CLASSES, EMBED_DIM, HIDDEN); ValueError before
    any device work.  EMBED_DIM and HIDDEN are K of the fc_attr / attr_score FCs (EMBED_DIM as the second source's channels),
    which the conv kernel walks in 32-channel k-blocks."""
    a, e, h = node["NUM_CLASSES"], node["EMBED_DIM"], node["HIDDEN"]
    if not _is_int(a) or not (a == 0 or 2 <= a <= MAX_CLASSES):
        raise ValueError("ATTRIBUTES.NUM_CLASSES must be an integer, 0 (no attribute head) or in [2, %d], got %r" % (MAX_CLASSES, a))
    for key, v in (("EMBED_DIM", e), ("HIDDEN", h)):
        if not _is_int(v) or v <= 0 or v % 32:
            raise ValueError("ATTRIBUTES.%s must be a positive multiple of 32, got %r" % (key, v))
    return None if a == 0 else (int(a), int(e), int(h))


def check_pool_boxes(pooling_mode, boxes, im_scales, blob_hw):
    """In 'align' and 'pool' mode, refuse caller boxes (original-image pixels) that are not finite or that, scaled into the
    blob as boxes_to_rois does (fp32 box * fp32 scale), leave [-W, 2W] x [-H, 2H] of the H x W blob: RoIAlign's adaptive
    grid grows with the box (this keeps it at most about ceil(3 * map size / POOLING_SIZE) per axis), and RoIPool's integer
    corners must not overflow.  Crop mode takes any box, as before."""
    if pooling_mode == "crop":
        return
    h, w = float(blob_hw[0]), float(blob_hw[1])
    for i, (a, s) in enumerate(zip(boxes, im_scales)):
        if not np.isfinite(a).all():
            raise ValueError("boxes[%d] has a non-finite coordinate (POOLING_MODE %r)" % (i, pooling_mode))
        r = a * F(s)
        x, y = r[:, 0::2], r[:, 1::2]
        if (x < -w).any() or (x > 2 * w).any() or (y < -h).any() or (y > 2 * h).any():
            raise ValueError("boxes[%d]: in POOLING_MODE %r a box scaled into the %dx%d blob must lie within [-W, 2W] x [-H, 2H]"
                             % (i, pooling_mode, int(h), int(w)))


def f32_not_below(t):
    """The smallest fp32 value >= the float64 t: for every fp32 x, x >= t (in float64) <=> x >= f32_not_below(t) (in fp32)."""
    t32 = F(t)
    if float(t32) < float(t):
        t32 = np.nextafter(t32, F(np.inf))
    return t32


def _is_int(v):
    return isinstance(v, (int, np.integer)) and not isinstance(v, (bool, np.bool_))


MAX_CLASSES = 4096   # classes (background included) every detection path handles (include/frcnn_b200.h)


def check_num_classes(num_classes):
    """The class count of a network: an int in [2, MAX_CLASSES], else ValueError."""
    if not _is_int(num_classes) or not 2 <= num_classes <= MAX_CLASSES:
        raise ValueError("num_classes must be an integer in [2, %d] (background included), got %r" % (MAX_CLASSES, num_classes))
    return int(num_classes)


def region_args(conf_thresh, min_boxes, max_boxes):
    """Bottom-up region parameters -> (fp32 conf threshold: the smallest fp32 not below conf_thresh, min_boxes, max_boxes);
    raises ValueError before any device work."""
    try:
        t = float(conf_thresh)
    except (TypeError, ValueError):
        raise ValueError("conf_thresh must be a number in [0, 1], got %r" % (conf_thresh,))
    if isinstance(conf_thresh, (bool, np.bool_)) or not np.isfinite(t) or not 0.0 <= t <= 1.0:
        raise ValueError("conf_thresh must be a finite number in [0, 1], got %r" % (conf_thresh,))
    if not (_is_int(min_boxes) and _is_int(max_boxes)):
        raise ValueError("min_boxes / max_boxes must be integers, got %r / %r" % (min_boxes, max_boxes))
    if min_boxes < 0 or max_boxes < 1 or min_boxes > max_boxes:
        raise ValueError("need 0 <= min_boxes <= max_boxes and max_boxes >= 1, got min_boxes %d, max_boxes %d" % (min_boxes, max_boxes))
    return float(f32_not_below(t)), int(min_boxes), int(max_boxes)


def check_feature_mode(max_per_image):
    if max_per_image <= 0:
        raise ValueError("per-detection features need max_per_image > 0: without the cap the record buffer holds every "
                         "(RoI, class) pair, R*(C-1) feature rows per image (hundreds of MB)")


def soft_nms_args(method, sigma, score_thresh):
    """Soft-NMS parameters -> (FRCNN_SOFT_NMS_* code, fp32 sigma, fp32 prune threshold); raises ValueError before any device work."""
    if method not in N.SOFT_NMS_METHODS:
        raise ValueError("Soft-NMS METHOD %r: expected one of %s" % (method, ", ".join(sorted(N.SOFT_NMS_METHODS))))
    s32, t32 = F(sigma), F(score_thresh)
    if not s32 > 0:
        raise ValueError("Soft-NMS SIGMA must be > 0, got %r" % (sigma,))
    if not t32 > 0:
        raise ValueError("Soft-NMS SCORE_THRESH must be > 0 (the record cap assumes positive scores), got %r" % (score_thresh,))
    return N.SOFT_NMS_METHODS[method], float(s32), float(t32)


def soft_nms_option(node):
    """cfg.TEST.SOFT_NMS -> the network option: None when disabled, else the checked (METHOD, SIGMA, SCORE_THRESH)."""
    if not node["ENABLED"]:
        return None
    soft_nms_args(node["METHOD"], node["SIGMA"], node["SCORE_THRESH"])
    return (node["METHOD"], float(node["SIGMA"]), float(node["SCORE_THRESH"]))


def box_vote_args(vote_th, scoring_method="ID", beta=1.0):
    """Box-voting parameters -> (fp32 VOTE_TH, FRCNN_BOX_VOTE_* code, fp32 beta); raises ValueError before any device work."""
    if scoring_method not in N.BOX_VOTE_METHODS:
        raise ValueError("box voting SCORING_METHOD %r: expected one of %s" % (scoring_method, ", ".join(N.BOX_VOTE_METHODS)))
    t32, b32 = F(vote_th), F(beta)
    if not 0 < t32 <= 1:
        raise ValueError("box voting VOTE_TH must lie in (0, 1], got %r" % (vote_th,))
    if not (np.isfinite(b32) and b32 > 0):
        raise ValueError("box voting SCORING_METHOD_BETA must be finite and > 0, got %r" % (beta,))
    return float(t32), N.BOX_VOTE_METHODS[scoring_method], float(b32)


def box_vote_option(node):
    """cfg.TEST.BBOX_VOTE -> the network option: None when disabled, else the checked (VOTE_TH, SCORING_METHOD, SCORING_METHOD_BETA)."""
    if not node["ENABLED"]:
        return None
    box_vote_args(node["VOTE_TH"], node["SCORING_METHOD"], node["SCORING_METHOD_BETA"])
    return (float(node["VOTE_TH"]), node["SCORING_METHOD"], float(node["SCORING_METHOD_BETA"]))


def nms_threshold(thresh, use_gpu_nms):
    """(fp32 threshold, flags) reproducing the reference's two '+1' predicates:
    cpu_nms compares the fp32 overlap with a DOUBLE threshold using >= (cpu_nms.pyx:17,65)  <=> ovr >= ceil32(t);
    gpu_nms compares with float(t) using > (nms_kernel.cu:34,71)."""
    if use_gpu_nms:
        return float(F(thresh)), N.NMS_MODE_GPU_NMS
    return float(f32_not_below(thresh)), N.NMS_MODE_CPU_NMS
