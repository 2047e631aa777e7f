"""The poisoned-replay audit of the `detect` graph (helper of test_graph_audit_gpu.py, test_config_audit_gpu.py and
test_wide_head_gpu.py).

`build` makes a network of any architecture option (anchor set, RPN_CHANNELS, MobileNet depth multiplier, pooling mode and
size, RESNET.MAX_POOL, ...) on synth weights of that architecture and records every tape step's outputs; `run_audit` builds
the plan on other images, fills every tape and record buffer with 0xff bytes, replays the cached graph once on the audited
images and audits every step against float64 (or its exact model) fed the device outputs of its own inputs
(`net_ref64.audit`), then re-runs the steps eagerly one at a time: each step's outputs equal the replay's bit for bit, and no
step changes a buffer it does not declare as its output.  test_graph_audit_gpu.py says what the ordering check covers.

A MobileNet whose layer depths are not multiples of 32 runs them zero-padded to one (nets/mobilenet_v1.py, pad_depths): the
audit holds the pad channels to exactly 0 and audits the real channels against the unpadded checkpoint."""

import numpy as np
import torch

import front_ref64 as FR
import net_ref64 as R
import roi_pool_oracle as RP
import stage_ref64 as S
from oracle import pipeline as P
from tf_faster_rcnn_b200 import synth

F = np.float32

ORACLE_KEYS = ("rpn_nms_thresh", "rpn_pre_nms_top_n", "rpn_post_nms_top_n", "rpn_top_n", "test_mode", "use_e2e_tf", "use_gpu_nms",
               "pooling_size", "resnet_max_pool", "bbox_stds", "bbox_means", "nms_thresh", "max_per_image")


def _set_cfg(cfg, updates):
    saved = {}
    for k, v in updates.items():
        node = cfg
        *parents, leaf = k.split(".")
        for p_ in parents:
            node = node[p_]
        saved[k] = node[leaf]
        node[leaf] = v
    return saved


def build(monkeypatch, net_name, C, scales, cfg_updates, impl, weights=None, anchor_ratios=(0.5, 1, 2), rpn_channels=None,
          depth_multiplier=None):
    """The network, its checkpoint tensors and the recorder of every tape step's outputs (label, outputs, conv plan).
    cfg_updates (dotted cfg keys) hold while the network is made; rpn_channels and depth_multiplier are the cfg keys
    RPN_CHANNELS and MOBILENET.DEPTH_MULTIPLIER.  The checkpoint is synth's for that architecture (RPN channels, depth
    multiplier, anchors, POOLING_SIZE)."""
    from model.config import cfg
    from nets.vgg16 import vgg16
    from nets.resnet_v1 import resnetv1
    from nets.mobilenet_v1 import mobilenetv1
    from tf_faster_rcnn_b200 import engine
    if impl is not None:
        monkeypatch.setenv("FRCNN_CONV_IMPL", impl)
    updates = dict(cfg_updates)
    if rpn_channels is not None:
        updates["RPN_CHANNELS"] = rpn_channels
    if depth_multiplier is not None:
        updates["MOBILENET.DEPTH_MULTIPLIER"] = depth_multiplier
    saved = _set_cfg(cfg, updates)
    try:
        cfg.TEST.HAS_RPN = True
        net = vgg16() if net_name == "vgg16" else mobilenetv1() if net_name == "mobile" else resnetv1(num_layers=int(net_name[3:]))
        net.create_architecture("TEST", C, tag="default", anchor_scales=scales, anchor_ratios=anchor_ratios)
        arch = dict(rpn_channels=int(cfg.RPN_CHANNELS), depth_multiplier=float(cfg.MOBILENET.DEPTH_MULTIPLIER),
                    pooling_size=int(cfg.POOLING_SIZE))
    finally:
        _set_cfg(cfg, saved)
    w = synth.make(net_name, C, net.num_anchors, **arch)
    net.load_weights(weights(w) if weights else w)
    rec = []

    def wrap(name):
        orig = getattr(engine.Tape, name)

        def f(self, *a, **k):
            n = len(self.conv_plans)
            out = orig(self, *a, **k)
            plan = self.conv_plans[-1] if len(self.conv_plans) > n else None
            rec.append((self.steps[-1][0], out, plan))
            return out
        monkeypatch.setattr(engine.Tape, name, f)
    for name in ("conv", "conv_first", "depthwise", "max_pool", "spatial_mean"):
        wrap(name)
    return net, w, rec


def step_outputs(plan, rec):
    """[(label, {name: tensor}, conv plan)] for every step of the detect launch, in launch order."""
    it = iter(rec)
    multi = {"rpn_decode": ("rpn_scores", "rpn_props"), "sort_desc": ("order", "sorted_scores"),
             "proposals": ("rois", "roi_scores", "roi_keep", "num_rois"), "crop_pool": ("pool5",), "roi_align": ("pool5",),
             "roi_pool": ("pool5",), "cls_finish": ("cls_score", "cls_prob", "bbox_pred"), "bbox_decode": ("pred_boxes",)}
    out = []
    for label, _ in plan.tape.steps[:plan.n_im_detect_steps]:
        if label in multi:
            out.append((label, {k: getattr(plan, k) for k in multi[label]}, None))
        else:
            lab, t, cp = next(it)
            assert lab == label, (lab, label)
            out.append((label, {"out": t}, cp))
    out.append(("detect_post", {"rec": plan.rec, "keep": plan.keep, "keep_cnt": plan.keep_cnt, "keep_score": plan.keep_score,
                                "post_ws": plan.post_ws}, None))
    return out


class Tail:
    """References of the index work of the detection tail, bit for bit (softmaxes within stage_ref64's bounds)."""

    def __init__(self, plan, o, B, hw, meta):
        self.plan, self.o, self.B, self.hw, self.meta = plan, o, B, hw, meta
        self.R = plan.R

    def valid(self, bufs):
        n = bufs["proposals"]["num_rois"]
        return np.concatenate([np.arange(b * self.R, b * self.R + n[b]) for b in range(self.B)])

    def __call__(self, lay, bufs):
        B, o, plan, nR = self.B, self.o, self.plan, self.R
        g = bufs[lay.key]
        if lay.kind == "rpn_decode":
            heads = bufs[lay.ins[0]]
            A, dcol = lay.p["A"], lay.p["dcol"]
            nan = heads.shape[1] * heads.shape[2] * A
            worst = 0.0
            for b in range(B):
                cls, box = heads[b:b + 1, :, :, :2 * A], heads[b:b + 1, :, :, dcol:dcol + 4 * A]
                _, props, _ = P.rpn_decode(cls, box, np.array([self.hw[0], self.hw[1], 1.0], F), o)
                R._exact(lay.label, g["rpn_props"][b * nan:(b + 1) * nan], props, "proposal boxes, image %d" % b)
                p64, bound = S.rpn_fg_ref(cls[0, :, :, :A].reshape(-1), cls[0, :, :, A:].reshape(-1))
                r, _ = R._check(lay.label, g["rpn_scores"][b * nan:(b + 1) * nan], p64, bound, lambda i: "image %d anchor %d" % (b, i[0]))
                worst = max(worst, r)
            return worst, "fg scores", 0
        if lay.kind == "sort_desc":
            sc = bufs["rpn_decode"]["rpn_scores"].reshape(B, -1)
            for b in range(B):
                order, keys = FR.sort_ref(sc[b])
                R._exact(lay.label, g["order"].reshape(B, -1)[b], order, "order, image %d" % b)
                R._exact(lay.label, g["sorted_scores"].reshape(B, -1)[b], keys, "keys, image %d" % b)
            return 0.0, "", 0
        if lay.kind == "proposals":
            d = bufs["rpn_decode"]
            sc, props = d["rpn_scores"].reshape(B, -1), d["rpn_props"].reshape(B, -1, 4)
            for b in range(B):
                rois, scores, keep = P.proposals(sc[b], props[b], o)
                k = rois.shape[0]
                assert g["num_rois"][b] == k, "%s: image %d has %d RoIs, want %d" % (lay.label, b, g["num_rois"][b], k)
                rows = slice(b * nR, b * nR + k)
                R._exact(lay.label, g["rois"][rows, 1:], rois[:, 1:], "boxes, image %d" % b)
                R._exact(lay.label, g["rois"][rows, 0], np.full(k, b, F), "image index, image %d" % b)
                R._exact(lay.label, g["roi_keep"][rows], keep.astype(np.int32), "keep, image %d" % b)
                R._exact(lay.label, g["roi_scores"][rows], scores.reshape(-1), "scores, image %d" % b)
            return 0.0, "", 0
        if lay.kind == "pool":
            feat, rois = bufs[lay.ins[0]], bufs["proposals"]["rois"]
            v = self.valid(bufs)
            if lay.p["mode"] == "align":
                sr, aligned = self.plan.net.options["roi_align"]
                want = RP.roi_align_model(feat, rois[v], o["pooling_size"], sr, aligned)
            elif lay.p["mode"] == "pool":
                want = RP.roi_pool_model(feat, rois[v], o["pooling_size"])
            else:
                want = np.zeros((len(v),) + g.shape[1:], F)
                for b in range(B):
                    sel = rois[v, 0] == b
                    net = "res" if not lay.p["pre_pool"] else "vgg16"
                    want[sel] = P.crop_pool(net, feat[b:b + 1], rois[v][sel], o)
            return R._exact(lay.label, g[v], want, "pooled RoIs") + (0,)
        if lay.kind == "cls_finish":
            C = lay.p["C"]
            v = self.valid(bufs)
            head = bufs[lay.ins[0]].reshape(B * nR, -1)[v]
            R._exact(lay.label, g["cls_score"][v], head[:, :C], "cls_score")
            R._exact(lay.label, g["bbox_pred"][v], S.denorm_ref(head[:, C:5 * C], o["bbox_stds"], o["bbox_means"]), "bbox_pred")
            p64, bound = S.softmax_ref(head[:, :C], S.cls_depth(C))
            return R._check(lay.label, g["cls_prob"][v], p64, bound, lambda i: "(RoI, class) = (%d, %d)" % (v[i[0]], i[1])) + (0,)
        if lay.kind == "bbox_decode":
            f = bufs["cls_finish"]
            rois = bufs["proposals"]["rois"]
            for b in range(B):
                v = np.arange(b * nR, b * nR + bufs["proposals"]["num_rois"][b])
                s, oh, ow = self.meta[b]
                _, pred = P.im_detect_post(rois[v], f["cls_prob"][v], f["bbox_pred"][v], s, oh, ow)
                try:
                    S.check_boxes_exact(g[v], pred, "%s image %d" % (lay.label, b))
                except AssertionError as e:
                    raise R.Finding(str(e))
            return 0.0, "", 0
        if lay.kind == "detect_post":
            f, pb = bufs["cls_finish"], bufs["bbox_decode"]
            rec = g["rec"]
            md = plan.max_det
            for b in range(B):
                v = np.arange(b * nR, b * nR + bufs["proposals"]["num_rois"][b])
                want = P.test_net_post(f["cls_prob"][v], pb[v], o, thresh=float(plan.net.options["score_thresh"]))
                nd = int(rec[b].view(np.int32)[0])
                det = rec[b, 8:8 + md * 6].reshape(md, 6)
                try:
                    S.check_records(det, nd, None, want, md, "%s image %d" % (lay.label, b))
                except AssertionError as e:
                    raise R.Finding(str(e))
            return 0.0, "", 0
        raise KeyError(lay.kind)


def host(outs):
    v = {k: t.cpu().numpy() for k, t in outs.items()}
    return next(iter(v.values())) if len(v) == 1 else v


def depth(lay, w):
    """The checkpoint's output depth of a layer the device may run zero-padded (SIMT convs, unfused tensor-core convs), else
    None."""
    if lay.kind == "depthwise":
        return int(w[lay.key + "/depthwise_weights"].shape[2])
    if lay.kind == "conv_first":
        return int(w[lay.key + "/weights"].shape[-1])
    if lay.kind == "conv" and "fused" not in lay.p and not lay.p["fc"]:
        return int(w[lay.p["parts"][0] + "/weights"].shape[-1])
    return None


def real_channels(lay, w, v):
    """The device output v of layer lay cut to the checkpoint's depth; the pad channels must hold exactly +0."""
    d = depth(lay, w)
    if d is None or v.shape[-1] == d:
        return v
    pad = v[..., d:]
    if pad.view(np.uint32).any():
        i = np.unravel_index(np.argmax(pad.view(np.uint32) != 0), pad.shape)
        raise R.Finding("%s: pad channel %d holds %r at %s, want +0" % (lay.label, d + i[-1], pad[i], i[:-1]))
    return np.ascontiguousarray(v[..., :d])


def poison(tensors):
    for t in tensors:
        t.view(torch.uint8).fill_(0xff)


def run_audit(net_name, C, scales, hw, B, net, w, rec, mode, label, corrupt=None):
    """Poisoned replay, audit every layer, re-run eagerly and compare.  corrupt(walk, steps): called after the replay (the
    teeth tests)."""
    warm = np.concatenate([synth.synthetic_blob(hw[0], hw[1], seed) for seed in range(100, 100 + B)], axis=0)
    blobs = np.concatenate([synth.synthetic_blob(hw[0], hw[1], seed) for seed in range(3, 3 + B)], axis=0)
    meta = [(1.0, hw[0], hw[1])] * B
    _, plan = net.detect_batch(warm, [1.0] * B, [hw] * B)           # eager warm-up, capture, one replay, on other images
    graphs = dict(plan.graphs)
    assert ("detect", 0) in graphs and not plan.double_buffer
    poison([b for b in plan.tape.bufs if b is not plan.post_ws] + list(plan.recs))
    torch.cuda.synchronize()
    _, plan2 = net.detect_batch(blobs, [1.0] * B, [hw] * B)         # the audited run: the cached graph, replayed once
    torch.cuda.synchronize()
    assert plan2 is plan and plan.graphs == graphs, "the audited call did not replay the cached graph"
    steps = step_outputs(plan, rec)
    o = P.opts(anchor_scales=scales, anchor_ratios=net._anchor_ratios, **{k: plan.net.options[k] for k in ORACLE_KEYS})
    walk = R.walk(net_name, net.num_anchors, C, plan.net.options["pooling_mode"], o["resnet_max_pool"])
    assert [s[0] for s in steps] == [l.label for l in walk], "the tape's steps differ from the walk"
    if corrupt is not None:
        corrupt(walk, steps)
    snap = [{k: t.clone() for k, t in outs.items()} for _, outs, _ in steps]
    # ---- the audit: each layer on the device outputs of its inputs, a buffer fetched when first needed, dropped after its last use
    index = {l.key: i for i, l in enumerate(walk)}
    last = {}
    for i, l in enumerate(walk):
        for k in l.ins:
            last[k] = i
    bufs = {"image": blobs}
    tail = Tail(plan, o, B, hw, meta)
    rows = []
    for i, lay in enumerate(walk):
        for k in lay.ins + (lay.key,):
            if k not in bufs:
                bufs[k] = real_channels(walk[index[k]], w, host(steps[index[k]][1]))
        if index.get("proposals", i) < i and "proposals" not in bufs:      # the tail's RoI counts
            bufs["proposals"] = host(steps[index["proposals"]][1])
        pl = {}
        cp = steps[i][2]
        if cp is not None:
            info = cp.info()
            per_roi = None
            if index.get("pool5", i) < i:
                # per-RoI layer: RoIs per image, RoIs per M tile (an FC layer's rows are RoIs, tiled along w; a map layer
                # tiles tile_n RoIs), the RoI count of every image
                per_roi = (plan.R, info["tile_w"] if lay.p["fc"] else info["tile_n"], bufs["proposals"]["num_rois"])
            pl = dict(tile=(info["tile_h"], info["tile_w"]), per_roi=per_roi)
        rows += R.audit([lay], w, bufs, mode, {lay.key: pl}, seed=i, tail=tail)
        for k in list(bufs):                              # the tail's multi-output steps stay
            if k != "image" and isinstance(bufs[k], np.ndarray) and last.get(k, -1) <= i:
                del bufs[k]
    worst = R.worst_by_kind(rows)
    print("\n[%s] %d steps audited, F16X3 inputs below 2^-14 sampled: %d" % (label, len(rows), sum(r.tiny for r in rows)))
    for k, r in sorted(worst.items()):
        print("  %-28s worst err/bound %.3f  %s %s" % (k, r.ratio, r.label, r.at))
    # ---- eager re-run, one step at a time, its outputs poisoned first: bit-equal to the replay, and no stray stores
    bufs_all = list(plan.tape.bufs)
    for i, (label, outs, _) in enumerate(steps):
        fn = plan.tape.steps[i][1] if i < plan.n_im_detect_steps else plan.post_steps[plan.slot]
        mine = {t.data_ptr() for t in outs.values()}
        poison([t for k, t in outs.items() if k != "post_ws"])
        before = [b.clone() for b in bufs_all]
        fn()
        torch.cuda.synchronize()
        for b, c in zip(bufs_all, before):
            if b.data_ptr() not in mine:
                assert torch.equal(b.view(torch.uint8), c.view(torch.uint8)), "%s changed a buffer it does not own %s" % (label, tuple(b.shape))
        del before
        for k, t in outs.items():
            if k != "post_ws":
                assert torch.equal(t.contiguous().view(torch.uint8), snap[i][k].contiguous().view(torch.uint8)), \
                    "%s: eager %s differs from the graph replay" % (label, k)
    return rows
