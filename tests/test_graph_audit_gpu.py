"""Every step of the detection graph at production shapes, each against float64 (or its exact model) on its own device inputs.

Per config: a first `detect` call on other images builds the plan (eager warm-up, graph capture, one replay); then every tape
buffer and record buffer except the post step's scratch workspace is filled with 0xff bytes (NaN as fp32, -1 as int32) and a
second call on the audited images is a pure replay of the cached graph.  The tape's step labels must match `net_ref64.walk`
one for one (so no step goes unaudited), and every step is audited (`net_ref64.audit`, fed the device outputs of the steps the
oracle says feed it).  Then the same steps run eagerly, one at a time with a synchronise between them, each step's declared
outputs poisoned the same way before it runs: each step's outputs equal the replay's bit for bit, and no step changes a tape
buffer it does not declare as its output.

What the ordering check covers: a step missing from the graph, or one that in this replay read a buffer before its producer
wrote it (a missing or misplaced PDL wait or stream dependency), reads poison or the wrong images' values instead of the
warm-up's, and fails its audit or the eager comparison.  It cannot prove a race absent: a premature read that happens to land
after the producer's store in this replay passes.

Observed on an H100 80 GB HBM3 (700 W limit), worst err / bound over all steps: ResNet-101 0.40 (batch 4: 0.40, align mode: 0.40),
VGG16 0.35, MobileNet-v1 0.77 (a head depthwise conv), ResNet-152 at 1000 RoIs 0.38, ResNet-50 TF32X3 0.34, F16X1 0.34 (against
its operand model); the module runs in about 4 minutes."""

import numpy as np
import pytest
import torch

import conv_split_model as M
import front_ref64 as FR
import net_ref64 as R
import roi_pool_oracle as RP
import stage_ref64 as S
from oracle import pipeline as P
from tf_faster_rcnn_b200 import synth

pytestmark = pytest.mark.gpu
F = np.float32

# (id, net, classes, anchor scales, blob H x W, batch, cfg updates, FRCNN_CONV_IMPL)
CONFIGS = [
    ("res101", "res101", 81, (4, 8, 16, 32), (600, 800), 1, {}, None),
    ("vgg16", "vgg16", 21, (8, 16, 32), (600, 800), 1, {}, None),
    ("mobile", "mobile", 81, (4, 8, 16, 32), (600, 800), 1, {}, None),
    ("res152_1000", "res152", 81, (2, 4, 8, 16, 32), (800, 1067), 1, {"TEST.RPN_POST_NMS_TOP_N": 1000}, None),
    ("res101_b4", "res101", 81, (4, 8, 16, 32), (600, 800), 4, {}, None),
    ("res101_align", "res101", 81, (4, 8, 16, 32), (600, 800), 1, {"POOLING_MODE": "align"}, None),
    ("res50_tf32", "res50", 21, (8, 16, 32), (600, 800), 1, {}, "tf32"),
    ("res50_f16x1", "res50", 21, (8, 16, 32), (600, 800), 1, {}, "f16x1"),
]
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


def build(monkeypatch, net_name, C, scales, cfg_updates, impl, weights=None):
    """The network, its checkpoint tensors and the recorder of every tape step's outputs (label, outputs, conv plan)."""
    from model.config import cfg
    from nets.vgg16 import vgg16
    from nets.resnet_v1 import resnetv1
    from nets.mobilenet_v1 import mobilenetv1
    from tf_faster_rcnn_b200 import engine
    if impl is not None:
        monkeypatch.setenv("FRCNN_CONV_IMPL", impl)
    saved = _set_cfg(cfg, cfg_updates)
    try:
        cfg.TEST.HAS_RPN = True
        net = vgg16() if net_name == "vgg16" else mobilenetv1() if net_name == "mobile" else resnetv1(num_layers=int(net_name[3:]))
        net.create_architecture("TEST", C, tag="default", anchor_scales=scales, anchor_ratios=(0.5, 1, 2))
    finally:
        _set_cfg(cfg, saved)
    w = synth.make(net_name, C, 3 * len(scales))
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
    o = P.opts(anchor_scales=scales, **{k: plan.net.options[k] for k in ORACLE_KEYS})
    walk = R.walk(net_name, 3 * len(scales), C, plan.net.options["pooling_mode"], o["resnet_max_pool"])
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
                bufs[k] = host(steps[index[k]][1])
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


@pytest.mark.parametrize("cid,net_name,C,scales,hw,B,cfg_updates,impl", CONFIGS, ids=[c[0] for c in CONFIGS])
def test_graph_audit(cuda, monkeypatch, cid, net_name, C, scales, hw, B, cfg_updates, impl):
    net, w, rec = build(monkeypatch, net_name, C, scales, cfg_updates, impl)
    mode = M.MODES[{"tf32": "tf32x3", "f16x1": "f16x1"}.get(impl, "f16x3")]
    rows = run_audit(net_name, C, scales, hw, B, net, w, rec, mode, cid)
    assert max(r.ratio for r in rows) <= 1


TEETH_LAYER = "resnet_v1_50/block2/unit_2/bottleneck_v1/conv2"


def test_audit_names_a_corrupted_buffer(cuda, monkeypatch):
    """One element of one intermediate buffer moved by 1e-3 relative after the replay: the audit fails at that layer.  The
    element lies on the map's top border, which the audit samples whole (an element it does not sample fails the next layer)."""
    net, w, rec = build(monkeypatch, "res50", 21, (8, 16, 32), {}, None)

    def corrupt(walk, steps):
        i = [l.key for l in walk].index(TEETH_LAYER)
        row = steps[i][1]["out"][0, 0]                       # [w, c]: image 0's first row
        j = int(torch.argmax(row.abs()))
        row.view(-1)[j] *= 1 + 1e-3
    with pytest.raises(R.Finding) as e:
        run_audit("res50", 21, (8, 16, 32), (304, 400), 1, net, w, rec, M.F16X3, "corrupted", corrupt)
    assert str(e.value).startswith("conv:" + TEETH_LAYER + ":"), str(e.value)


def test_audit_names_a_shifted_variance(cuda, monkeypatch):
    """The engine's weights move one layer's moving_variance by 1e-3 - 1e-5 (what an eps mix-up does), the reference keeps
    the true tensors: the audit fails at that layer."""
    key = TEETH_LAYER + "/BatchNorm/moving_variance"

    def shifted(w):
        w2 = dict(w)
        w2[key] = (w[key] + F(1e-3 - 1e-5)).astype(F)
        return w2
    net, w, rec = build(monkeypatch, "res50", 21, (8, 16, 32), {}, None, weights=shifted)
    with pytest.raises(R.Finding) as e:
        run_audit("res50", 21, (8, 16, 32), (304, 400), 1, net, w, rec, M.F16X3, "variance")
    assert str(e.value).startswith("conv:" + TEETH_LAYER + ":"), str(e.value)
