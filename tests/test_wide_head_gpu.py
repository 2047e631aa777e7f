"""The detection head of detectors past 1024 classes on the GPU, held to float64 (or to its exact model) where it is computed,
not only where its outputs reach the post:

* the fused cls_score | bbox_pred FC (engine.py, fused_cls: ld_head = ceil(5C/4)*4 columns) through the conv kernel, per
  element in all three arithmetic modes, with test_conv_gpu.py's criteria: (a) against the split model in every mode, (b)
  against float64 in F16X3 and TF32X3; synth-like weights (std 0.02 class columns, 0.01 box columns, one matrix), the bias as
  the epilogue's shift, the pad columns exactly 0.  Each case asserts the decomposition it exists for (test_wide_head.py's
  HEAD_CASES: 48 to 160 N tiles, ragged-round splits 2 and 8 ways, a forced 3-way split with a short last split, block_n 64,
  last N tiles 4 / 8 / 72 / 128 columns wide, 5000 rows); guard bands, unchanged inputs, two runs bit-equal; the raster orders
  bit-equal with no tile and with every tile split, and on every tile the ragged split treats alike in both orders;
* cls_finish at 1025 to 4096 classes (test_stage_edges_gpu's edge body: every logit row kind, NaN in the pad columns) and
  bbox_decode at 1025 to 4096 classes with three images, and at 5000 RoIs x 4096 classes;
* the detect graph audited step by step (graph_audit's run_audit, unchanged) at 1204 to 4096 classes, with teeth: one
  element of the head's last N tile moved by 1e-3 relative, and two cls_score columns swapped in the engine's weights, each
  fail at the cls_bbox layer;
* Soft-NMS, box voting and the flip augmentation of a 1601-class ResNet-101 against the oracles' post of its own outputs.

Observed on an H100 80 GB HBM3 (SXM, 700 W limit), max over elements of err / (u S) for the head FC: (a) F16X3 1.09, TF32X3
1.33, F16X1 0.55; (b) F16X3 1.12, TF32X3 1.34 (both on the 160-N-tile head); F16X1 misses (b) by 629 .. 1255 x.  cls_prob
err / bound <= 0.40.  The audits' worst err / bound over all steps: ResNet-101 1601 classes batch 2 0.40, 4096 classes 0.40,
VGG16 0.35, MobileNet-v1 1204 classes 0.77 (a head depthwise conv, as at 81 classes), ResNet-50 TF32X3 0.34, F16X1 0.34, 1000
RoIs 0.35; the cls_bbox layer itself <= 0.17.  The teeth fail at 268 x and 1.3e5 x their bound.  The raster orders differ on
the 28 of 1600 tiles the ragged split treats differently.  The module runs in 4 to 6 minutes, mostly its CPU references."""
import os
import sys
import zlib

import cv2
import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import aug_oracle as AO  # noqa: E402
import box_vote_oracle as BV  # noqa: E402
import conv_split_model as M  # noqa: E402
import net_ref64 as R  # noqa: E402
import soft_nms_oracle as SO  # noqa: E402
import stage_ref64 as S  # noqa: E402
from oracle import pipeline as P  # noqa: E402
from test_conv_gpu import ALPHA, BETA, conv_run, epilogue64, ratio, reference  # noqa: E402
from graph_audit import build as audit_build, run_audit  # noqa: E402
from test_regions_gpu import _release_networks, build as net_build  # noqa: E402,F401
from test_soft_nms_gpu import own_outputs, records_from  # noqa: E402
from test_stage_edges_gpu import check_decode_per_image, decode_rois, run_bbox_decode  # noqa: E402
from test_stage_edges_gpu import test_cls_finish_edges as cls_finish_edges  # noqa: E402
from test_wide_head import HEAD_CASES, ld_head  # noqa: E402
from tf_faster_rcnn_b200 import synth  # noqa: E402

pytestmark = pytest.mark.gpu
F = np.float32
MODES = ["f16x3", "tf32x3", "f16x1"]


def _release_plans(net):
    for plan in net._plans.values():
        plan.release()
    net._plans.clear()
    net._aug_plans.clear()


@pytest.fixture(scope="module", autouse=True)
def _room_for_wide_plans(cuda):
    """The audits' 600x800 plans at 1601 / 4096 classes, with their eager re-run's copy of every tape buffer, need most of the
    device.  Networks that modules run earlier in the same process keep their shape plans (graphs, activation buffers) while
    anything references them -- a module-level cache, or the network registry -- so those plans are released first: a network
    whose plans were released re-creates a plan when it is next used."""
    import gc
    from nets import network
    gc.collect()
    before = torch.cuda.memory_allocated()
    nets = [o for o in gc.get_objects() if issubclass(type(o), network.Network)]
    for net in nets:
        _release_plans(net)
    gc.collect()
    torch.cuda.empty_cache()
    print("\n[wide head] plans of %d earlier networks released: %.2f -> %.2f GB allocated" %
          (len(nets), before / 2 ** 30, torch.cuda.memory_allocated() / 2 ** 30))
    yield


GEOM = ("block_n", "m_tiles", "n_tiles", "tiles", "split_tiles", "splits", "kb_per_split", "k_blocks", "units", "grid")


# ---- the fused cls_score | bbox_pred FC, per element ---------------------------------------------------------------------------
_DATA = {}


def head_data(C, K, rows):
    """fc7-like activations [1, 1, rows, K] (|N(0, 1)|) and the fused head of C classes as engine.fused_cls lays it out: class
    columns N(0, 0.02^2), box columns N(0, 0.01^2), zero pad columns; biases N(0, 0.5^2) / N(0, 0.01^2) / 0 (synth.py's
    head).  One data set at a time is kept, with its split models."""
    key = (C, K, rows)
    if key not in _DATA:
        _DATA.clear()
        rng = np.random.default_rng(zlib.crc32(("head_%d_%d_%d" % key).encode()))
        ld = ld_head(C)
        x = np.abs(rng.standard_normal((1, 1, rows, K))).astype(F)
        w = np.zeros((1, 1, K, ld), F)
        w[0, 0, :, :C] = rng.standard_normal((K, C)) * 0.02
        w[0, 0, :, C:5 * C] = rng.standard_normal((K, 4 * C)) * 0.01
        b = np.zeros(ld, F)
        b[:C] = rng.standard_normal(C) * 0.5
        b[C:5 * C] = rng.standard_normal(4 * C) * 0.01
        _DATA[key] = dict(x=x, w=w, b=b, model={})
    return _DATA[key]


def fc_model(d, rows, impl):
    """conv_split_model's model of a 1x1 layer as one matrix product: the device's operand roundings, float64 sums."""
    if impl not in d["model"]:
        x = d["x"][0, 0] if rows is None else d["x"][0, 0][rows]
        xh, xl = M.split_activations(x, impl)
        wh, wl = M.split_weights(d["w"][0, 0], impl)
        m = xh @ wh
        if impl != M.F16X1:
            m += xl @ wh + xh @ wl
        d["model"][impl] = m
    return d["model"][impl]


def sampled_rows(g, rows, rng, n_random=256):
    """Rows of a tall head checked against float64: the first and last row of every M tile, every row of the M tile that holds
    the first split tile (the seam between whole and split tiles, under either raster order) and the one before it, and
    `n_random` random rows."""
    tw = g["tile_w"]
    out = {r for t in range(0, rows, tw) for r in (t, min(t + tw, rows) - 1)}
    if g["split_tiles"]:
        t0 = g["tiles"] - g["split_tiles"]                    # the split tiles are the last tile indices
        for mt in (t0 % g["m_tiles"], t0 // g["n_tiles"]):     # raster m, raster n
            for m in (mt - 1, mt):
                out.update(range(max(m, 0) * tw, min((m + 1) * tw, rows)))
    out.update(int(r) for r in rng.choice(rows, n_random, replace=False))
    return np.array(sorted(out), np.int64)


@pytest.mark.parametrize("case", HEAD_CASES, ids=[c[0] for c in HEAD_CASES])
def test_head_fc_per_element(cuda, case):
    name, C, K, rows, opt, covers = case
    d = head_data(C, K, rows)
    ld = ld_head(C)
    sel = None
    for mode in MODES:
        impl = M.MODES[mode]
        (got, got2), info, g, _ = conv_run(d["x"], d["w"], impl, shift=d["b"], block_n=opt.get("block_n", 0),
                                            split_k=opt.get("split_k", 0), runs=2)
        assert covers(g), "%s no longer covers its path: %s" % (name, g)
        assert np.array_equal(got.view(np.int32), got2.view(np.int32)), "two runs differ"
        assert np.isfinite(got).all(), "non-finite output (unwritten rows?) %s" % g
        got = got[0, 0]
        assert not got[:, 5 * C:].any(), "pad columns not 0"
        if rows > 1200 and sel is None:
            sel = sampled_rows(g, rows, np.random.default_rng(rows))
        xs = d["x"] if sel is None else d["x"][:, :, sel]
        n = xs.shape[2]
        want64, s = reference("head_%d_%d_%d" % (C, K, rows), xs, d["w"], 1, 0, 0, 1, n)
        want64, s = want64[0, 0], s[0, 0]
        g_rows = got if sel is None else got[sel]
        y_m, sc, rnd_m = epilogue64(fc_model(d, sel, impl), None, d["b"], None, 0)
        y_r, _, rnd_r = epilogue64(want64, None, d["b"], None, 0)
        ra = ratio(g_rows, y_m, s, sc, rnd_m)
        rb = ratio(g_rows, y_r, s, sc, rnd_r)
        line = "[%s %s] cout=%d rows=%d checked=%d a=%.2f b=%.2f" % (name, mode, ld, rows, n, ra, rb)
        print("\n" + line + " last_n_tile=%d geom=%s" % (ld - (g["n_tiles"] - 1) * g["block_n"], {k: g[k] for k in GEOM}))
        assert ra <= BETA, line
        if mode != "f16x1":
            assert rb <= ALPHA, line


def split_tiles_of(g, raster_n):
    """[m_tiles, n_tiles] bool: the tiles of the split (the last split_tiles tile indices) under raster n or m."""
    mt, nb = np.meshgrid(np.arange(g["m_tiles"]), np.arange(g["n_tiles"]), indexing="ij")
    idx = mt * g["n_tiles"] + nb if raster_n else nb * g["m_tiles"] + mt
    return idx >= g["tiles"] - g["split_tiles"]


@pytest.mark.parametrize("mode", MODES)
def test_head_fc_raster_order(cuda, mode, monkeypatch):
    """FRCNN_CONV_RASTER m and n on the 160-N-tile head (4096 classes, batch 4).  With no tile split (split_k 1) and with every
    tile split (split_k 3) the two orders give the same bits.  The ragged-round split takes the last tile indices, so there the
    raster decides which 16 tiles are split: every tile split in both orders or in neither is bit-equal, the tiles split in one
    order only differ, and the raster-n output meets criteria (a) and (b) on its own."""
    name, C, K, rows, _, covers = [c for c in HEAD_CASES if c[0] == "b4_4096"][0]
    d = head_data(C, K, rows)
    impl = M.MODES[mode]
    for split_k in (1, 3, 0):
        outs = {}
        for r in ("m", "n"):
            monkeypatch.setenv("FRCNN_CONV_RASTER", r)
            (o,), _, g, _ = conv_run(d["x"], d["w"], impl, shift=d["b"], split_k=split_k)
            outs[r] = o[0, 0]
        monkeypatch.delenv("FRCNN_CONV_RASTER")
        same = outs["m"].view(np.int32) == outs["n"].view(np.int32)
        if split_k:
            assert g["n_tiles"] == 160 and g["split_tiles"] == (0 if split_k == 1 else g["tiles"]), g
            assert same.all(), "split_k %d: raster m and n differ" % split_k
            continue
        assert covers(g), g
        moved_tiles = split_tiles_of(g, False) != split_tiles_of(g, True)
        moved = np.repeat(np.repeat(moved_tiles, g["tile_w"], 0), g["block_n"], 1)[:rows, :outs["m"].shape[1]]
        assert moved.any() and same[~moved].all(), "raster m and n differ on a tile split in both orders or in neither"
        want64, s = reference("head_%d_%d_%d" % (C, K, rows), d["x"], d["w"], 1, 0, 0, 1, rows)
        y_m, sc, rnd_m = epilogue64(fc_model(d, None, impl), None, d["b"], None, 0)
        y_r, _, rnd_r = epilogue64(want64[0, 0], None, d["b"], None, 0)
        ra, rb = ratio(outs["n"], y_m, s[0, 0], sc, rnd_m), ratio(outs["n"], y_r, s[0, 0], sc, rnd_r)
        print("\n[raster %s] ragged split: %d of %d tiles split in one order only, %d elements differ; raster n a=%.2f b=%.2f"
              % (mode, int(moved_tiles.sum()), g["tiles"], int((~same).sum()), ra, rb))
        assert ra <= BETA
        if mode != "f16x1":
            assert rb <= ALPHA


# ---- cls_finish and bbox_decode past 1024 classes ------------------------------------------------------------------------------
@pytest.mark.parametrize("r", [1, 7, 300, 1001])
@pytest.mark.parametrize("C", [1025, 1204, 1601, 2048, 4095, 4096])
def test_cls_finish_many_classes(cuda, C, r):
    """test_stage_edges_gpu.test_cls_finish_edges' body: production ld with NaN pad columns, the six logit row kinds;
    cls_score and bbox_pred value for value, cls_prob within softmax_ref(x, cls_depth(C)) (ceil(C/32) terms per lane)."""
    cls_finish_edges(cuda, C, r)


META3 = [(1.6, 375, 500), (600 / 720, 720, 960), (2.4, 250, 333)]


@pytest.mark.parametrize("C,R", [(1025, 301), (1601, 301), (4096, 301), (4096, 5000)])
def test_bbox_decode_many_classes(cuda, C, R):
    """Three images with three im_meta rows, RoI rows interleaved, edge deltas; each image against the oracle value for value
    and the one-sided clip reached.  R * C is off a multiple of the 256-thread block unless C is a multiple of 256."""
    if C % 256:
        assert (R * C) % 256
    rng = np.random.default_rng(C + R)
    rois = decode_rois(rng, R, 3)
    assert len(set(rois[:, 0].tolist())) == 3
    deltas = S.edge_deltas(rng, R, C)
    check_decode_per_image(run_bbox_decode(rois, deltas, C, META3), rois, deltas, C, META3)


# ---- graph audits at many classes ----------------------------------------------------------------------------------------------
def _free(net, rec):
    """Release a network's plans and the recorded step outputs now (test_regions_gpu._release_networks releases every network
    of this module at its end)."""
    rec.clear()
    _release_plans(net)
    torch.cuda.empty_cache()


# (id, net, classes, anchor scales, blob H x W, batch, cfg updates, FRCNN_CONV_IMPL)
AUDITS = [
    ("res101_1601_b2", "res101", 1601, (4, 8, 16, 32), (600, 800), 2, {}, None),
    ("res101_4096", "res101", 4096, (4, 8, 16, 32), (600, 800), 1, {}, None),
    ("vgg16_1601", "vgg16", 1601, (8, 16, 32), (600, 800), 1, {}, None),
    ("mobile_1204", "mobile", 1204, (4, 8, 16, 32), (600, 800), 1, {}, None),
    ("res50_1601_tf32", "res50", 1601, (8, 16, 32), (600, 800), 1, {}, "tf32"),
    ("res50_1601_f16x1", "res50", 1601, (8, 16, 32), (600, 800), 1, {}, "f16x1"),
    ("res50_1601_1000", "res50", 1601, (8, 16, 32), (600, 800), 1, {"TEST.RPN_POST_NMS_TOP_N": 1000}, None),
]


def head_info(rec):
    cps = [cp for label, _, cp in rec if label.endswith("/cls_bbox")]
    return cps[-1].info()


@pytest.mark.parametrize("cid,net_name,C,scales,hw,B,cfg_updates,impl", AUDITS, ids=[c[0] for c in AUDITS])
def test_graph_audit_many_classes(cuda, monkeypatch, cid, net_name, C, scales, hw, B, cfg_updates, impl):
    net, w, rec = audit_build(monkeypatch, net_name, C, scales, cfg_updates, impl)
    try:
        mode = M.MODES[{"tf32": "tf32x3", "f16x1": "f16x1"}.get(impl, "f16x3")]
        rows = run_audit(net_name, C, scales, hw, B, net, w, rec, mode, cid)
        info = head_info(rec)
        worst = max(r.ratio for r in rows)
        print("  head cls_bbox: cout %d, block_n %d, grid %dx%d, splits %d; worst err/bound over all steps %.3f"
              % (ld_head(C), info["block_n"], info["grid_m"], info["grid_n"], info["splits"], worst))
        assert worst <= 1
    finally:
        _free(net, rec)


TEETH = ("res50", 1601, (8, 16, 32), (304, 400))
HEAD_LAYER = "resnet_v1_50/cls_bbox"


def test_audit_names_a_corrupted_head_element(cuda, monkeypatch):
    """One element of RoI 0 in the head's last N tile (a box column >= 62 * 128) moved by 1e-3 relative after the replay: the
    audit fails at the cls_bbox layer."""
    net_name, C, scales, hw = TEETH
    net, w, rec = audit_build(monkeypatch, net_name, C, scales, {}, None)
    ld = ld_head(C)

    def corrupt(walk, steps):
        i = [l.key for l in walk].index(HEAD_LAYER)
        flat = steps[i][1]["out"].view(-1)
        lo = 62 * 128                                          # the first column of the last of 63 N tiles
        assert C <= lo < 5 * C <= ld
        j = lo + int(torch.argmax(flat[lo:5 * C].abs()))       # RoI 0 is row 0 of the head
        flat[j] *= 1 + 1e-3
    try:
        with pytest.raises(R.Finding) as e:
            run_audit(net_name, C, scales, hw, 1, net, w, rec, M.F16X3, "corrupted head", corrupt)
        print("\n" + str(e.value))
        assert str(e.value).startswith("conv:" + HEAD_LAYER + ":"), str(e.value)
    finally:
        _free(net, rec)


def test_audit_names_swapped_class_columns(cuda, monkeypatch):
    """cls_score columns 5 and 1500 swapped in the engine's weights only, the reference keeps the true tensors: the audit fails
    at the cls_bbox layer."""
    net_name, C, scales, hw = TEETH
    key = "resnet_v1_50/cls_score/weights"

    def swapped(w):
        w2 = dict(w)
        a = np.array(w[key], copy=True)
        a[..., [5, 1500]] = a[..., [1500, 5]]
        w2[key] = a
        return w2
    net, w, rec = audit_build(monkeypatch, net_name, C, scales, {}, None, weights=swapped)
    try:
        with pytest.raises(R.Finding) as e:
            run_audit(net_name, C, scales, hw, 1, net, w, rec, M.F16X3, "swapped columns")
        print("\n" + str(e.value))
        assert str(e.value).startswith("conv:" + HEAD_LAYER + ":"), str(e.value)
    finally:
        _free(net, rec)


# ---- post extensions at network level, 1601 classes ----------------------------------------------------------------------------
@pytest.fixture(scope="module")
def net1601():
    """The bottom-up-attention layout (ResNet-101, 1601 classes, 12 anchors), built once for this module."""
    return net_build("res101", 1601, (4, 8, 16, 32))


@pytest.fixture
def post_cfg(net1601):
    from model.config import cfg
    saved = (dict(cfg.TEST.SOFT_NMS), dict(cfg.TEST.BBOX_VOTE), dict(cfg.TEST.BBOX_AUG), tuple(cfg.TEST.SCALES), cfg.USE_GPU_NMS,
             net1601.options["use_gpu_nms"])
    yield cfg
    from model.test import _set_post_options
    cfg.TEST.SOFT_NMS.update(saved[0]); cfg.TEST.BBOX_VOTE.update(saved[1]); cfg.TEST.BBOX_AUG.update(saved[2])
    cfg.TEST.SCALES, cfg.USE_GPU_NMS = saved[3:5]
    net1601.options["use_gpu_nms"] = saved[5]
    _set_post_options(net1601, 0.0, 100)


HW = (600, 800)
SCALES2, ORIG2 = [1.0, 1.25], [(600, 800), (480, 640)]


def blobs2():
    return np.concatenate([synth.synthetic_blob(HW[0], HW[1], seed) for seed in (1, 2)], axis=0)


def check_detect_and_batch(net, want_of):
    """detect on image 0 and detect_batch on both images: every image's records == want_of(scores, boxes) of the plan's own
    cls_prob / pred_boxes rows."""
    blobs = blobs2()
    det, plan = net.detect(blobs[:1], np.array([HW[0], HW[1], 1.0], F), HW)
    scores, boxes = own_outputs(plan, 0)
    assert det.shape[0] >= 100 and det.tobytes() == records_from(want_of(scores, boxes)).tobytes()
    dets, plan2 = net.detect_batch(blobs, SCALES2, ORIG2)
    for b in range(2):
        scores, boxes = own_outputs(plan2, b)
        assert dets[b].shape[0] > 0 and dets[b].tobytes() == records_from(want_of(scores, boxes)).tobytes(), b
    return det.shape[0], [d.shape[0] for d in dets]


@pytest.mark.parametrize("method", ["linear", "gaussian"])
def test_soft_nms_1601_classes(cuda, net1601, post_cfg, method):
    from model.test import _set_post_options
    post_cfg.TEST.SOFT_NMS.update(ENABLED=True, METHOD=method)
    _set_post_options(net1601, 0.0, 100)
    soft, nt = net1601.options["soft_nms"], net1601.options["nms_thresh"]
    n = check_detect_and_batch(net1601, lambda s, x: SO.test_net_post_soft(s, x, soft, nt, 100)[0])
    print("\n[1601 classes soft-NMS %s] records detect %d, detect_batch %s" % (method, n[0], n[1]))


@pytest.mark.parametrize("soft_on,method", [(False, "AVG"), (True, "ID")])
def test_box_vote_1601_classes(cuda, net1601, post_cfg, soft_on, method):
    from model.test import _set_post_options
    post_cfg.TEST.SOFT_NMS.update(ENABLED=soft_on, METHOD="linear")
    post_cfg.TEST.BBOX_VOTE.update(ENABLED=True, SCORING_METHOD=method, VOTE_TH=0.7)
    _set_post_options(net1601, 0.0, 100)
    soft, vote, nt = net1601.options["soft_nms"], net1601.options["box_vote"], net1601.options["nms_thresh"]
    n = check_detect_and_batch(net1601, lambda s, x: BV.test_net_post_vote(s, x, vote, nt, 100, soft=soft)[0])
    print("\n[1601 classes %s + box voting %s] records detect %d, detect_batch %s" % ("soft-NMS" if soft_on else "greedy", method,
                                                                                    n[0], n[1]))


def test_tta_flip_1601_classes(cuda, net1601, post_cfg):
    """TEST.BBOX_AUG with H_FLIP at one scale: the records are the oracle's post of the union of the GPU's own per-view outputs."""
    from model.test import _run_aug, _set_post_options
    post_cfg.TEST.SCALES, post_cfg.USE_GPU_NMS = (288,), False
    post_cfg.TEST.BBOX_AUG.update(ENABLED=True, H_FLIP=True)
    net1601.options["use_gpu_nms"] = False
    _set_post_options(net1601, 0.0, 100)
    im = cv2.blur(np.random.default_rng(2).integers(0, 256, (240, 320, 3), dtype=np.uint8), (5, 5))
    aug = _run_aug(net1601, [im], detect=True)
    sc, bx = [], []
    for v, (h, wd, _) in enumerate(aug.views):
        p = aug.subs[(h, wd)]
        k = aug.view_slot[v] * aug.batch
        n, Rr = int(p.num_rois[k].item()), p.R
        sc.append(p.cls_prob[k * Rr:k * Rr + n].cpu().numpy()); bx.append(p.pred_boxes[k * Rr:k * Rr + n].cpu().numpy())
    assert [v[2] for v in aug.views] == [True, False]
    s, x = AO.union(sc, bx, [v[2] for v in aug.views], im.shape[1])
    want = records_from(AO.post(s, x, P.opts(use_gpu_nms=False, nms_thresh=post_cfg.TEST.NMS)))
    recs = aug.records()[0]
    print("\n[1601 classes flip TTA] union rows %d, records %d" % (s.shape[0], recs.shape[0]))
    assert recs.shape[0] > 0 and recs.tobytes() == want.tobytes()
