"""Bottom-up regions on the GPU (frcnn_detect_regions, Network.detect_regions, tools/extract_features.py --regions), exact against
the numpy oracle of tests/regions_oracle.py run on the same inputs: at stage level through ops on seeded inputs, at network
level on the plan's own device cls_prob / rois / num_rois / fc7."""
import base64
import csv
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import regions_oracle as RO  # noqa: E402
from tf_faster_rcnn_b200 import engine, ops, synth  # noqa: E402

pytestmark = pytest.mark.gpu
F = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = 64                                                   # guard elements on each side of every output / scratch buffer
SENTINEL = {torch.float32: 0x7fc0dead, torch.int32: -7777, torch.int64: -0x123456789}


@pytest.fixture(scope="module", autouse=True)
def _release_networks():
    """Networks register themselves process-wide, and a network and its plans reference each other, so dropping them from the
    registry alone frees nothing until a full garbage collection.  This module's plans (GBs of device memory at 600x800) are
    released and collected at its end, and the allocator's cache is returned to the driver: the library's own cudaMalloc
    calls (conv plan workspaces) in later modules cannot use torch's cached blocks."""
    import gc
    from nets import network
    before = list(network._REGISTRY)
    yield
    for net in network._REGISTRY:
        if not any(net is b for b in before):
            for plan in net._plans.values():
                plan.release()
            net._plans.clear()
            net._aug_plans.clear()
    network._REGISTRY[:] = before
    gc.collect()
    torch.cuda.empty_cache()


def make_batch(rng, B, R, C, nrois, spread=600.0, size=(20, 200), fdim=64):
    """cls_prob [B*R, C] (softmax rows, filled also past num_rois), rois [B*R, 5] (zeros past num_rois), fc7 [B*R, fdim]."""
    logits = rng.normal(0, 2, (B * R, C))
    p = np.exp(logits - logits.max(1, keepdims=True))
    probs = (p / p.sum(1, keepdims=True)).astype(F)
    xy = rng.uniform(0, spread, (B * R, 2))
    wh = rng.uniform(size[0], size[1], (B * R, 2))
    rois = np.hstack([np.repeat(np.arange(B), R)[:, None], xy, xy + wh]).astype(F)
    for b, n in enumerate(nrois):
        rois[b * R + n:(b + 1) * R] = 0
    fc7 = rng.normal(0, 1, (B * R, fdim)).astype(F)
    return probs, rois, fc7


def guarded(shape, dtype):
    """(integer view of the whole buffer with its guard bands, the [shape] dtype view between them)"""
    n = int(np.prod(shape))
    raw = torch.full((n + 2 * G,), SENTINEL[dtype], dtype=torch.int32 if dtype == torch.float32 else dtype, device="cuda")
    return raw, raw[G:G + n].view(dtype).view(*shape)


def run_stage(probs, rois, fc7, nrois, scales, nms, gpu_pred, conf, mn, mx):
    """frcnn_detect_regions through ops -> per image dicts (count rows); checks guards, padding rows and unchanged inputs."""
    B = len(nrois)
    R, C = probs.shape[0] // B, probs.shape[1]
    fdim = fc7.shape[1]
    ins = dict(cls_prob=torch.from_numpy(probs).cuda(), rois=torch.from_numpy(rois).cuda(),
               num_rois=torch.tensor(nrois, dtype=torch.int32).cuda(),
               im_meta=torch.tensor([[float(F(s)), 600.0, 800.0] for s in scales], dtype=torch.float32).cuda(),
               fc7=torch.from_numpy(fc7).cuda())
    before = {k: v.clone() for k, v in ins.items()}
    M = min(mx, R)
    bufs = dict(roi_box=guarded((B * R, C, 4), torch.float32), key=guarded((B * R,), torch.int64),
                boxes=guarded((B, M, 4), torch.float32), features=guarded((B, M, fdim), torch.float32),
                conf=guarded((B, M), torch.float32), classes=guarded((B, M), torch.int32), roi_index=guarded((B, M), torch.int32),
                count=guarded((B,), torch.int32))
    guards = {k: (b[:G].clone(), b[-G:].clone()) for k, (b, _) in bufs.items()}
    keep = torch.empty((B, C, R), dtype=torch.int32, device="cuda")
    keep_cnt = torch.empty((B, C), dtype=torch.int32, device="cuda")
    keep_score = torch.empty((B, C, R), dtype=torch.float32, device="cuda")
    ws = ops.detect_post_workspace(R, C, B)
    thr, flags = engine.nms_threshold(nms, gpu_pred)
    t32, mn, mx = engine.region_args(conf, mn, mx)
    out = {k: v for k, (_, v) in bufs.items() if k not in ("roi_box", "key")}
    ops.detect_regions(ins["cls_prob"], ins["rois"], ins["num_rois"], ins["im_meta"], ins["fc7"], C, thr, flags, t32, mn, mx, keep,
                       keep_cnt, keep_score, ws, bufs["roi_box"][1], bufs["key"][1], out, batch=B)
    torch.cuda.synchronize()
    for k, (b, _) in bufs.items():
        assert torch.equal(b[:G], guards[k][0]) and torch.equal(b[-G:], guards[k][1]), "guard band of %s overwritten" % k
    for k in ins:
        assert torch.equal(ins[k], before[k]), "input %s changed" % k
    host = {k: v.cpu().numpy() for k, v in out.items()}
    res = []
    for b in range(B):
        n = int(host["count"][b])
        assert 0 <= n <= M
        assert (host["roi_index"][b, n:] == -1).all() and not host["boxes"][b, n:].any() and not host["conf"][b, n:].any()
        assert not host["classes"][b, n:].any() and not host["features"][b, n:].any()
        res.append({k: host[k][b, :n] for k in engine.REGION_FIELDS})
    return res


def check_stage(probs, rois, fc7, nrois, scales, nms, gpu_pred, conf, mn, mx):
    B = len(nrois)
    R = probs.shape[0] // B
    res = run_stage(probs, rois, fc7, nrois, scales, nms, gpu_pred, conf, mn, mx)
    for b in range(B):
        s = slice(b * R, (b + 1) * R)
        want = RO.image_regions(probs[s], rois[s], nrois[b], F(scales[b]), nms, gpu_pred, conf, mn, mx, fc7=fc7[s])
        RO.compare(res[b], want)
    return res


@pytest.mark.parametrize("C,R,B", [(2, 300, 2), (21, 300, 3), (81, 300, 2), (21, 1000, 2), (81, 1000, 1), (2, 5000, 1), (21, 5000, 2),
                                   (81, 5000, 1)])
def test_stage_capacities(cuda, C, R, B):
    rng = np.random.default_rng(C * 7 + R + B)
    nrois = [R - 17, 0, 5][:B] if B > 1 else [R - 3]
    probs, rois, fc7 = make_batch(rng, B, R, C, nrois)
    scales = [1.6, 0.8, 1.25][:B]
    for gpu_pred in (True, False):
        for conf, mn, mx in ((0.2, 10, 100), (0.0, 10, 100), (1.0, 10, 100), (0.2, 36, 36)):
            check_stage(probs, rois, fc7, nrois, scales, 0.3, gpu_pred, conf, mn, mx)
    # the count inside [min_boxes, max_boxes]: the threshold at the 25th best confidence of image 0
    boxes = RO.roi_boxes(rois[:nrois[0]], F(scales[0]))
    conf0, _ = RO.best_kept_class(boxes, probs[:nrois[0]], 0.3, True)
    t = float(np.sort(conf0)[-25])
    res = check_stage(probs, rois, fc7, nrois, scales, 0.3, True, t, 10, 100)
    assert res[0]["roi_index"].shape[0] == 25 and np.array_equal(res[0]["roi_index"], np.sort(res[0]["roi_index"]))


def test_stage_edges(cuda):
    """Scores one ulp either side of the threshold, tied confidences, tied scores within a class, an RoI suppressed in every
    class, num_rois below min_boxes and 0."""
    rng = np.random.default_rng(11)
    R, C = 300, 21
    probs, rois, fc7 = make_batch(rng, 1, R, C, [R], spread=6000.0, size=(10, 20))   # isolated boxes
    probs *= F(0.45)                                                                # every score < 0.5 ...
    half = F(0.5)
    probs[3, 5], probs[4, 2], probs[5, 7] = half, np.nextafter(half, F(0)), np.nextafter(half, F(1))   # ... except these
    probs[11], probs[12], probs[40] = probs[10], probs[10], probs[10]                # tied confidences
    rois[21, 1:] = rois[20, 1:]                                                       # same box, same scores: 21 loses every class
    probs[21] = probs[20]
    rois[31, 1:] = rois[30, 1:]                                                       # lower score in every class: 30 loses
    probs[30] = probs[31] * F(0.5)
    for gpu_pred in (True, False):
        res = check_stage(probs, rois, fc7, [R], [1.0], 0.3, gpu_pred, 0.5, 0, 100)
        assert res[0]["roi_index"].tolist() == [3, 5]
        res = check_stage(probs, rois, fc7, [R], [1.0], 0.5, gpu_pred, 0.5, 10, 100)     # count 2 < 10: sorted, ties to the lower row
        idx = res[0]["roi_index"].tolist()
        assert idx[:2] == [5, 3] and len(idx) == 10
        res = check_stage(probs, rois, fc7, [R], [1.0], 0.3, gpu_pred, 0.5, R, R)       # every row, sorted
        conf = dict(zip(res[0]["roi_index"].tolist(), res[0]["conf"].tolist()))
        assert conf[21] == 0.0 and conf[30] == 0.0 and conf[20] > 0 and conf[31] > 0
        pos = {i: k for k, i in enumerate(res[0]["roi_index"].tolist())}
        assert pos[10] < pos[11] < pos[12] < pos[40]
    for nr in (0, 4, 9):
        res = check_stage(probs, rois, fc7, [nr], [1.0], 0.3, True, 0.2, 10, 100)
        assert res[0]["roi_index"].shape[0] == nr


def test_stage_batch_equals_single_images(cuda):
    rng = np.random.default_rng(12)
    R, C, nrois, scales = 300, 21, [280, 0, 7], [1.6, 0.8, 1.25]
    probs, rois, fc7 = make_batch(rng, 3, R, C, nrois)
    batch = run_stage(probs, rois, fc7, nrois, scales, 0.3, False, 0.2, 10, 100)
    for b in range(3):
        s = slice(b * R, (b + 1) * R)
        r1 = rois[s].copy()
        r1[:, 0] = 0
        single = run_stage(probs[s], r1, fc7[s], [nrois[b]], [scales[b]], 0.3, False, 0.2, 10, 100)[0]
        for k in engine.REGION_FIELDS:
            assert single[k].tobytes() == batch[b][k].tobytes(), k


# ---- network level ------------------------------------------------------------------------------------------------------------
def build(net_name, num_classes, scales):
    from model.config import cfg
    from nets.mobilenet_v1 import mobilenetv1
    from nets.resnet_v1 import resnetv1
    from nets.vgg16 import vgg16
    cfg.TEST.HAS_RPN = True
    net = vgg16() if net_name == "vgg16" else mobilenetv1() if net_name == "mobile" else resnetv1(num_layers=int(net_name[3:]))
    net.create_architecture("TEST", num_classes, tag="default", anchor_scales=scales, anchor_ratios=(0.5, 1, 2))
    net.load_weights(synth.make(net_name, num_classes, 3 * len(scales)))
    return net


def check_net(net, plan, res, conf, mn, mx):
    """detect_regions' output == the oracle on the plan's own device cls_prob / rois / num_rois / fc7 / im_meta."""
    B, R = plan.batch, plan.R
    probs, rois, fc7 = plan.cls_prob.cpu().numpy(), plan.rois.cpu().numpy(), plan.fc7.cpu().numpy()
    nroi, meta = plan.num_rois.cpu().numpy(), plan.im_meta.cpu().numpy()
    o = net.options
    for b in range(B):
        s = slice(b * R, (b + 1) * R)
        want = RO.image_regions(probs[s], rois[s], nroi[b], meta[b, 0], o["nms_thresh"], o["use_gpu_nms"], conf, mn, mx, fc7=fc7[s])
        RO.compare(res[b], want)
        assert want["roi_index"].shape[0] > 0


def test_network_resnet101_batch2(cuda):
    net = build("res101", 81, (4, 8, 16, 32))
    hw = (600, 800)
    blobs = np.concatenate([synth.synthetic_blob(hw[0], hw[1], s) for s in (1, 2)], axis=0)
    scales, orig = [1.0, 1.25], [(600, 800), (480, 640)]
    before, plan = net.detect_batch(blobs, scales, orig)
    res, plan2 = net.detect_regions(blobs, scales, orig)
    assert plan2 is plan and len(res) == 2
    check_net(net, plan, res, 0.2, 10, 100)
    after, _ = net.detect_batch(blobs, scales, orig)
    assert all(a.tobytes() == b.tobytes() for a, b in zip(before, after))
    # a threshold that leaves the count inside the range, the other predicate, min = max = 36
    t = float(np.sort(res[0]["conf"])[-1]) * 0.5
    net.options["use_gpu_nms"] = not net.options["use_gpu_nms"]
    for args in ((t, 1, 100), (0.2, 36, 36)):
        res, _ = net.detect_regions(blobs, scales, orig, *args)
        check_net(net, plan, res, *args)
    # graph replay == eager launches
    graph, _ = net.detect_regions(blobs, scales, orig)
    plan.use_graph = False
    try:
        eager, _ = net.detect_regions(blobs, scales, orig)
    finally:
        plan.use_graph = True
    for g, e in zip(graph, eager):
        for k in engine.REGION_FIELDS:
            assert g[k].tobytes() == e[k].tobytes(), k


@pytest.mark.parametrize("net_name,C,scales,mode", [("vgg16", 21, (8, 16, 32), "crop"), ("mobile", 81, (4, 8, 16, 32), "crop"),
                                                    ("res50", 21, (8, 16, 32), "align")])
def test_network_backbones_and_pooling(cuda, net_name, C, scales, mode):
    from model.config import cfg
    old = cfg.POOLING_MODE
    cfg.POOLING_MODE = mode
    try:
        net = build(net_name, C, scales)
    finally:
        cfg.POOLING_MODE = old
    assert net.options["pooling_mode"] == mode
    hw = (320, 480)
    blob = synth.synthetic_blob(*hw)
    res, plan = net.detect_regions(blob, [1.0], [hw])
    fdim = {"vgg16": 4096, "mobile": 1024}.get(net_name, 2048)
    assert res[0]["features"].shape[1] == fdim
    check_net(net, plan, res, 0.2, 10, 100)


def test_extract_features_regions_tool(cuda, tmp_path):
    import cv2
    from datasets.factory import get_imdb
    from model.test import _get_blobs
    tool = os.path.join(ROOT, "tools", "extract_features.py")
    r = subprocess.run([sys.executable, tool, "--imdb", "synthetic_4_21", "--net", "res50", "--batch", "2", "--regions",
                        "--tsv", str(tmp_path / "regions.tsv"), "--out", str(tmp_path / "reg")], capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    imdb = get_imdb("synthetic_4_21")
    net = build("res50", 21, (8, 16, 32))
    ims = [cv2.imread(imdb.image_path_at(i)) for i in range(4)]
    prep = [_get_blobs(im) for im in ims]
    with open(tmp_path / "regions.tsv", newline="") as f:
        rows = list(csv.DictReader(f, delimiter="\t", fieldnames=["image_id", "image_w", "image_h", "num_boxes", "boxes", "features"]))
    assert [row["image_id"] for row in rows] == [str(x) for x in imdb.image_index]
    for g in ((0, 1), (2, 3)):
        blobs = np.concatenate([prep[i][0]["data"] for i in g], axis=0)
        res, _ = net.detect_regions(blobs, [float(prep[i][1][0]) for i in g], [ims[i].shape[:2] for i in g])
        for i, reg in zip(g, res):
            z = np.load(tmp_path / "reg" / ("%s.npz" % imdb.image_index[i]))
            assert sorted(z.files) == sorted(["boxes", "features", "conf", "classes", "roi_index", "image_h", "image_w", "num_boxes"])
            n = int(z["num_boxes"])
            assert 10 <= n <= 100 and (int(z["image_h"]), int(z["image_w"])) == ims[i].shape[:2]
            for k in engine.REGION_FIELDS:
                assert z[k].tobytes() == reg[k].tobytes() and z[k].shape[0] == n, k
            row = rows[i]
            assert int(row["num_boxes"]) == n and (int(row["image_h"]), int(row["image_w"])) == ims[i].shape[:2]
            assert np.frombuffer(base64.b64decode(row["boxes"]), F).reshape(n, 4).tobytes() == reg["boxes"].tobytes()
            assert np.frombuffer(base64.b64decode(row["features"]), F).reshape(n, -1).tobytes() == reg["features"].tobytes()


def test_bench_regions_tool_runs(cuda):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "bench_regions.py"), "--net", "mobile", "--batch", "1",
                        "--steps", "2", "--warmup", "1", "--rounds", "1"], capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    line = json.loads([x for x in r.stdout.splitlines() if x.startswith("{")][-1])
    assert line["detect"]["value"] > 0 and line["regions"]["value"] > 0 and line["step"]["us"] > 0
