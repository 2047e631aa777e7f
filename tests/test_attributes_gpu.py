"""The attribute head on the bottom-up regions, on the GPU, against tests/attr_oracle.py: the two kernels at stage level on seeded
inputs (guard-banded outputs, inputs unchanged), and whole networks through Network.detect_regions on each layer's own device
inputs, with the five region fields bit-identical to a network without the head."""
import base64
import csv
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import attr_oracle as AO  # noqa: E402
import stage_ref64 as S  # noqa: E402
from tf_faster_rcnn_b200 import engine, ops, synth  # noqa: E402

pytestmark = pytest.mark.gpu
F = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = 64
SENTINEL = {torch.float32: 0x7fc0dead, torch.int32: -7777}
VG = (401, 256, 512)


@pytest.fixture(scope="module", autouse=True)
def _release_networks():
    """This module's plans (GBs of device memory at 600x800) are released and collected at its end: networks register
    themselves process-wide and reference their plans, so dropping them from the registry alone frees nothing."""
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


def guarded(shape, dtype):
    n = int(np.prod(shape))
    raw = torch.full((n + 2 * G,), SENTINEL[dtype], dtype=torch.int32, device="cuda")
    return raw, raw[G:G + n].view(dtype).view(*shape)


def check_guards(bufs, saved):
    for k, (raw, _) in bufs.items():
        assert torch.equal(raw[:G], saved[k][0]) and torch.equal(raw[-G:], saved[k][1]), "guard band of %s overwritten" % k


# ---- frcnn_regions_attr_embed --------------------------------------------------------------------------------------------------
def edge_logits(rng, n, C):
    """Class-logit rows: random, ties for the maximum, a NaN (first NaN wins), all equal, -inf rows, +inf ties."""
    z = rng.normal(0, 2, (n, C)).astype(F)
    for i in range(n):
        kind = i % 6
        if kind == 1:
            j = rng.choice(C, 2, replace=False)
            z[i, j] = z[i].max() + 1
        elif kind == 2:
            j = rng.choice(C, min(C, 2), replace=False)
            z[i, j] = np.nan
        elif kind == 3:
            z[i] = F(0.25)
        elif kind == 4:
            z[i] = -np.inf
        elif kind == 5:
            z[i, rng.choice(C, 2, replace=False)] = np.inf
    return z


@pytest.mark.parametrize("C", [2, 81, 1601, 4096])
def test_embed_equals_oracle(cuda, C):
    rng = np.random.default_rng(C)
    B, R, M, E = 3, 300, 100, 256
    z = edge_logits(rng, B * R, C)
    table = rng.normal(0, 1, (C, E)).astype(F)
    table[:, 0] = np.arange(C)                          # the class is readable from the row, exactly
    counts = [0, 37, M]
    index = np.full((B, M), -1, np.int32)
    for b, n in enumerate(counts):
        index[b, :n] = rng.choice(R, n, replace=False)
    ins = dict(z=torch.from_numpy(z).cuda(), index=torch.from_numpy(index).cuda(), count=torch.tensor(counts, dtype=torch.int32).cuda(),
               table=torch.from_numpy(table).cuda())
    before = {k: v.clone() for k, v in ins.items()}
    bufs = dict(emb=guarded((B * M, E), torch.float32))
    saved = {k: (r[:G].clone(), r[-G:].clone()) for k, (r, _) in bufs.items()}
    ops.regions_attr_embed(ins["z"], C, ins["index"], ins["count"], ins["table"], bufs["emb"][1])
    torch.cuda.synchronize()
    check_guards(bufs, saved)
    for k in ins:
        assert torch.equal(ins[k].view(torch.int32) if ins[k].dtype == torch.float32 else ins[k],
                           before[k].view(torch.int32) if before[k].dtype == torch.float32 else before[k]), "input %s changed" % k
    emb = bufs["emb"][1].cpu().numpy().reshape(B, M, E)
    for b, n in enumerate(counts):
        rows = z[b * R + index[b, :n]]
        want_c, want_e = AO.embed(rows, table)
        assert np.array_equal(want_c, np.argmax(rows, axis=1))
        S.check_exact(emb[b, :n, 0].astype(np.int64), want_c, "class of image %d" % b)
        assert emb[b, :n].tobytes() == want_e.tobytes(), "embedding rows of image %d" % b
        assert not emb[b, n:].any() and not np.signbit(emb[b, n:]).any(), "padding rows of image %d" % b


# ---- frcnn_attr_finish ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("A", [2, 401, 1024, 4096])
def test_finish_within_the_softmax_bound(cuda, A):
    rng = np.random.default_rng(A + 1)
    B, M = 2, 37
    ld = (A + 3) // 4 * 4 + 4
    x, _ = S.logit_rows(rng, B * M, A)
    x[5, A // 2] = np.nan                               # a NaN logit: every probability NaN, attributes 1
    score = np.full((B * M, ld), 1e30, F)                # columns past A must not be read
    score[:, :A] = x
    counts = [M, 11]
    ins = dict(score=torch.from_numpy(score).cuda(), count=torch.tensor(counts, dtype=torch.int32).cuda())
    before = {k: v.clone() for k, v in ins.items()}
    bufs = dict(prob=guarded((B, M, A), torch.float32), attr=guarded((B, M), torch.int32), conf=guarded((B, M), torch.float32))
    saved = {k: (r[:G].clone(), r[-G:].clone()) for k, (r, _) in bufs.items()}
    ops.attr_finish(ins["score"], A, ins["count"], bufs["prob"][1], bufs["attr"][1], bufs["conf"][1])
    torch.cuda.synchronize()
    check_guards(bufs, saved)
    for k in ins:
        assert torch.equal(ins[k].view(torch.int32), before[k].view(torch.int32)), "input %s changed" % k
    prob = bufs["prob"][1].cpu().numpy().reshape(B * M, A)
    attr = bufs["attr"][1].cpu().numpy().reshape(-1)
    conf = bufs["conf"][1].cpu().numpy().reshape(-1)
    valid = np.concatenate([np.arange(b * M, b * M + n) for b, n in enumerate(counts)])
    pad = np.setdiff1d(np.arange(B * M), valid)
    assert not prob[pad].any() and (attr[pad] == -1).all() and not conf[pad].any()
    assert not np.signbit(prob[pad]).any() and not np.signbit(conf[pad]).any()
    assert np.isnan(prob[5]).all() and attr[5] == 1 and np.isnan(conf[5])
    ok = valid[valid != 5]
    p64, bound = AO.softmax64(x[ok], A)
    _, decided = AO.check_attributes(prob[ok], attr[ok], conf[ok], p64, bound, "A=%d" % A)
    assert decided > len(ok) // 2
    eq = ok[(x[ok] == x[ok, :1]).all(axis=1)]            # the 'equal' rows: all probabilities tie, the first (1) wins
    assert eq.size and (attr[eq] == 1).all()


# ---- network level --------------------------------------------------------------------------------------------------------------
def build(net_name, C, scales, attributes, weights=None, mode="nms"):
    from model.config import cfg
    from nets.mobilenet_v1 import mobilenetv1
    from nets.resnet_v1 import resnetv1
    from nets.vgg16 import vgg16
    saved = (dict(cfg.ATTRIBUTES), cfg.TEST.MODE)
    cfg.TEST.HAS_RPN = True
    cfg.ATTRIBUTES.NUM_CLASSES = attributes[0] if attributes else 0
    cfg.TEST.MODE = mode
    try:
        net = vgg16() if net_name == "vgg16" else mobilenetv1() if net_name == "mobile" else resnetv1(num_layers=int(net_name[3:]))
        net.create_architecture("TEST", C, tag="default", anchor_scales=scales, anchor_ratios=(0.5, 1, 2))
    finally:
        cfg.ATTRIBUTES.update(saved[0])
        cfg.TEST.MODE = saved[1]
    net.load_weights(weights if weights is not None else synth.make(net_name, C, 3 * len(scales), attributes=VG))
    return net


def check_plan(net, plan, res):
    """The head on the plan's own device buffers: the embedding rows exact, fc_attr and attr_score within the conv bound on their
    own device inputs, attr_prob within the softmax bound on the device's attr_score, attributes / attr_conf by check_attributes;
    the returned dicts equal the device buffers.  -> worst err/bound per layer."""
    A, E, H = net.options["attributes"]
    sc, w, C = net.scope, net.weights, net.num_classes
    B, R = plan.batch, plan.R
    out = {k: v.cpu().numpy() for k, v in plan.reg_out.items()}
    M = out["conf"].shape[1]
    bufs = {k: plan.attr_bufs[k].cpu().numpy() for k in ("emb", "hidden", "score")}
    counts = out["count"]
    z = plan.cls_score.cpu().numpy()
    feats = out["features"].reshape(B * M, -1)
    worst = dict(fc_attr=0.0, attr_score=0.0, attr_prob=0.0)
    y, bound = AO.fc64(np.concatenate([feats, bufs["emb"]], axis=1), w[sc + "/fc_attr/weights"], w[sc + "/fc_attr/biases"], relu=True)
    worst["fc_attr"] = S.check_bounded(bufs["hidden"], y, bound, "fc_attr")
    y, bound = AO.fc64(bufs["hidden"], w[sc + "/attr_score/weights"], w[sc + "/attr_score/biases"], relu=False)
    worst["attr_score"] = S.check_bounded(bufs["score"][:, :A], y, bound, "attr_score")
    assert not bufs["score"][:, A:].any()
    for b in range(B):
        n = int(counts[b])
        rows = slice(b * M, b * M + n)
        want_c, want_e = AO.embed(z[b * R + out["roi_index"][b, :n]], w[sc + "/cls_embedding/weights"])
        assert bufs["emb"][rows].tobytes() == want_e.tobytes(), "embedding rows of image %d" % b
        assert not bufs["emb"][b * M + n:(b + 1) * M].any()
        p64, pb = AO.softmax64(bufs["score"][rows], A)
        r, _ = AO.check_attributes(out["attr_prob"][b, :n], out["attributes"][b, :n], out["attr_conf"][b, :n], p64, pb, "image %d" % b)
        worst["attr_prob"] = max(worst["attr_prob"], r)
        assert not out["attr_prob"][b, n:].any() and (out["attributes"][b, n:] == -1).all() and not out["attr_conf"][b, n:].any()
        for k in engine.REGION_FIELDS + engine.ATTR_FIELDS:
            assert res[b][k].tobytes() == out[k][b, :n].tobytes(), k
    return worst


def same_regions(a, b):
    for x, y in zip(a, b):
        for k in engine.REGION_FIELDS:
            assert x[k].tobytes() == y[k].tobytes(), k


def test_network_resnet101_visual_genome(cuda):
    """1601 classes, 401 attributes, 12 anchors at 600x800: batch 1 and batch 3, head off vs on, max_boxes 36 then 100 on one
    plan, graph replay == eager launches."""
    scales = (4, 8, 16, 32)
    weights = synth.make("res101", 1601, 12, attributes=VG)
    on, off = build("res101", 1601, scales, VG, weights), build("res101", 1601, scales, None, weights)
    hw = (600, 800)
    blobs = np.concatenate([synth.synthetic_blob(hw[0], hw[1], s) for s in (1, 2, 3)], axis=0)
    scl, orig = [1.0, 1.25, 0.8], [(600, 800), (480, 640), (750, 1000)]
    singles = []
    for b in range(3):
        res_on, plan = on.detect_regions(blobs[b:b + 1], scl[b:b + 1], orig[b:b + 1])
        res_off, _ = off.detect_regions(blobs[b:b + 1], scl[b:b + 1], orig[b:b + 1])
        assert sorted(res_on[0]) == sorted(engine.REGION_FIELDS + engine.ATTR_FIELDS) and sorted(res_off[0]) == sorted(engine.REGION_FIELDS)
        same_regions(res_on, res_off)
        print("res101 1601 batch 1 image %d: %s" % (b, check_plan(on, plan, res_on)))
        singles.append(res_on[0])
    res_on, plan = on.detect_regions(blobs, scl, orig)
    res_off, _ = off.detect_regions(blobs, scl, orig)
    same_regions(res_on, res_off)
    print("res101 1601 batch 3: %s" % check_plan(on, plan, res_on))
    # batch 3 against the single images: conv plans at another M may split K differently (DESIGN §2), so the network outputs,
    # and with them the regions, may differ in their last bits; the regions both runs select agree to a relative 1e-4
    for b in range(3):
        s, t = singles[b], res_on[b]
        common, i, j = np.intersect1d(s["roi_index"], t["roi_index"], return_indices=True)
        assert len(common) >= 0.9 * max(len(s["roi_index"]), 1)
        np.testing.assert_allclose(s["attr_prob"][i], t["attr_prob"][j], rtol=1e-4, atol=1e-9)
    # max_boxes 36, then 100 again on the same plan
    for mx in (36, 100):
        res, plan2 = on.detect_regions(blobs, scl, orig, 0.2, 10, mx)
        assert plan2 is plan and plan.reg_out["attr_prob"].shape == (3, mx, VG[0])
        check_plan(on, plan, res)
        same_regions(res, off.detect_regions(blobs, scl, orig, 0.2, 10, mx)[0])
    # graph replay == eager
    graph, _ = on.detect_regions(blobs, scl, orig)
    plan.use_graph = False
    try:
        eager, _ = on.detect_regions(blobs, scl, orig)
    finally:
        plan.use_graph = True
    for g, e in zip(graph, eager):
        for k in engine.REGION_FIELDS + engine.ATTR_FIELDS:
            assert g[k].tobytes() == e[k].tobytes(), k


def test_network_top_mode_5000_rois(cuda):
    scales = (4, 8, 16, 32)
    weights = synth.make("res101", 1601, 12, attributes=VG)
    net = build("res101", 1601, scales, VG, weights, mode="top")
    hw = (600, 800)
    res, plan = net.detect_regions(synth.synthetic_blob(*hw), [1.0], [hw])
    assert plan.R == 5000
    print("res101 1601 top 5000: %s" % check_plan(net, plan, res))


@pytest.mark.parametrize("net_name", ["mobile", "vgg16"])
def test_network_backbones(cuda, net_name):
    scales = (4, 8, 16, 32)
    weights = synth.make(net_name, 81, 12, attributes=VG)
    on, off = build(net_name, 81, scales, VG, weights), build(net_name, 81, scales, None, weights)
    hw = (320, 480)
    blob = synth.synthetic_blob(*hw)
    res, plan = on.detect_regions(blob, [1.0], [hw])
    same_regions(res, off.detect_regions(blob, [1.0], [hw])[0])
    assert res[0]["features"].shape[1] == {"vgg16": 4096, "mobile": 1024}[net_name]
    print("%s 81: %s" % (net_name, check_plan(on, plan, res)))


def test_extract_features_regions_with_attributes(cuda, tmp_path):
    import cv2
    from datasets.factory import get_imdb
    from model.test import _get_blobs
    tool = os.path.join(ROOT, "tools", "extract_features.py")
    r = subprocess.run([sys.executable, tool, "--imdb", "synthetic_4_21", "--net", "res50", "--batch", "2", "--regions",
                        "--tsv", str(tmp_path / "regions.tsv"), "--out", str(tmp_path / "reg"), "--set", "ATTRIBUTES.NUM_CLASSES", "401"],
                       capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    imdb = get_imdb("synthetic_4_21")
    net = build("res50", 21, (8, 16, 32), VG)
    ims = [cv2.imread(imdb.image_path_at(i)) for i in range(4)]
    prep = [_get_blobs(im) for im in ims]
    with open(tmp_path / "regions.tsv", newline="") as f:
        rows = list(csv.reader(f, delimiter="\t"))
    assert [row[0] for row in rows] == [str(x) for x in imdb.image_index] and all(len(row) == 8 for row in rows)
    for g in ((0, 1), (2, 3)):
        blobs = np.concatenate([prep[i][0]["data"] for i in g], axis=0)
        res, _ = net.detect_regions(blobs, [float(prep[i][1][0]) for i in g], [ims[i].shape[:2] for i in g])
        for i, reg in zip(g, res):
            z = np.load(tmp_path / "reg" / ("%s.npz" % imdb.image_index[i]))
            assert sorted(z.files) == sorted(list(engine.REGION_FIELDS + engine.ATTR_FIELDS) + ["image_h", "image_w", "num_boxes"])
            n = int(z["num_boxes"])
            for k in engine.REGION_FIELDS + engine.ATTR_FIELDS:
                assert z[k].tobytes() == reg[k].tobytes() and z[k].shape[0] == n, k
            assert z["attr_prob"].shape == (n, 401) and z["attributes"].dtype == np.int32
            row = rows[i]
            assert int(row[3]) == n
            assert np.frombuffer(base64.b64decode(row[4]), F).reshape(n, 4).tobytes() == reg["boxes"].tobytes()
            assert np.frombuffer(base64.b64decode(row[5]), F).reshape(n, -1).tobytes() == reg["features"].tobytes()
            assert np.frombuffer(base64.b64decode(row[6]), np.int32).tobytes() == reg["attributes"].tobytes()
            assert np.frombuffer(base64.b64decode(row[7]), F).tobytes() == reg["attr_conf"].tobytes()


def test_bench_attributes_tool_runs(cuda):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "bench_attributes.py"), "--batch", "1", "--steps", "2",
                        "--warmup", "1", "--rounds", "1", "--classes", "81"], capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    import json
    line = json.loads([x for x in r.stdout.splitlines() if x.startswith("{")][-1])
    assert line["region_fields_identical"] and line["head_launches"]["us"] > 0
