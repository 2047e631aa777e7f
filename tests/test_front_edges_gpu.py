"""The kernels ahead of the head at their edges, through the C ABI, against the models and float64 references of
front_ref64.py and the oracle:

* bit for bit: the preprocess blob (against the op-order model, and within its float64 bound), max pool (against the
  oracle), the sort order and sorted keys, and the proposals / gather_top / nms_sorted_dev survivors and records;
* within the fma-chain bound: conv_first and depthwise3x3 (max err / bound printed);
* the NaN rule (DESIGN.md): ReLU / ReLU6 epilogues and max pool use fmaxf, so a NaN becomes 0 or drops out of the window.
Every output sits between sentinel guard bands and every input is checked unchanged afterwards."""
import numpy as np
import pytest
import torch

import front_ref64 as R
from oracle import nms as ONMS
from stage_ref64 import GUARD, SENTINEL, check_exact, check_guarded, guarded_out

pytestmark = pytest.mark.gpu
F = np.float32
MEANS = (102.9801, 115.9465, 122.7717)


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def unchanged(d, a, what):
    assert np.array_equal(d.cpu().numpy().view(np.uint8), np.ascontiguousarray(a).view(np.uint8)), "%s was modified" % what


def guarded_int(shape, fill=-7):
    numel = int(np.prod(shape))
    buf = torch.full((numel + 2 * GUARD,), int(SENTINEL), dtype=torch.int32, device="cuda")
    out = buf[GUARD:GUARD + numel].view(shape)
    out.fill_(fill)
    return buf, out


# ---- preprocess -------------------------------------------------------------------------------------------------------------
GEOMS = R.preprocess_geometries() + R.tta_geometries()
OTHER_MEANS = (0.5, 127.25, 255.0)


@pytest.mark.parametrize("hflip", [False, True])
@pytest.mark.parametrize("geom", [pytest.param(g, id=g[0]) for g in GEOMS])
def test_preprocess_edges(cuda, geom, hflip):
    from tf_faster_rcnn_b200 import ops
    name, h0, w0, fx, fy, H, W = geom
    worst = 0.0
    for means in (MEANS, OTHER_MEANS) if name in ("x1", "fx!=fy", "2x2") else (MEANS,):
        im = R.edge_image(np.random.default_rng(h0 * 7 + w0), h0, w0)
        imd = dev(im)
        buf, out = guarded_out((1, H, W, 3))
        ops.preprocess(imd, np.asarray(means, np.float64), fx, fy, out, hflip=hflip)
        got = out.cpu().numpy()[0]
        check_guarded(buf, out.numel(), "blob")
        unchanged(imd, im, "image")
        check_exact(got, R.preprocess_model(im, means, fx, fy, H, W, hflip), "preprocess %s" % name)
        truth, bound = R.preprocess_truth(im, means, fx, fy, H, W, hflip)
        err = np.abs(got.astype(np.float64) - truth)
        assert (err <= bound).all(), "max err/bound %.3g" % (err / bound).max()
        worst = max(worst, float((err / bound).max()))
    print("\n[preprocess %s hflip=%d] max err/bound %.3f" % (name, hflip, worst))


# ---- conv_first / depthwise -----------------------------------------------------------------------------------------------
CONV1 = {"resnet": (7, 2, 64, "EXPLICIT", 1, True), "vgg": (3, 1, 64, "SAME", 1, False), "mobilenet": (3, 2, 32, "EXPLICIT", 2, True)}


def run_conv_first(rng, x, k, stride, cout, mode, act, scale, shift):
    from tf_faster_rcnn_b200 import ops
    n, h, w, _ = x.shape
    wt = (rng.standard_normal((k, k, 3, cout)) * 0.01).astype(F)
    ho, wo, pt, pl = ops.conv_out_hw(h, w, k, stride, mode)
    xd, wd = dev(x), dev(wt)
    sd, hd = (None if scale is None else dev(scale)), (None if shift is None else dev(shift))
    buf, out = guarded_out((n, ho, wo, cout))
    ops.conv_first(xd, wd, sd, hd, out, k, stride, pt, pl, act)
    got = out.cpu().numpy()
    check_guarded(buf, out.numel())
    unchanged(xd, x, "input")
    unchanged(wd, wt, "weights")
    return got, wt.transpose(3, 2, 0, 1), (ho, wo, pt, pl)


def check_chain(got, x, w_oihw, stride, geo, K, scale, shift, act, groups=1):
    ho, wo, pt, pl = geo
    worst = 0.0
    for b in range(x.shape[0]):                         # image by image: the float64 reference of a 600 x 1000 map is large
        y, bound = R.fma_chain_ref(x[b:b + 1], w_oihw, stride, pt, pl, ho, wo, K, scale, shift, act, groups)
        assert np.isfinite(got[b]).all(), "unwritten output"
        err = np.abs(got[b:b + 1].astype(np.float64) - y)
        assert (err <= bound).all(), "max err/bound %.3g" % (err / bound).max()
        worst = max(worst, float((err / bound).max()))
    return worst


def epilogue(rng, c, variant):
    scale = rng.uniform(0.5, 1.5, c).astype(F) if variant in (0, 1) else None
    shift = rng.standard_normal(c).astype(F) if variant in (0, 2) else None
    return scale, shift


@pytest.mark.parametrize("n", [1, 3])
@pytest.mark.parametrize("net", sorted(CONV1))
def test_conv_first_production(cuda, net, n):
    k, stride, cout, mode, act, bn = CONV1[net]
    rng = np.random.default_rng(k + 10 * n)
    x = (rng.standard_normal((n, 600, 1000, 3)) * 50).astype(F)
    scale, shift = epilogue(rng, cout, 0 if bn else 2)
    got, w, geo = run_conv_first(rng, x, k, stride, cout, mode, act, scale, shift)
    r = check_chain(got, x, w, stride, geo, k * k * 3, scale, shift, act)
    print("\n[conv_first %s 600x1000 n=%d] max err/bound %.3f" % (net, n, r))


@pytest.mark.parametrize("hw", [(1, 1), (5, 5), (8, 32), (9, 33)])
def test_conv_first_small_maps(cuda, hw):
    worst = 0.0
    for i, net in enumerate(sorted(CONV1)):
        k, stride, cout, mode, _, _ = CONV1[net]
        for act in (0, 1, 2):
            rng = np.random.default_rng(100 * i + 10 * act + hw[0])
            x = (rng.standard_normal((2, hw[0], hw[1], 3)) * 50).astype(F)
            scale, shift = epilogue(rng, cout, (act + i) % 4)
            got, w, geo = run_conv_first(rng, x, k, stride, cout, mode, act, scale, shift)
            worst = max(worst, check_chain(got, x, w, stride, geo, k * k * 3, scale, shift, act))
    print("\n[conv_first %dx%d] max err/bound %.3f" % (hw[0], hw[1], worst))


@pytest.mark.parametrize("c", [4, 8, 36, 1024])
def test_depthwise_edges(cuda, c):
    from tf_faster_rcnn_b200 import ops
    worst = 0.0
    for hw in ((1, 1), (2, 2), (5, 5), (9, 33)):
        for stride in (1, 2):
            for act in (0, 1, 2):
                rng = np.random.default_rng(c + 7 * act + stride + hw[1])
                x = rng.standard_normal((3 if c < 1024 else 1, hw[0], hw[1], c)).astype(F)
                w = rng.standard_normal((3, 3, c)).astype(F)
                scale, shift = epilogue(rng, c, (act + stride) % 4)
                ho, wo, pt, pl = ops.conv_out_hw(hw[0], hw[1], 3, stride, "SAME" if stride == 1 else "EXPLICIT")
                xd, wd = dev(x), dev(w)
                buf, out = guarded_out((x.shape[0], ho, wo, c))
                ops.depthwise3x3(xd, wd, None if scale is None else dev(scale), None if shift is None else dev(shift), out, stride, pt,
                                 pl, act)
                got = out.cpu().numpy()
                check_guarded(buf, out.numel())
                unchanged(xd, x, "input")
                w_oihw = w.reshape(3, 3, c, 1).transpose(2, 3, 0, 1)
                worst = max(worst, check_chain(got, x, w_oihw, stride, (ho, wo, pt, pl), 9, scale, shift, act, groups=c))
    print("\n[depthwise C=%d] max err/bound %.3f" % (c, worst))


# ---- max pool -----------------------------------------------------------------------------------------------------------
POOLS = [("SAME", 2, 2), ("ZEROPAD1", 3, 2), ("VALID", 1, 2)]     # VGG / ResNet pool1 / shortcut subsample (engine.py)


def run_pool(x, k, s, mode):
    from tf_faster_rcnn_b200 import ops
    n, h, w, c = x.shape
    ho, wo, pt, pl, neg = R.pool_geometry(h, w, k, s, mode)
    xd = dev(x)
    buf, out = guarded_out((n, ho, wo, c))
    ops.max_pool(xd, out, k, s, pt, pl, neg)
    got = out.cpu().numpy()
    check_guarded(buf, out.numel())
    unchanged(xd, x, "input")
    return got, (ho, wo, pt, pl, neg)


@pytest.mark.parametrize("c", [4, 2048])
@pytest.mark.parametrize("pool", POOLS, ids=[p[0] for p in POOLS])
def test_max_pool_edges(cuda, pool, c):
    mode, k, s = pool
    rng = np.random.default_rng(c + k)
    for hw in ((1, 1), (2, 2), (7, 9)):
        x = -np.abs(rng.standard_normal((3,) + hw + (c,))).astype(F) - F(0.25)   # all negative: next to the ZEROPAD1 zeros
        x[1] = rng.standard_normal(hw + (c,))
        x[0, 0, 0, :2] = [np.inf, -np.inf]
        x[2, -1, -1, -2:] = [-np.inf, np.inf]
        got, _ = run_pool(x, k, s, mode)
        check_exact(got, R.pool_oracle(x, k, s, mode), "max_pool %s %s" % (mode, hw))


# ---- the NaN rule --------------------------------------------------------------------------------------------------------
def test_nan_rule_max_pool(cuda):
    """A NaN drops out of its window (fmaxf); a window of NaN only is -Inf, or 0 next to the ZEROPAD1 zeros."""
    rng = np.random.default_rng(3)
    x = rng.standard_normal((2, 6, 7, 8)).astype(F)
    x[0, 2, 3, :] = np.nan
    x[1, :2, :2, 4] = np.nan                            # a whole top-left window
    for mode, k, s in POOLS:
        got, (ho, wo, pt, pl, neg) = run_pool(x, k, s, mode)
        check_exact(got, R.max_pool_model(x, k, s, pt, pl, ho, wo, neg), "max_pool %s" % mode)
        assert not np.isnan(got).any()
    assert np.isnan(R.pool_oracle(x, 2, 2, "SAME")).any()          # the oracle propagates it


def nan_input(rng, shape, places):
    x = rng.standard_normal(shape).astype(F)
    for p in places:
        x[p] = np.nan
    return x


def hit_mask(x, k, stride, geo, c_out):
    ho, wo, pt, pl = geo
    ind = np.isnan(x).any(axis=-1, keepdims=True).astype(np.float64)
    hit = R.conv64_nhwc(ind, np.ones((1, 1, k, k)), stride, pt, pl, ho, wo)[..., 0] > 0
    return np.repeat(hit[..., None], c_out, axis=-1)


@pytest.mark.parametrize("act", [1, 2])
def test_nan_rule_conv_first_and_depthwise(cuda, act):
    """ReLU / ReLU6 are fmaxf(v, 0) (then fminf 6): an output whose window holds a NaN is exactly 0; the others keep their bound."""
    from tf_faster_rcnn_b200 import ops
    rng = np.random.default_rng(act)
    x = nan_input(rng, (2, 19, 41, 3), [(0, 0, 0, 1), (1, 9, 20, 0)]) * F(50)
    scale, shift = epilogue(rng, 64, 0)
    got, w, geo = run_conv_first(rng, x, 7, 2, 64, "EXPLICIT", act, scale, shift)
    hit = hit_mask(x, 7, 2, geo, 64)
    assert hit.any() and (got[hit] == 0).all()
    xc = np.where(np.isnan(x), F(0), x)
    y, bound = R.fma_chain_ref(xc, w, 2, geo[2], geo[3], geo[0], geo[1], 147, scale, shift, act)
    assert (np.abs(got[~hit] - y[~hit]) <= bound[~hit]).all()
    c = 36
    x = nan_input(rng, (2, 9, 11, c), [(0, 4, 5, 3), (1, 0, 10, 35)])
    wt = rng.standard_normal((3, 3, c)).astype(F)
    ho, wo, pt, pl = ops.conv_out_hw(9, 11, 3, 1, "SAME")
    buf, out = guarded_out((2, ho, wo, c))
    ops.depthwise3x3(dev(x), dev(wt), None, dev(shift[:c]), out, 1, pt, pl, act)
    got = out.cpu().numpy()
    check_guarded(buf, out.numel())
    ind = np.isnan(x).astype(np.float64)
    hit = R.conv64_nhwc(ind, np.ones((c, 1, 3, 3)), 1, pt, pl, ho, wo, groups=c) > 0
    assert hit.any() and (got[hit] == 0).all() and np.isfinite(got).all()


def test_nan_rule_packed_conv(cuda):
    """The same rule in the wgmma conv epilogue (ReLU of a PackedConv layer): NaN windows give 0, nothing else changes."""
    from tf_faster_rcnn_b200 import ops, _native as N
    rng = np.random.default_rng(11)
    x = nan_input(rng, (2, 13, 17, 64), [(0, 0, 0, 5), (1, 6, 9, 63)])
    w = (rng.standard_normal((3, 3, 64, 32)) * 0.06).astype(F)
    ho, wo, pt, pl = ops.conv_out_hw(13, 17, 3, 1, "SAME")
    pc = ops.PackedConv(w)
    buf, out = guarded_out((2, ho, wo, 32))
    ops.ConvPlan(dev(x), pc, out, 1, pt, pl, N.ACT_RELU).run()
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    check_guarded(buf, out.numel())
    hit = hit_mask(x, 3, 1, (ho, wo, pt, pl), 32)
    assert hit.any() and (got[hit] == 0).all() and np.isfinite(got).all()


# ---- sort ---------------------------------------------------------------------------------------------------------------------
def run_sort(keys, batch=1, fill_order=-7):
    from tf_faster_rcnn_b200 import ops
    kd = dev(keys.reshape(-1))
    obuf, order = guarded_int((keys.size,), fill_order)
    sbuf, sk = guarded_out((keys.size,))
    try:
        ops.sort_desc(kd, order, sk, batch=batch)
    finally:
        torch.cuda.synchronize()
        check_guarded(obuf, keys.size, "order")
        check_guarded(sbuf, keys.size, "sorted keys")
        unchanged(kd, keys.reshape(-1), "keys")
    return order.cpu().numpy(), sk.cpu().numpy()


def check_sorted(order, sk, keys, what):
    want_o, want_k = R.sort_ref(keys)
    check_exact(order, want_o, what + " order")
    assert np.array_equal(sk.view(np.uint32), want_k.view(np.uint32)), what + " sorted keys (bits)"


def test_sort_special_and_one_byte_keys(cuda):
    rng = np.random.default_rng(17)
    sets = {"special5000": R.special_keys(rng, 5000), "special90112": R.special_keys(rng, 90112),
            "equal90112": np.full(90112, 0.5, F)}
    for byte in range(4):
        sets["byte%d" % byte] = R.one_byte_keys(rng, 22800, byte)
    for name, keys in sets.items():
        check_sorted(*run_sort(keys), keys, name)


def test_sort_capacity_refusal_writes_nothing(cuda):
    from tf_faster_rcnn_b200 import ops
    keys = np.random.default_rng(1).random(90113).astype(F)
    obuf, order = guarded_int((90113,))
    sbuf, sk = guarded_out((90113,))
    with pytest.raises(RuntimeError, match="capacity"):
        ops.sort_desc(dev(keys), order, sk)
    torch.cuda.synchronize()
    check_guarded(obuf, 90113, "order")
    check_guarded(sbuf, 90113, "sorted keys")
    assert (order.cpu().numpy() == -7).all() and np.isnan(sk.cpu().numpy()).all()


@pytest.mark.parametrize("batch,n", [(8, 22800), (3, 5)])
def test_sort_segments(cuda, batch, n):
    rng = np.random.default_rng(batch * n)
    keys = R.special_keys(rng, batch * n).reshape(batch, n) if n > 100 else rng.choice(np.asarray([1, -1, 0, np.nan], F), (batch, n))
    order, sk = run_sort(keys, batch)
    for b in range(batch):
        check_sorted(order.reshape(batch, n)[b], sk.reshape(batch, n)[b], keys[b], "segment %d" % b)


# ---- proposals --------------------------------------------------------------------------------------------------------------
def shuffled(rng, boxes):
    """Boxes in priority order -> (props, scores) in a random input order whose descending score order is the priority."""
    m = boxes.shape[0]
    prio = ((m - np.arange(m)) / m).astype(F)                     # distinct, descending
    q = rng.permutation(m)                                        # input j holds priority position q[j]
    return np.ascontiguousarray(boxes[q]), np.ascontiguousarray(prio[q])


def thr_for(mode, thr):
    return float(ONMS.thresh_f32(thr, mode == "cpu_nms")) if mode != "tf" else float(F(thr))


def oracle_proposals(props, scores, pre, post, thr, mode):
    order = ONMS.argsort_desc(scores)
    m = pre if 0 < pre < scores.shape[0] else scores.shape[0]
    order = order[:m]
    pos = R.oracle_keep(props[order], scores[order], thr, R.MODES[mode], post)
    return order[pos]


def run_proposals(props, scores, batch, pre, post, thr, flags):
    from tf_faster_rcnn_b200 import ops
    n = scores.size // batch
    pd, sd = dev(props.reshape(-1, 4)), dev(scores.reshape(-1))
    order, sk = torch.empty(batch * n, dtype=torch.int32, device="cuda"), torch.empty(batch * n, dtype=torch.float32, device="cuda")
    ops.sort_desc(sd, order, sk, batch=batch)
    rbuf, rois = guarded_out((batch * post, 5))
    sbuf, rs = guarded_out((batch * post,))
    kbuf, keep = guarded_int((batch * post,))
    nbuf, num = guarded_int((batch,))
    ops.proposals(pd, sd, order, pre, post, thr, flags, rois, rs, keep, num, batch=batch)
    torch.cuda.synchronize()
    for b, k, what in ((rbuf, 5, "rois"), (sbuf, 1, "roi scores"), (kbuf, 1, "keep")):
        check_guarded(b, batch * post * k, what)
    check_guarded(nbuf, batch, "num")
    unchanged(pd, props.reshape(-1, 4), "props")
    unchanged(sd, scores.reshape(-1), "scores")
    return (rois.cpu().numpy().reshape(batch, post, 5), rs.cpu().numpy().reshape(batch, post), keep.cpu().numpy().reshape(batch, post),
            num.cpu().numpy())


def check_proposals(got, b, props, scores, src, what):
    rois, rs, keep, num = (g[b] for g in got)
    k = src.shape[0]
    assert num == k, "%s: %d proposals, want %d" % (what, num, k)
    check_exact(keep[:k], src, what + " keep")
    check_exact(rois[:k], np.hstack([np.full((k, 1), b, F), props[src]]), what + " rois")
    check_exact(rs[:k], scores[src], what + " roi scores")
    assert (keep[k:] == -1).all() and not rois[k:].any() and not rs[k:].any(), what + " rows past the count"


PROPOSAL_CAP = 1024                  # post_nms_top_n of the NMS modes (the kept set lives in shared memory)
PROPOSAL_CASES = [(c[0], c[1], c[2], min(c[3], PROPOSAL_CAP), c[4]) for c in R.nms_cases()] + \
    [("grid_post%d" % p, R.grid_boxes(1100), 0.7, p, dict(cuts=0)) for p in (256, 257, 512, 1000, 1024)]


@pytest.mark.parametrize("mode", sorted(R.MODES))
@pytest.mark.parametrize("case", PROPOSAL_CASES, ids=[c[0] for c in PROPOSAL_CASES])
def test_proposals_paths(cuda, case, mode):
    from tf_faster_rcnn_b200 import _native as N
    name, boxes, thr, post, expect = case
    kept, st = R.greedy_nms_model(boxes, thr_for(mode, thr), R.MODES[mode], post)
    R.check_path(st, kept, expect, name)
    rng = np.random.default_rng(len(name) + post)
    props, scores = shuffled(rng, boxes)
    t = thr_for(mode, thr)
    for pre in (0, scores.shape[0], scores.shape[0] + 5):           # pre_nms_top_n >= n: every candidate
        got = run_proposals(props, scores, 1, pre, post, t, R.MODES[mode])
        src = oracle_proposals(props, scores, pre, post, thr, mode)
        check_exact(src, ONMS.argsort_desc(scores)[kept], name + " model")
        check_proposals(got, 0, props, scores, src, "%s %s pre=%d" % (name, mode, pre))
    print("\n[proposals %s %s] rounds %d (4-thread %d), cuts %d, max_out mid-chunk %s, kept %d"
          % (name, mode, st["rounds"], st["tpc4"], st["cuts"], st["maxout_mid_chunk"], kept.shape[0]))
    assert N.NMS_MODE_TF == R.MODES["tf"] and N.NMS_MODE_CPU_NMS == R.MODES["cpu_nms"] and N.NMS_MODE_GPU_NMS == R.MODES["gpu_nms"]


def test_proposals_exact_threshold(cuda):
    thr, cases = R.exact_threshold_cases()
    for mode, (boxes, survivors) in cases.items():
        props, scores = boxes, np.asarray([0.9, 0.8], F)
        got = run_proposals(props, scores, 1, 0, 8, thr, R.MODES[mode])
        check_proposals(got, 0, props, scores, np.asarray(survivors), "exact threshold %s" % mode)


def test_proposals_capacity_refusal(cuda):
    from tf_faster_rcnn_b200 import ops
    props, scores = shuffled(np.random.default_rng(0), R.grid_boxes(1100))
    pd, sd = dev(props), dev(scores)
    order = torch.empty(1100, dtype=torch.int32, device="cuda"); sk = torch.empty(1100, dtype=torch.float32, device="cuda")
    ops.sort_desc(sd, order, sk)
    rbuf, rois = guarded_out((1025, 5))
    sbuf, rs = guarded_out((1025,))
    kbuf, keep = guarded_int((1025,))
    nbuf, num = guarded_int((1,))
    with pytest.raises(RuntimeError, match="capacity"):
        ops.proposals(pd, sd, order, 0, 1025, 0.7, R.MODES["tf"], rois, rs, keep, num)
    torch.cuda.synchronize()
    assert np.isnan(rois.cpu().numpy()).all() and np.isnan(rs.cpu().numpy()).all()
    assert (keep.cpu().numpy() == -7).all() and (num.cpu().numpy() == -7).all()


@pytest.mark.parametrize("mode", sorted(R.MODES))
def test_proposals_batch_regimes(cuda, mode):
    """Three images, three regimes: every box kept, one kept of many identical, the window cut."""
    rng = np.random.default_rng(5)
    cut = {c[0]: c[1] for c in R.nms_cases()}["cut"]
    images = [R.grid_boxes(cut.shape[0]), R.identical_boxes(cut.shape[0]), cut]
    pairs = [shuffled(rng, b) for b in images]
    props = np.stack([p for p, _ in pairs]); scores = np.stack([s for _, s in pairs])
    t = thr_for(mode, 0.5)
    got = run_proposals(props, scores, 3, 0, 1000, t, R.MODES[mode])
    for b in range(3):
        src = oracle_proposals(props[b], scores[b], 0, 1000, 0.5, mode)
        check_proposals(got, b, props[b], scores[b], src, "%s image %d" % (mode, b))
    assert [int(v) for v in got[3]] == [1000, 1, 1000]


@pytest.mark.parametrize("pre", [0, 50])
def test_gather_top_pads_past_the_count(cuda, pre):
    """'top' mode (thresh < 0) with fewer candidates than post_nms_top_n: keep = -1 and zero rows past the count."""
    rng = np.random.default_rng(pre)
    props, scores = shuffled(rng, R.grid_boxes(100))
    got = run_proposals(props[None], scores[None], 1, pre, 300, -1.0, 0)
    src = ONMS.argsort_desc(scores)[:pre or 100]
    check_proposals(got, 0, props, scores, src, "gather_top pre=%d" % pre)


# ---- nms_sorted_dev ------------------------------------------------------------------------------------------------------
def test_nms_sorted_dev(cuda):
    """Against the oracle with max_out < n, = n and > n, n growing (the kept-set workspace regrows), interleaved with nms_host."""
    from tf_faster_rcnn_b200 import ops
    rng = np.random.default_rng(23)
    for n in (100, 1000, 3000):
        boxes = np.vstack([R.grid_boxes(n // 2), R.grid_boxes(n - n // 2) + rng.uniform(-6, 6, (n - n // 2, 4)).astype(F)])
        boxes = np.round(boxes[rng.permutation(n)]).astype(F)
        scores = np.full(n, 0.5, F)
        for mode in sorted(R.MODES):
            flags, t = R.MODES[mode], thr_for(mode, 0.5)
            for max_out in (n // 3, n, n + 17):
                bd = dev(boxes)
                kbuf, keep = guarded_int((max_out,))
                nbuf, num = guarded_int((1,))
                ops.nms_sorted_dev(bd, t, flags, max_out, keep, num)
                torch.cuda.synchronize()
                check_guarded(kbuf, max_out, "keep")
                check_guarded(nbuf, 1, "num")
                unchanged(bd, boxes, "boxes")
                want = R.oracle_keep(boxes, scores, 0.5, flags, max_out)
                k = int(num.item())
                assert k == want.shape[0], (n, mode, max_out, k, want.shape[0])
                check_exact(keep.cpu().numpy()[:k], want, "nms_sorted_dev n=%d %s max_out=%d" % (n, mode, max_out))
                host = ops.nms_host(np.hstack([boxes, scores[:, None]]), t, flags)
                check_exact(host, R.oracle_keep(boxes, scores, 0.5, flags, n), "nms_host")
