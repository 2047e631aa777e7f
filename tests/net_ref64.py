"""Layer-by-layer float64 audit of the detection graph (CPU helper of `test_net_ref64.py` and `test_graph_audit_gpu.py`).

`walk()` restates, from `oracle/nets.py` (RESNET_UNITS, MOBILENET_DEFS) and `oracle/pipeline.py`, the ordered launch list the
engine records for one network: every layer's tape label, the layers whose outputs feed it, and its parameters.  It does not
read the product's `lib/nets/*`: the engine's wiring is checked against an independent reading.

`audit()` walks those layers over a dict of device outputs (one entry per layer key) and holds every layer, fed with the
device outputs of its own inputs, to a reference:

* tensor-core convolutions and FC layers (`conv`): float64 from the raw checkpoint tensors -- conv weights, biases, BatchNorm
  gamma / beta / moving stats with the oracle's eps -- on a deterministic sample of output positions, all output channels:
  the four borders, the seams of the plan's tiles, the first and last rows of every image, and `n_random` interior
  positions; per-RoI layers on the first and last RoI of every image, the RoIs at the M-tile seams and `n_rois` random ones.
  With u = 2^-24, per part j of the layer (conv3 and the folded projection shortcut are two parts), acc_j = x_j . W_j in
  float64, S_j = |x_j| . |W_j|, inv_j = gamma / sqrt(var + eps), shift_j = beta - mean inv_j (float64), and
  a = sum_j acc_j inv_j, b = a + sum_j shift_j, c = b + residual, the output act(c) is held to
      ALPHA u sum_j |inv_j| S_j                         the kernel against float64 (tests/test_conv_gpu.py (b), F16X3 / TF32X3)
    + sum_j (|acc_j| d_inv_j + d_shift_j)              the fp32 BatchNorm fold: d_inv = gamma_4 |inv| (var + eps, sqrt,
                                                        1 / ., gamma * .), d_shift = gamma_6 |mean inv| + u |shift|
    + u sum_j |inv_j| S_j + u |sum_j shift_j|          projection units: the fp32 products W_j inv_j and the fp32 shift sum
                                                        (tests/test_conv_fused.py)
    + 2 u (|a| + |b| + |c|)                            the epilogue's three fp32 operations, doubled for the error already
                                                        in their operands (tests/test_conv_fused.py)
    + ALPHA' sum_j |inv_j| (|x_j - hi - lo| . |W_j|)   F16X3 inputs below 2^-14, where the fp16 split keeps fewer than 22
                                                        bits (tests/conv_split_model.py): the split's actual loss, counted
  F16X1 is held to its operand model instead (conv_split_model.model, BETA u S, tests/test_conv_gpu.py (a)).  The activations
  are 1-Lipschitz.  The mean epilogue (the ResNet head's last conv) is held to the mean of the per-position bounds plus
  stage_ref64's spatial-mean bound.
* SIMT convolutions (`conv_first`, `depthwise`): front_ref64.fma_chain_ref on the whole map with the float64 BatchNorm, plus
  the same fold terms.
* max pool, RoI crop / align / pool, box decodes, sort, proposals and the detection post: bit for bit against their models
  (front_ref64, the oracle crop, roi_pool_oracle, oracle/pipeline.py, stage_ref64); the softmaxes and the MobileNet spatial
  mean within stage_ref64's bounds.

A failure names the layer, the element and err / bound."""
import collections

import numpy as np

import conv_split_model as M
import front_ref64 as FR
import fused_ref64 as R
import stage_ref64 as S
from oracle import nets as ON

F = np.float32
U = M.U
ALPHA = 8.0           # tests/test_conv_gpu.py (b)
BETA = 8.0            # tests/test_conv_gpu.py (a)
TINY16 = 2.0 ** -14   # below it the F16X3 activation split keeps fewer than 22 bits (tests/conv_split_model.py)
RELU, RELU6, NONE = 1, 2, 0

Layer = collections.namedtuple("Layer", "label kind key ins p")


# ---- the walk ----------------------------------------------------------------------------------------------------------
def _same(n, k, s):
    out = -(-n // s)
    return out, max((out - 1) * s + k - n, 0) // 2


def _explicit(n, k, s):
    return (n - 1) // s + 1, (k - 1) // 2


def conv_geometry(h, w, k, stride, pad):
    """(ho, wo, pad_t, pad_l): TF 'SAME', or slim conv2d_same's explicit (k - 1) // 2 before the VALID conv for stride > 1."""
    f = _same if pad == "SAME" else _explicit
    (ho, pt), (wo, pl) = f(h, k, stride), f(w, k, stride)
    return ho, wo, pt, pl


def walk(net, num_anchors, num_classes, pooling="crop", resnet_max_pool=False, rpn=True, head=True):
    """The launch list of `net` ('vgg16', 'res50' / 'res101' / 'res152', 'mobile'), from the image to the detection post.
    Keys: 'image' is the input blob; every other key is the output of the layer that has it."""
    L = []
    sc = ON.scope_of(net)

    def add(label, kind, key, ins, **p):
        L.append(Layer(label, kind, key, tuple(ins), p))
        return key

    def conv(name, x, k=1, stride=1, pad="SAME", act=RELU, eps=None, residual=None, x2=None, mean=False, parts=None, fc=False):
        return add("conv:" + name, "conv", name, [x] + [v for v in (residual, x2) if v is not None], name=name, k=k,
                   stride=stride, pad=pad, act=act, eps=eps, residual=residual, x2=x2, mean=mean, parts=parts or [name], fc=fc)

    def bottleneck(x, x_depth, p, base, stride, eps, mean=False):
        depth = 4 * base
        r = conv(p + "/conv1", x, eps=eps)
        r = conv(p + "/conv2", r, 3, stride, "SAME" if stride == 1 else "EXPLICIT", eps=eps)
        if x_depth == depth:
            sc_ = x
            if stride != 1:
                sc_ = add("max_pool", "max_pool", p + "/shortcut_pool", [x], k=1, stride=stride, mode="VALID")
            return conv(p + "/conv3", r, eps=eps, residual=sc_, mean=mean)
        return conv(p + "/conv3", r, eps=eps, x2=x, mean=mean, parts=[p + "/conv3", p + "/shortcut"])

    x = "image"
    if net == "vgg16":
        for b, n in enumerate([2, 2, 3, 3, 3], start=1):
            for i in range(1, n + 1):
                nm = "vgg_16/conv%d/conv%d_%d" % (b, b, i)
                if b == i == 1:
                    x = add("conv_first:" + nm, "conv_first", nm, [x], name=nm, k=3, stride=1, pad="SAME", act=RELU, eps=None)
                else:
                    x = conv(nm, x, 3)
            if b < 5:
                x = add("max_pool", "max_pool", "vgg_16/pool%d" % b, [x], k=2, stride=2, mode="SAME")
    elif net == "mobile":
        for i in range(12):
            kind, stride, _ = ON.MOBILENET_DEFS[i]
            nm = "MobilenetV1/Conv2d_%d" % i
            if kind == "conv":
                x = add("conv_first:" + nm, "conv_first", nm, [x], name=nm, k=3, stride=stride, pad="EXPLICIT", act=RELU6, eps=1e-3)
            else:
                x = add("depthwise:" + nm + "_depthwise", "depthwise", nm + "_depthwise", [x], name=nm + "_depthwise", k=3,
                        stride=stride, pad="SAME" if stride == 1 else "EXPLICIT", act=RELU6, eps=1e-3)
                x = conv(nm + "_pointwise", x, act=RELU6, eps=1e-3)
    else:
        nl = int(net[3:])
        x = add("conv_first:" + sc + "/conv1", "conv_first", sc + "/conv1", [x], name=sc + "/conv1", k=7, stride=2,
                pad="EXPLICIT", act=RELU, eps=1e-5)
        x = add("max_pool", "max_pool", sc + "/pool1", [x], k=3, stride=2, mode="ZEROPAD1")
        depth = 64
        for bname, base, strides in ON._block_plan(nl)[:3]:
            for u, s in enumerate(strides, start=1):
                x = bottleneck(x, depth, "%s/%s/unit_%d/bottleneck_v1" % (sc, bname, u), base, s, 1e-5)
                depth = 4 * base
    feat = x
    if not rpn:
        return L
    A = num_anchors
    dcol = (2 * A + 3) // 4 * 4
    ld = (dcol + 4 * A + 3) // 4 * 4
    r = conv(sc + "/rpn_conv/3x3", feat, 3)
    heads = conv(sc + "/rpn_heads", r, act=NONE)
    L[-1].p.update(fused=[(sc + "/rpn_cls_score", 0, 2 * A), (sc + "/rpn_bbox_pred", dcol, 4 * A)], cout=ld)
    add("rpn_decode", "rpn_decode", "rpn_decode", [heads], A=A, dcol=dcol)
    add("sort_desc", "sort_desc", "sort_desc", ["rpn_decode"])
    add("proposals", "proposals", "proposals", ["rpn_decode", "sort_desc"])
    if not head:
        return L
    pre_pool = not net.startswith("res") or resnet_max_pool
    pool_label = {"crop": "crop_pool", "align": "roi_align", "pool": "roi_pool"}[pooling]
    x = add(pool_label, "pool", "pool5", [feat, "proposals"], mode=pooling, pre_pool=pre_pool)
    C = num_classes
    if net == "vgg16":
        x = conv("vgg_16/fc6", x, fc=True)
        x = conv("vgg_16/fc7", x, fc=True)
    elif net == "mobile":
        for i in (12, 13):
            nm = "MobilenetV1/Conv2d_%d" % i
            x = add("depthwise:" + nm + "_depthwise", "depthwise", nm + "_depthwise", [x], name=nm + "_depthwise", k=3,
                    stride=1, pad="SAME", act=RELU6, eps=1e-3)
            x = conv(nm + "_pointwise", x, act=RELU6, eps=1e-3)
        x = add("spatial_mean", "spatial_mean", "fc7", [x])
    else:
        nl = int(net[3:])
        bname, base, strides = ON._block_plan(nl)[3]
        depth = 1024
        for u, s in enumerate(strides, start=1):
            x = bottleneck(x, depth, "%s/%s/unit_%d/bottleneck_v1" % (sc, bname, u), base, s, 1e-5, mean=u == len(strides))
            depth = 4 * base
    conv(sc + "/cls_bbox", x, act=NONE, fc=True)
    L[-1].p.update(fused=[(sc + "/cls_score", 0, C), (sc + "/bbox_pred", C, 4 * C)], cout=(5 * C + 3) // 4 * 4)
    add("cls_finish", "cls_finish", "cls_finish", [sc + "/cls_bbox"], C=C)
    add("bbox_decode", "bbox_decode", "bbox_decode", ["proposals", "cls_finish"], C=C)
    add("detect_post", "detect_post", "detect_post", ["cls_finish", "bbox_decode", "proposals"], C=C)
    return L


# ---- float64 layer parameters from the raw tensors ---------------------------------------------------------------------
def bn64(w, name, eps):
    """(inv, shift, d_inv, d_shift) in float64 from the raw tensors of layer `name` (eps None: its biases, exact)."""
    if eps is None:
        b = w.get(name + "/biases") if hasattr(w, "get") else w[name + "/biases"]
        cout = w[name + "/weights"].shape[-1]
        sh = np.zeros(cout) if b is None else np.asarray(b, np.float64)
        z = np.zeros(cout)
        return np.ones(cout), sh, z, z
    p = name + "/BatchNorm/"
    g, be, mu, var = (np.asarray(w[p + k], np.float64) for k in ("gamma", "beta", "moving_mean", "moving_variance"))
    inv = g / np.sqrt(var + eps)
    shift = be - mu * inv
    return inv, shift, S.gamma(4) * np.abs(inv), S.gamma(6) * np.abs(mu * inv) + U * np.abs(shift)


def fused_weights(w, p):
    """HWIO weights and biases of a fused 1x1 layer (RPN heads, cls_score | bbox_pred): each part at its column, zeros
    elsewhere -- the pad columns must come out exactly 0."""
    parts, cout = p["fused"], p["cout"]
    first = w[parts[0][0] + "/weights"]
    cin = first.shape[-2]
    wt = np.zeros((1, 1, cin, cout), F)
    b = np.zeros(cout, np.float64)
    for nm, c0, n in parts:
        wt[..., c0:c0 + n] = np.asarray(w[nm + "/weights"]).reshape(1, 1, cin, n)
        b[c0:c0 + n] = w[nm + "/biases"]
    return wt, b


# ---- samples -----------------------------------------------------------------------------------------------------------
def sample_positions(n, ho, wo, tile, rng, n_random=256):
    """Output positions (img, y, x) of a map layer: the four borders, the tile seams, every image's first and last rows,
    `n_random` interior positions.  tile = (th, tw) of the plan."""
    th, tw = tile
    pts = set()
    for b in range(n):
        for y in (0, ho - 1):
            pts.update((b, y, x) for x in range(wo))
        for x in (0, wo - 1):
            pts.update((b, y, x) for y in range(ho))
    ys = sorted({y for t in range(th, ho, th) for y in (t - 1, t)})
    xs = sorted({x for t in range(tw, wo, tw) for x in (t - 1, t)})
    for b in range(n):
        for y in ys:
            pts.update((b, y, int(x)) for x in rng.choice(wo, min(wo, 8), replace=False))
            pts.update((b, y, x) for x in xs[:16])
        for x in xs:
            pts.update((b, int(y), x) for y in rng.choice(ho, min(ho, 8), replace=False))
    for _ in range(n_random):
        pts.add((int(rng.integers(n)), int(rng.integers(ho)), int(rng.integers(wo))))
    return np.array(sorted(pts), np.int64).reshape(-1, 3)


def sample_rois(r_total, per_image, tn, counts=None, rng=None, n_rois=32):
    """RoI rows of a per-RoI layer: first and last of every image, the rows at the M-tile seams (tn RoIs per tile), ~n_rois
    random ones; only rows holding one of the counts[b] RoIs of image b (rows past a count carry no RoI)."""
    nb = r_total // per_image
    counts = [per_image] * nb if counts is None else [int(c) for c in counts]
    valid = np.concatenate([np.arange(b * per_image, b * per_image + counts[b]) for b in range(nb)])
    rows = set()
    for b in range(nb):
        if counts[b]:
            rows.update((b * per_image, b * per_image + counts[b] - 1))
    if tn > 0:
        seams = [i for t in range(tn, r_total, tn) for i in (t - 1, t)]
        rows.update(seams[::max(1, len(seams) // 16)][:32])
    rows.update(int(i) for i in rng.choice(valid, min(len(valid), n_rois), replace=False))
    return np.intersect1d(np.array(sorted(rows), np.int64), valid)


def patches(x, k, stride, pt, pl, pos):
    """[P, k*k*cin] float64 receptive fields (HWI order, zero padding) of output positions pos (img, y, x)."""
    n, h, w, c = x.shape
    xp = np.zeros((n, h + 2 * k, w + 2 * k, c), np.float64)
    xp[:, k:k + h, k:k + w] = x
    b, y0, x0 = pos[:, 0], pos[:, 1] * stride - pt + k, pos[:, 2] * stride - pl + k
    dy, dx = np.meshgrid(np.arange(k), np.arange(k), indexing="ij")
    return xp[b[:, None], (y0[:, None] + dy.reshape(-1)), (x0[:, None] + dx.reshape(-1))].reshape(len(pos), -1)


# ---- per-layer references ----------------------------------------------------------------------------------------------
class Finding(AssertionError):
    pass


def _check(label, got, want, bound, where):
    got = np.asarray(got, np.float64)
    err = np.abs(got - want)
    with np.errstate(invalid="ignore", divide="ignore"):
        ratio = np.where(err == 0, 0.0, err / bound)
    bad = ~np.isfinite(got) | ~(err <= bound)
    if bad.any():
        i = np.unravel_index(np.argmax(np.where(bad, np.inf, ratio)), ratio.shape)
        raise Finding("%s: %d of %d sampled elements outside the bound, worst at %s: got %r, want %r, err/bound %.3g"
                      % (label, int(bad.sum()), bad.size, where(i), got[i], want[i], ratio[i]))
    i = np.unravel_index(np.argmax(ratio), ratio.shape) if ratio.size else (0,)
    return float(ratio.max()) if ratio.size else 0.0, where(i)


def _exact(label, got, want, what=""):
    try:
        S.check_exact(got, want, label + (" " + what if what else ""))
    except AssertionError as e:
        raise Finding(str(e))
    return 0.0, what


def _act(v, act):
    return v if act == NONE else np.maximum(v, 0) if act == RELU else np.minimum(np.maximum(v, 0), 6)


def conv_ref(lay, w, xs, mode, pos):
    """(y64, bound, tiny) at output positions pos (img, y, x) of a tensor-core conv / FC layer, all channels.
    xs: the device inputs [x, residual?, x2?] as NHWC."""
    p = lay.p
    x = xs[0]
    res = xs[1] if p["residual"] is not None else None
    x2 = xs[-1] if p["x2"] is not None else None
    k, stride = p["k"], p["stride"]
    n, h, wd, _ = x.shape
    ho, wo, pt, pl = conv_geometry(h, wd, k, stride, p["pad"])
    parts = []
    if "fused" in p:
        wt, b = fused_weights(w, p)
        one = np.ones(wt.shape[-1])
        z = np.zeros(wt.shape[-1])
        parts.append((x, wt, one, b, z, z))
    else:
        for j, nm in enumerate(p["parts"]):
            inv, sh, dinv, dsh = bn64(w, nm, p["eps"])
            wt = np.asarray(w[nm + "/weights"], F)
            parts.append((x if j == 0 else x2, wt.reshape((1, 1) + wt.shape) if wt.ndim == 2 else wt, inv, sh, dinv, dsh))
    concat = len(parts) > 1
    whi_parts = None
    if concat and mode == M.F16X1:
        # F16X1's operand model of a projection unit: the device packs W' = [W_1 inv32_1 ; W_2 inv32_2] (fp32 products,
        # engine.concat_layers) as W' / sigma (sigma: a power of two per column, fused_ref64.pack_columns) with ONE weight
        # exponent for the whole matrix and multiplies by sigma in the epilogue, so the split is taken on that matrix
        folded = np.concatenate([(wt * fold32(w, nm, p["eps"])[0]).astype(F) for (_, wt, *_), nm in zip(parts, p["parts"])],
                                axis=2)
        packed, sigma = R.pack_columns(folded)
        whi, _ = M.split_weights(packed.reshape(-1, packed.shape[-1]), M.F16X1)
        whi = whi * sigma.astype(np.float64)
        cuts = np.cumsum([0] + [q[1].shape[2] for q in parts])
        whi_parts = [whi[cuts[j]:cuts[j + 1]] for j in range(len(parts))]
    a = np.zeros((len(pos), parts[0][1].shape[-1]))
    shift = np.zeros(a.shape[1])
    bound = np.zeros_like(a)
    tiny = 0
    for j, (xin, wt, inv, sh, dinv, dsh) in enumerate(parts):
        kk = wt.shape[0]
        wm = wt.reshape(-1, wt.shape[-1]).astype(np.float64)
        P = patches(xin, kk, stride, pt, pl, pos)
        Sj = np.abs(P) @ np.abs(wt.reshape(-1, wt.shape[-1]).astype(np.float64))
        if mode == M.F16X1:
            hi, _ = M.split_activations(P.astype(F), M.F16X1)
            acc = hi @ (whi_parts[j] if concat else M.split_weights(wm.astype(F), M.F16X1)[0])
            if concat:
                acc = acc / inv          # a += acc inv below then adds the model of the packed weights itself
            bound += BETA * U * np.abs(inv) * Sj
        else:
            acc = P @ wm
            bound += ALPHA * U * np.abs(inv) * Sj
            if mode == M.F16X3:
                small = (np.abs(P) < TINY16) & (P != 0)
                if small.any():
                    tiny += int(small.sum())
                    e = np.where(small, M.activation_error(P.astype(F), M.F16X3) * np.abs(P), 0.0)
                    bound += ALPHA * np.abs(inv) * (np.nan_to_num(e) @ np.abs(wm))
        if concat:      # the scale is folded into every weight: its error scales S, not |acc|
            bound += Sj * dinv + U * np.abs(inv) * Sj + dsh
        else:
            bound += np.abs(acc) * dinv + dsh
        a += acc * inv
        shift += sh
    b = a + shift
    c = b if res is None else b + res[pos[:, 0], pos[:, 1], pos[:, 2]].astype(np.float64)
    if concat:
        bound += U * np.abs(shift)
    bound += 2 * U * (np.abs(a) + np.abs(b) + np.abs(c))
    return _act(c, p["act"]), bound, tiny


def map_positions(n, ho, wo, tile, rng, n_random, per_roi):
    if per_roi:
        rows = sample_rois(n, *per_roi, rng=rng)
        yy, xx = np.meshgrid(np.arange(ho), np.arange(wo), indexing="ij")
        return np.stack([np.repeat(rows, ho * wo), np.tile(yy.reshape(-1), len(rows)), np.tile(xx.reshape(-1), len(rows))], 1)
    return sample_positions(n, ho, wo, tile, rng, n_random)


def audit_conv(lay, w, bufs, mode, rng, tile=(8, 16), per_roi=None, n_random=256):
    p = lay.p
    xs = [np.asarray(bufs[k]) for k in lay.ins]
    x = xs[0]
    fc = x.ndim == 2 or p["fc"]
    if fc and not (x.ndim == 4 and x.shape[:2] == (1, 1)):   # FC input [r, k]; VGG's fc6 takes the flattened pool5 (h, w, c)
        x = xs[0] = x.reshape(1, 1, x.shape[0], -1)
    n, h, wd, _ = x.shape
    ho, wo, _, _ = conv_geometry(h, wd, p["k"], p["stride"], p["pad"])
    if fc:                                           # rows of an FC layer: sampled RoIs
        rows = sample_rois(wd, *(per_roi or (wd, 0)), rng=rng)
        pos = np.stack([np.zeros_like(rows), np.zeros_like(rows), rows], 1)
    else:
        pos = map_positions(n, ho, wo, tile, rng, n_random, per_roi)
    y64, bound, tiny = conv_ref(lay, w, xs, mode, pos)
    got = np.asarray(bufs[lay.key])
    if p["mean"]:
        hw = ho * wo
        rows = pos[::hw, 0]
        y = y64.reshape(len(rows), hw, -1)
        bd = bound.reshape(len(rows), hw, -1)
        m64 = y.mean(axis=1)
        # the device sums its own per-position values v, |v - y| <= bd: |mean - m64| <= mean(bd) + the spatial-mean bound
        # of v, which spatial_mean_ref's bound of |y| + bd majorises (both of its terms grow with |x|)
        _, smb = S.spatial_mean_ref((np.abs(y) + bd).reshape(len(rows), ho, wo, -1))
        mb = bd.mean(axis=1) + smb
        r, at = _check(lay.label, got[rows], m64, mb, lambda i: "RoI %d channel %d" % (rows[i[0]], i[1]))
    else:
        if fc:
            g = got.reshape(wd, -1)[pos[:, 2]]
        else:
            g = got[pos[:, 0], pos[:, 1], pos[:, 2]]
        r, at = _check(lay.label, g, y64, bound,
                       lambda i: "(n, h, w, c) = (%d, %d, %d, %d)" % (pos[i[0], 0], pos[i[0], 1], pos[i[0], 2], i[1]))
    return r, at, tiny


def audit_simt(lay, w, bufs):
    p = lay.p
    x = np.asarray(bufs[lay.ins[0]])
    n, h, wd, c = x.shape
    ho, wo, pt, pl = conv_geometry(h, wd, p["k"], p["stride"], p["pad"])
    if lay.kind == "depthwise":
        wt = np.asarray(w[p["name"] + "/depthwise_weights"], F).reshape(3, 3, c)
        w_oihw = wt.transpose(2, 0, 1)[:, None]
        groups, K = c, 9
    else:
        wt = np.asarray(w[p["name"] + "/weights"], F)
        w_oihw = wt.transpose(3, 2, 0, 1)
        groups, K = 1, wt.shape[0] * wt.shape[1] * wt.shape[2]
    inv, sh, dinv, dsh = bn64(w, p["name"], p["eps"])
    y64, bound = FR.fma_chain_ref(x, w_oihw, p["stride"], pt, pl, ho, wo, K, inv, sh, p["act"], groups)
    v = FR.conv64_nhwc(x, w_oihw, p["stride"], pt, pl, ho, wo, groups)
    bound = bound + np.abs(v) * dinv + dsh
    got = np.asarray(bufs[lay.key])
    return _check(lay.label, got, y64, bound, lambda i: "(n, h, w, c) = %s" % (tuple(int(v) for v in i),)) + (0,)


def audit_max_pool(lay, bufs):
    p = lay.p
    x = np.asarray(bufs[lay.ins[0]])
    ho, wo, pt, pl, neg = FR.pool_geometry(x.shape[1], x.shape[2], p["k"], p["stride"], p["mode"])
    want = FR.max_pool_model(x, p["k"], p["stride"], pt, pl, ho, wo, neg)
    return _exact(lay.label, np.asarray(bufs[lay.key]), want) + (0,)


def audit_spatial_mean(lay, bufs):
    m64, bound = S.spatial_mean_ref(np.asarray(bufs[lay.ins[0]]))
    return _check(lay.label, np.asarray(bufs[lay.key]), m64, bound, lambda i: "(RoI, c) = %s" % (tuple(int(v) for v in i),)) + (0,)


AuditRow = collections.namedtuple("AuditRow", "label kind ratio at tiny")


def audit(layers, w, bufs, mode=M.F16X3, plans=None, seed=0, n_random=256, tail=None):
    """Walk `layers` in order over the device outputs `bufs` (key -> numpy).  plans: key -> dict(tile=(th, tw), per_roi=
    (RoIs per image, RoIs per M tile, RoI count of every image) or None).  tail(layer, bufs) audits the kinds this module leaves to the caller (index
    work of the detection tail).  Returns one AuditRow per layer; raises Finding naming the first layer out of bound."""
    rng = np.random.default_rng(seed)
    rows = []
    for lay in layers:
        pl = (plans or {}).get(lay.key, {})
        if lay.kind == "conv":
            r = audit_conv(lay, w, bufs, mode, rng, pl.get("tile", (8, 16)), pl.get("per_roi"), n_random)
        elif lay.kind in ("conv_first", "depthwise"):
            r = audit_simt(lay, w, bufs)
        elif lay.kind == "max_pool":
            r = audit_max_pool(lay, bufs)
        elif lay.kind == "spatial_mean":
            r = audit_spatial_mean(lay, bufs)
        elif tail is not None:
            r = tail(lay, bufs)
        else:
            raise KeyError("no reference for layer kind %r (%s)" % (lay.kind, lay.label))
        rows.append(AuditRow(lay.label, lay.kind, r[0], r[1], r[2]))
    return rows


def worst_by_kind(rows):
    """{kind: AuditRow with the largest err / bound}."""
    out = {}
    for r in rows:
        k = r.kind if r.kind != "conv" else ("conv" + (":" + r.label.rsplit("/", 1)[-1] if "cls_bbox" in r.label or "rpn_heads" in r.label else ""))
        if k not in out or r.ratio > out[k].ratio:
            out[k] = r
    return out


# ---- a CPU stand-in of the device: conv_split_model + an fp32 epilogue -------------------------------------------------------
def fold32(w, name, eps):
    """TF's inference BatchNorm in fp32 (inv = gamma * rsqrt(var + eps), shift = beta - mean inv), as the device epilogue
    takes it; eps None: scale 1, the biases."""
    if eps is None:
        return None, np.asarray(w[name + "/biases"], F)
    p = name + "/BatchNorm/"
    g, be, mu, var = (np.asarray(w[p + k], F) for k in ("gamma", "beta", "moving_mean", "moving_variance"))
    inv = (g * (F(1) / np.sqrt(var + F(eps)))).astype(F)
    return inv, (be - mu * inv).astype(F)


def standin(layers, w, image, mode=M.F16X3, mutant=None, tile=(8, 16)):
    """Device outputs of the backbone and RPN convolutions of `layers` computed on the CPU: every tensor-core conv is
    conv_split_model.model (the device's operand roundings, float64 sums) with an fp32 epilogue, every SIMT conv the float64
    conv rounded to fp32 with its fp32 epilogue, max pool its model.  `mutant` = (kind, layer key) injects one wiring fault."""
    bufs = {"image": np.asarray(image, F)}
    mk, mkey = mutant if mutant else (None, None)
    keys = [l.key for l in layers]
    for lay in layers:
        p = lay.p
        xin = bufs[lay.ins[0]]
        if lay.kind == "max_pool":
            ho, wo, pt, pl, neg = FR.pool_geometry(xin.shape[1], xin.shape[2], p["k"], p["stride"], p["mode"])
            bufs[lay.key] = FR.max_pool_model(xin, p["k"], p["stride"], pt, pl, ho, wo, neg)
            continue
        eps = p.get("eps")
        if lay.key == mkey and mk == "eps":
            eps = 1e-3 if eps == 1e-5 else 1e-5
        n, h, wd, _ = xin.shape
        ho, wo, pt, pl = conv_geometry(h, wd, p["k"], p["stride"], p["pad"])
        if lay.key == mkey and mk == "pad":
            pt, pl = pt + 1, pl + 1
        if lay.kind == "conv_first":
            wt = np.asarray(w[p["name"] + "/weights"], F)
            sc, sh = fold32(w, p["name"], eps)
            v = M.conv64(xin, wt, p["stride"], pt, pl, ho, wo).astype(F)
            y = (v * (F(1) if sc is None else sc)).astype(F) + sh
            bufs[lay.key] = _act(y.astype(F), p["act"]).astype(F)
            continue
        if lay.kind != "conv":
            raise KeyError(lay.kind)
        if "fused" in p:
            q = dict(p)
            if lay.key == mkey and mk in ("cols+4", "cols-4"):     # the bbox part written 4 columns off
                d = 4 if mk == "cols+4" else -4
                q["fused"] = [q["fused"][0], (q["fused"][1][0], q["fused"][1][1] + d, q["fused"][1][2])]
                q["cout"] = p["cout"] + max(d, 0)
            wt, b = fused_weights(w, q)
            wt, sc, sh = wt[..., :p["cout"]], None, b[:p["cout"]].astype(F)
        elif len(p["parts"]) > 1:
            parts = [fold32(w, nm, eps) for nm in p["parts"]]
            wt = np.concatenate([(np.asarray(w[nm + "/weights"], F) * s).astype(F) for nm, (s, _) in zip(p["parts"], parts)], axis=2)
            wt, sc = R.pack_columns(wt)                                  # engine.concat_layers' packing
            sh = (parts[0][1] + parts[1][1]).astype(F)
        else:
            wt = np.asarray(w[p["name"] + "/weights"], F)
            sc, sh = fold32(w, p["name"], eps)
        x = xin
        if p["x2"] is not None:
            x2 = bufs[p["x2"]]
            if lay.key == mkey and mk == "swap":
                x, x2 = x2, x
            x = np.concatenate([x, x2], axis=3)
        if lay.key == mkey and mk == "kblock":
            x = x.copy()
            x[..., int(np.abs(x).sum(axis=(0, 1, 2)).argmax())] = 0      # the busiest input channel

        m, _ = M.model(x, wt, mode, p["stride"], pt, pl, ho, wo)
        acc = m.astype(F)
        y = acc if sc is None else (acc * sc).astype(F)
        shv = sh.copy()
        if lay.key == mkey and mk == "shift":
            shv[3] = 0
        y = (y + shv).astype(F)
        if p["residual"] is not None:
            rk = p["residual"]
            if lay.key == mkey and mk == "residual":      # the residual of the unit before
                rk = keys[keys.index(rk) - 3]
            y = (y + bufs[rk]).astype(F)
        y = _act(y, p["act"]).astype(F)
        if lay.key == mkey and mk == "seam":
            th, tw = tile
            v = y[0, min(th, ho - 1), min(tw, wo - 1)]
            v[int(np.abs(v).argmax())] *= F(1.01)
        bufs[lay.key] = y
    return bufs
