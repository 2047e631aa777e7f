"""The conv kernel's zero padding without a GPU: the case list of test_conv_pad_edges_gpu.py and the comparator its
non-finite and no-leak tests rely on.

`conv_gemm_kernel` never codes padding: a filter tap's A box {32 ch, tw*stride, th*stride, tn} starts at
(w0*stride + s - pad_l, h0*stride + r - pad_t) and TMA zero-fills whatever lies outside the map, per dimension, so the
padding of one RoI is never the neighbouring RoI's pixels.  A layer whose map is smaller than the filter, an EXPLICIT
stride-2 layer (slim conv2d_same: pad 1 before) on an even map, a 64-wide F16 k-block holding one padding and one live tap
(cin = 32), or a split-K range that is padding for some outputs: each is a place where skipping or reordering padding work
goes wrong.

* `PAD_CASES` names the plan path every case exists for; its `covers` predicates hold here under
  frcnn_conv_plan_geometry at 132 SMs (H100 SXM) in all three modes, so a change of decide_geometry that moves a case off
  its path fails without a GPU.
* `check_pad_outputs` is the per-element comparator: exactly the outputs whose receptive field (from pt / pl) holds a
  flagged input element are non-finite, every other output lies within criterion (b) (float64, ALPHA u S) or (a) (the split
  model, BETA u S), and an output whose receptive field is all padding equals act(shift) in fp32 exactly.  The split model
  (the device's operand roundings, float64 sums) passes it; one plausible padding mistake each, applied to the split
  model's operands, fails it: padding read as the clamped edge pixel, pad_t off by one (EXPLICIT computed as SAME at stride
  2 on an even map), the padding row read from the neighbouring RoI, a k-block dropped where its first tap is padding and
  its second live, and an all-padding output left unwritten."""
import ctypes as C
from collections import namedtuple

import numpy as np
import pytest

import conv_split_model as M
from test_conv_gpu import ALPHA, BETA, GEOM_KEYS, epilogue64, ratio
from tf_faster_rcnn_b200 import _native as N

F = np.float32
NAN_QUIET, NAN_DEVICE = np.int32(0x7fc00000).view(F), np.int32(0x7fffffff).view(F)   # numpy's NaN, the device's own

Layer = namedtuple("Layer", "n h w cin cout k stride pt pl ho wo")


def conv_out_hw(h, w, k, stride, mode):
    from tf_faster_rcnn_b200 import ops
    return ops.conv_out_hw(h, w, k, stride, mode)


def layer(shape):
    """Layer of a case's shape (n, h, w, cin, cout, k, stride, pad): pad is 'SAME', 'EXPLICIT' (ops.conv_out_hw) or an
    explicit (pt, pl, ho, wo)."""
    n, h, w, cin, cout, k, stride, pad = shape
    if isinstance(pad, str):
        ho, wo, pt, pl = conv_out_hw(h, w, k, stride, pad)
    else:
        pt, pl, ho, wo = pad
    return Layer(n, h, w, cin, cout, k, stride, pt, pl, ho, wo)


def plan_geometry(L, impl, sms, block_n=0, split_k=0):
    """frcnn_conv_plan_geometry of a layer: the decomposition the plan chooses on `sms` SMs."""
    d = N.ConvDesc(None, None, None, None, None, None, None, L.n, L.h, L.w, L.cin, L.cout, L.k, L.k, L.stride, L.pt, L.pl,
                   L.ho, L.wo, 0, block_n, 0, split_k, impl, 1.0)
    out = (C.c_int * 16)()
    N.check(N.lib().frcnn_conv_plan_geometry(C.byref(d), sms, out), "geometry")
    return dict(zip(GEOM_KEYS, list(out)))


# ---------------------------------------------------------------------------------------------------------------------
# Taps, k-blocks and splits of a layer (the K loop runs tap-major: K = (r, s, cin) flattened, 32 channels per A box)
def live_taps(L):
    """[k*k, ho, wo]: tap (r, s) of output (i, j) reads a pixel of the map (False: it reads padding)."""
    r, s = np.divmod(np.arange(L.k * L.k), L.k)
    ii = np.arange(L.ho)[None, :] * L.stride + r[:, None] - L.pt
    jj = np.arange(L.wo)[None, :] * L.stride + s[:, None] - L.pl
    return ((ii >= 0) & (ii < L.h))[:, :, None] & ((jj >= 0) & (jj < L.w))[:, None, :]


def all_padding(L):
    """[ho, wo]: outputs whose whole receptive field is padding."""
    return ~live_taps(L).any(0)


def kblock_taps(L, impl):
    """The filter taps each k-block reads: F16 modes 64 channels (two A boxes), TF32X3 32; the odd F16 tail's second box
    lies past the last channel (zero-filled) and reads no tap."""
    cc = L.cin // 32
    per = 1 if impl == M.TF32X3 else 2
    total = L.k * L.k * cc
    return [sorted({b // cc for b in range(kb * per, min(kb * per + per, total))}) for kb in range(-(-total // per))]


def mixed_kblocks(L, impl):
    """(k-block, output) pairs where the k-block holds a padding tap and a live one."""
    lv = live_taps(L)
    return int(sum(((lv[t].any(0)) & ~(lv[t].all(0))).sum() for t in kblock_taps(L, impl) if len(t) > 1))


def padding_splits(L, impl, g):
    """(split, output) pairs where every tap the split's K range reads is padding (0 when no tile is split)."""
    if g["split_tiles"] == 0:
        return 0
    lv, kbt = live_taps(L), kblock_taps(L, impl)
    cnt = 0
    for z in range(g["splits"]):
        taps = sorted({t for kb in kbt[z * g["kb_per_split"]:(z + 1) * g["kb_per_split"]] for t in kb})
        cnt += int((~lv[taps].any(0)).sum()) if taps else 0
    return cnt


def live_tap_cut_by_split(L, impl, g):
    """A split boundary falls inside the k-blocks of one tap."""
    if g["split_tiles"] == 0:
        return False
    kbt = kblock_taps(L, impl)
    return any(kbt[z * g["kb_per_split"] - 1][-1] == kbt[z * g["kb_per_split"]][0] for z in range(1, g["splits"]))


def runs_past(g, L):
    """The last RoI tile runs past the last RoI."""
    return g["tile_n"] > 1 and L.n % g["tile_n"] != 0


def whole_map_per_tile(g, L):
    return g["tile_h"] >= L.ho and g["tile_w"] >= L.wo


def pads_are(L, pt, pl, ho, wo):
    return (L.pt, L.pl, L.ho, L.wo) == (pt, pl, ho, wo)


# ---------------------------------------------------------------------------------------------------------------------
# group, name, (n, h, w, cin, cout, k, stride, pad), options, what the case covers (asserted on (geometry, impl, layer))
#   options: split_k / block_n (forced plan options), act (0 / 1 ReLU / 2 ReLU6: with it a BatchNorm scale and shift)
def _small(n, h, w):
    if n == 1:
        return lambda g, i, L: g["m_tiles"] == 1 and whole_map_per_tile(g, L) and g["split_tiles"] == g["tiles"]
    if n == 64:
        return lambda g, i, L: g["tile_n"] > 1 and whole_map_per_tile(g, L) and g["split_tiles"] == 0
    if n == 300:
        return lambda g, i, L: g["tile_n"] > 1 and whole_map_per_tile(g, L) and g["split_tiles"] == g["tiles"]
    return lambda g, i, L: runs_past(g, L)


PAD_CASES = []
# 1. maps smaller than the filter or the tile: 3x3 SAME stride 1.  RoI batches of 64 (whole tiles, forced unsplit), 300
#    (the auto split) and 301 (64 and 300 divide evenly into the plan's RoI tiles on the maps up to 2x2; 301 leaves the
#    last tile running past the last RoI on every map)
for _n in (1, 64, 300, 301):
    for _h, _w in ((1, 1), (1, 2), (2, 1), (2, 2), (3, 3)):
        PAD_CASES.append(("small_maps", "map%dx%d_n%d" % (_h, _w, _n), (_n, _h, _w, 64, 64, 3, 1, "SAME"),
                          {"split_k": 1} if _n == 64 else {}, _small(_n, _h, _w)))
PAD_CASES += [
    ("small_maps", "strip_h1_w300", (1, 1, 300, 64, 64, 3, 1, "SAME"), {},
     lambda g, i, L: g["tile_h"] == 1 and g["tiles_w"] > 1),                         # top and bottom taps all padding
    ("small_maps", "strip_h300_w1", (1, 300, 1, 64, 64, 3, 1, "SAME"), {},
     lambda g, i, L: g["tile_w"] == 1 and g["tiles_h"] > 1),                         # left and right taps all padding
    ("small_maps", "roi_p7_c512", (8, 7, 7, 512, 512, 3, 1, "SAME"), {},            # ResNet head 3x3 at P = 7
     lambda g, i, L: g["tile_n"] > 1 and whole_map_per_tile(g, L)),
    ("small_maps", "roi_p14", (64, 14, 14, 64, 64, 3, 1, "SAME"), {},               # crop P = 14: RoIs straddle M tiles
     lambda g, i, L: g["tile_n"] > 1 and g["tiles_h"] > 1 and g["tiles_w"] > 1 and g["split_tiles"] == 0),
]
# 2. stride-2 padding rules: EXPLICIT pads 1 before; SAME pads 0 before on even sizes, 1 on odd ones
for _nm, _n, _h, _w, _c, _pad, _want in [
        ("b1_600x1000_explicit", 1, 150, 250, 64, "EXPLICIT", (1, 1, 75, 125)),    # ResNet block1 unit 3 conv2
        ("b2_600x1000_explicit", 1, 75, 125, 128, "EXPLICIT", (1, 1, 38, 63)),     # ResNet block2 unit 4 conv2
        ("b1_600x800_explicit", 1, 150, 200, 64, "EXPLICIT", (1, 1, 75, 100)),
        ("b2_600x800_explicit", 1, 75, 100, 128, "EXPLICIT", (1, 1, 38, 50)),
        ("b1_600x1000_same", 1, 150, 250, 64, "SAME", (0, 0, 75, 125)),           # even: padding only bottom / right
        ("b2_600x800_same", 1, 75, 100, 128, "SAME", (1, 0, 38, 50)),             # odd h, even w
        ("even_explicit", 2, 6, 8, 64, "EXPLICIT", (1, 1, 3, 4)),
        ("even_same", 2, 6, 8, 64, "SAME", (0, 0, 3, 4)),
        ("odd_explicit", 1, 37, 51, 64, "EXPLICIT", (1, 1, 19, 26)),
        ("odd_same", 1, 37, 51, 64, "SAME", (1, 1, 19, 26)),
        ("map1x1_explicit", 64, 1, 1, 64, "EXPLICIT", (1, 1, 1, 1)),
        ("map1x1_same", 64, 1, 1, 64, "SAME", (1, 1, 1, 1)),
        ("map2x2_explicit", 64, 2, 2, 64, "EXPLICIT", (1, 1, 1, 1)),
        ("map2x2_same", 64, 2, 2, 64, "SAME", (0, 0, 1, 1)),
        ("map3x3_explicit", 64, 3, 3, 64, "EXPLICIT", (1, 1, 2, 2)),
        ("map3x3_same", 64, 3, 3, 64, "SAME", (1, 1, 2, 2))]:
    PAD_CASES.append(("stride2", "s2_" + _nm, (_n, _h, _w, _c, _c, 3, 2, _pad), {},
                      lambda g, i, L, _want=_want: pads_are(L, *_want)))
# 3. taps straddling k-blocks: cin = 32 / 96 / 160 put a padding tap and a live tap in one 64-wide F16 k-block on 1x1 and
#    2x2 maps; at the head width 512 every k-block lies inside one tap
for _cin in (32, 96, 160, 512):
    for _h in (1, 2):
        PAD_CASES.append(("kblocks", "cin%d_map%dx%d" % (_cin, _h, _h), (64, _h, _h, _cin, 64, 3, 1, "SAME"), {},
                          (lambda g, i, L: g["k_blocks"] == (9 * L.cin // 32 if i == M.TF32X3 else -(-9 * L.cin // 64))
                           and (i == M.TF32X3 or mixed_kblocks(L, i) > 0)) if _cin != 512 else
                          (lambda g, i, L: g["k_blocks"] == 9 * 512 // (32 if i == M.TF32X3 else 64)
                           and mixed_kblocks(L, i) == 0)))
# 4. split-K where whole splits are padding: block4 conv2 (3x3x512 -> 512) on P = 1 / P = 2 RoI maps
for _h in (1, 2):
    for _sk in (2, 3, 8):
        PAD_CASES.append(("splitk", "b4_map%dx%d_split%d" % (_h, _h, _sk), (64, _h, _h, 512, 512, 3, 1, "SAME"),
                          {"split_k": _sk, "act": 1} if _sk == 3 else {"split_k": _sk},
                          (lambda g, i, L, _sk=_sk: g["splits"] == _sk and g["split_tiles"] == g["tiles"]
                           and padding_splits(L, i, g) > 0) if _sk != 2 else
                          (lambda g, i, L: g["splits"] == 2 and g["split_tiles"] == g["tiles"]
                           and padding_splits(L, i, g) == 0 and live_tap_cut_by_split(L, i, g))))
PAD_CASES += [
    ("splitk", "b4_map2x2_n1_auto", (1, 2, 2, 512, 512, 3, 1, "SAME"), {},        # too small to fill the GPU: all split
     lambda g, i, L: g["split_tiles"] == g["tiles"] and g["splits"] >= 2 and padding_splits(L, i, g) > 0),
]
# 5. epilogue on padding-heavy layers: BatchNorm scale / shift + ReLU / ReLU6.  Padding beyond the filter (a 1x1 conv
#    padded by 1, a 3x3 conv padded by 3) leaves outputs whose receptive field is all padding: exactly act(shift)
PAD_CASES += [
    ("epilogue", "p1_bn_relu6", (64, 1, 1, 512, 128, 3, 1, "SAME"), {"act": 2, "split_k": 1},
     lambda g, i, L: g["split_tiles"] == 0),                                        # P = 1: 8 of 9 taps padding
    ("epilogue", "p2_bn_relu_split", (64, 2, 2, 256, 128, 3, 1, "SAME"), {"act": 1},
     lambda g, i, L: g["split_tiles"] == g["tiles"]),                               # tail_reduce epilogue
    ("epilogue", "allpad_pw_pad1_relu", (64, 1, 1, 64, 64, 1, 1, (1, 1, 3, 3)), {"act": 1},
     lambda g, i, L: all_padding(L).sum() == 8 and g["split_tiles"] == 0),
    ("epilogue", "allpad_pw_pad1_cout30_relu6", (64, 2, 2, 64, 30, 1, 1, (1, 1, 4, 4)), {"act": 2},
     lambda g, i, L: all_padding(L).sum() == 12 and L.cout % 4 != 0),               # scalar-tail epilogue
    ("epilogue", "allpad_c3_pad3_relu", (64, 2, 2, 64, 96, 3, 1, (3, 3, 6, 6)), {"act": 1, "split_k": 1},
     lambda g, i, L: all_padding(L).sum() == 20 and g["split_tiles"] == 0),
    ("epilogue", "allpad_c3_pad3_split3_relu6", (64, 2, 2, 64, 96, 3, 1, (3, 3, 6, 6)), {"act": 2, "split_k": 3},
     lambda g, i, L: all_padding(L).sum() == 20 and g["splits"] == 3 and padding_splits(L, i, g) > 0),
    ("epilogue", "allpad_c3_s2_pad3_relu", (8, 4, 4, 64, 64, 3, 2, (3, 3, 4, 4)), {"act": 1},
     lambda g, i, L: all_padding(L).sum() == 7),
]


def case_ids(cases):
    return [c[1] for c in cases]


IMPLS = {"f16x3": M.F16X3, "tf32x3": M.TF32X3, "f16x1": M.F16X1}


@pytest.mark.parametrize("mode", list(IMPLS))
@pytest.mark.parametrize("case", PAD_CASES, ids=case_ids(PAD_CASES))
def test_pad_cases_cover_their_paths(case, mode):
    group, name, shape, opt, covers = case
    L = layer(shape)
    g = plan_geometry(L, IMPLS[mode], 132, opt.get("block_n", 0), opt.get("split_k", 0))
    assert covers(g, IMPLS[mode], L), "%s no longer covers its path: %s %s" % (name, L, g)


def test_case_list_names_every_shape():
    """The shapes the padding work has to keep: P = 1 / 2 / 7 / 14 RoI maps, EXPLICIT stride 2 on even and odd maps, the
    F16 k-blocks that mix a padding and a live tap, splits that are all padding, all-padding outputs."""
    layers = {c[1]: layer(c[2]) for c in PAD_CASES}
    hw = {(L.h, L.w) for L in layers.values() if L.n > 1}
    assert {(1, 1), (2, 2), (7, 7), (14, 14)} <= hw
    ex = [L for nm, L in layers.items() if "explicit" in nm]
    assert any(L.h % 2 == 0 and L.w % 2 == 0 for L in ex) and any(L.h % 2 == 1 for L in ex)
    assert any(L.cin == 32 and mixed_kblocks(L, M.F16X3) > 0 for L in layers.values())
    assert sum(all_padding(L).any() for L in layers.values()) >= 5


# ---------------------------------------------------------------------------------------------------------------------
# The comparator
def receptive_hits(bad_pixels, L):
    """[n, ho, wo]: outputs whose receptive field (pt / pl, stride) holds a flagged pixel."""
    ind = bad_pixels.astype(np.float64)[..., None]
    return M.conv64(ind, np.ones((L.k, L.k, 1, 1)), L.stride, L.pt, L.pl, L.ho, L.wo)[..., 0] > 0


def act_shift(shift, act, cout):
    """act(shift) in fp32: what an output with an all-padding receptive field must be."""
    sh = np.zeros(cout, F) if shift is None else shift.astype(F)
    return np.maximum(sh, F(0)) if act == 1 else np.minimum(np.maximum(sh, F(0)), F(6)) if act == 2 else sh


def check_pad_outputs(got, x, wt, L, impl, crit="b", bad=None, scale=None, shift=None, act=0, refs=None, bound=None):
    """Per output element (see the module docstring); returns the worst err / (u S |scale|) over the finite outputs.

    bad:  bool mask of x's elements expected to make their outputs non-finite (None: none); they are zeroed for the bound.
    crit: 'b' float64 (refs = (ref64, S) of the zeroed x may be passed in), 'a' the split model of `impl`.
    bound: defaults to ALPHA for 'b', BETA for 'a'."""
    assert got.shape == (L.n, L.ho, L.wo, L.cout), got.shape
    bad_pix = np.zeros((L.n, L.h, L.w), bool) if bad is None else bad.any(-1)
    assert act == 0 or not bad_pix.any(), "ReLU / ReLU6 map NaN to a number: non-finite inputs are checked without them"
    hit = np.repeat(receptive_hits(bad_pix, L)[..., None], L.cout, axis=-1)
    nonfinite = ~np.isfinite(got)
    if not np.array_equal(nonfinite, hit):
        extra, missing = np.argwhere(nonfinite & ~hit), np.argwhere(hit & ~nonfinite)
        raise AssertionError("finite / non-finite pattern differs from the receptive fields: %d non-finite outside them "
                             "(first %s), %d finite inside (first %s)" % (len(extra), extra[:1].tolist(), len(missing),
                                                                       missing[:1].tolist()))
    xc = x if bad is None else np.where(bad, F(0), x)
    if crit == "a":
        want, s = M.model(xc, wt, impl, L.stride, L.pt, L.pl, L.ho, L.wo)
    elif refs is not None:
        want, s = refs
    else:
        want = M.conv64(xc, wt, L.stride, L.pt, L.pl, L.ho, L.wo)
        s = M.conv64(np.abs(xc), np.abs(wt), L.stride, L.pt, L.pl, L.ho, L.wo)
    y, sc, rnd = epilogue64(want, scale, shift, None, act)
    r = ratio(np.where(hit, y, got), y, s, sc, rnd)
    bound = (ALPHA if crit == "b" else BETA) if bound is None else bound
    if not r <= bound:
        raise AssertionError("err / (u S) = %.3g > %g" % (r, bound))
    pad_only = all_padding(L)
    if pad_only.any():
        exp = act_shift(shift, act, L.cout)
        sel = got[:, pad_only]                                      # [n, outputs, cout]
        if not (sel == exp).all():
            raise AssertionError("an all-padding output differs from act(shift): %d of %d" % ((sel != exp).sum(), sel.size))
    return r


# ---------------------------------------------------------------------------------------------------------------------
# The device's stand-in and the padding mistakes
def fp32_epilogue(v, scale, shift, act):
    y = v.astype(F)
    if scale is not None:
        y = (y * scale.astype(F)).astype(F)
    if shift is not None:
        y = (y + shift.astype(F)).astype(F)
    return np.maximum(y, F(0)) if act == 1 else np.minimum(np.maximum(y, F(0)), F(6)) if act == 2 else y


def stand_in(x, wt, L, impl, scale=None, shift=None, act=0):
    """The split model (the device's operand roundings, exact products, float64 sums), rounded to fp32, fp32 epilogue."""
    with np.errstate(invalid="ignore", over="ignore"):
        m, _ = M.model(x, wt, impl, L.stride, L.pt, L.pl, L.ho, L.wo)
    return fp32_epilogue(m, scale, shift, act)


def _tap_operand(x, L, r, s, read):
    """[n, ho, wo, cin] pixels tap (r, s) reads.  read: 'zero' (padding is 0), 'clamp' (padding reads the nearest edge pixel),
    'roi' (rows above / below the map come from the RoI before / after it: the batch read as one tall image)."""
    n, h, w = L.n, L.h, L.w
    ii = np.arange(L.ho) * L.stride + r - L.pt
    jj = np.arange(L.wo) * L.stride + s - L.pl
    okj = (jj >= 0) & (jj < w)
    jc = np.clip(jj, 0, w - 1)
    if read == "roi":
        rows = np.arange(n)[:, None] * h + ii[None, :]
        okr = (rows >= 0) & (rows < n * h)
        v = x.reshape(n * h, w, -1)[np.clip(rows, 0, n * h - 1)][:, :, jc]
        return np.where((okr[:, :, None] & okj[None, None, :])[..., None], v, 0.0)
    v = x[:, np.clip(ii, 0, h - 1)][:, :, jc]
    if read == "clamp":
        return v
    inside = ((ii >= 0) & (ii < h))[:, None] & okj[None, :]
    return np.where(inside[None, :, :, None], v, 0.0)


def tap_conv(x, w, L, read="zero", drop=None):
    """float64 convolution tap by tap; drop: [k*k, ho, wo] bool, the (tap, output) terms left out."""
    out = np.zeros((L.n, L.ho, L.wo, w.shape[3]))
    with np.errstate(invalid="ignore", over="ignore"):
        for t in range(L.k * L.k):
            r, s = divmod(t, L.k)
            term = np.einsum("nhwc,cd->nhwd", _tap_operand(x, L, r, s, read), w[r, s])
            if drop is not None:
                term = np.where(drop[t][None, :, :, None], 0.0, term)
            out += term
    return out


def dropped_second_taps(L, impl):
    """[k*k, ho, wo]: the live second tap of every k-block whose first tap is padding (a k-block skip that looked at its
    first tap only)."""
    lv = live_taps(L)
    drop = np.zeros_like(lv)
    for taps in kblock_taps(L, impl):
        if len(taps) == 2:
            drop[taps[1]] |= ~lv[taps[0]] & lv[taps[1]]
    return drop


def mutant(kind, x, wt, L, impl, scale=None, shift=None, act=0):
    """The stand-in with one padding mistake, on the split model's operands (hi + lo of x and w)."""
    xh, xl = M.split_activations(x, impl)
    wh, wl = M.split_weights(wt, impl)
    with np.errstate(invalid="ignore", over="ignore"):
        xs, ws = xh + xl, wh + wl
    if kind == "clamped_edge":
        v = tap_conv(xs, ws, L, "clamp")
    elif kind == "pad_t_off_by_one":
        ho, wo, pt, pl = conv_out_hw(L.h, L.w, L.k, L.stride, "SAME")
        assert (ho, wo) == (L.ho, L.wo) and (pt, pl) != (L.pt, L.pl)
        v = tap_conv(xs, ws, L._replace(pt=pt, pl=pl))
    elif kind == "neighbour_roi":
        v = tap_conv(xs, ws, L, "roi")
    elif kind == "dropped_kblock":
        drop = dropped_second_taps(L, impl)
        assert drop.any()
        v = tap_conv(xs, ws, L, drop=drop)
    elif kind == "unwritten_padding_output":
        y = stand_in(x, wt, L, impl, scale, shift, act)
        assert all_padding(L).any()
        y[:, all_padding(L)] = np.nan                                # the NaN prefill left in place
        return y
    else:
        raise ValueError(kind)
    return fp32_epilogue(v, scale, shift, act)


def place_bad(x, L, rois, kind, mode, rng):
    """Bad values at the corners and edge pixels of RoIs `rois` (next to padding), and on the last pixel of each RoI and
    the first pixel of the next: returns (x with them, bool element mask of those expected non-finite, or None)."""
    vals = {"nan": [NAN_QUIET, NAN_DEVICE, -NAN_DEVICE], "inf": [np.inf, -np.inf],
            "big": [65536.0, -1e5, 1e30]}[kind]
    x = x.copy()
    bad = np.zeros(x.shape, bool)
    places = []
    for b in rois:
        places += [(b, 0, 0), (b, L.h - 1, L.w - 1), (b, 0, L.w // 2), (b, L.h // 2, L.w - 1)]
        if b + 1 < L.n:
            places.append((b + 1, 0, 0))
    for q, (b, i, j) in enumerate(places):
        c = int(rng.integers(L.cin))
        x[b, i, j, c] = F(vals[q % len(vals)])
        bad[b, i, j, c] = True
    return x, (None if (kind == "big" and mode == M.TF32X3) else bad)


# the layers of the comparator's tests: each mistake shows on the layer it is paired with
MUTANT_LAYERS = {
    "clamped_edge": ((3, 2, 2, 64, 16, 3, 1, "SAME"), M.F16X3, {}),
    "pad_t_off_by_one": ((2, 6, 8, 64, 16, 3, 2, "EXPLICIT"), M.F16X3, {}),
    "neighbour_roi": ((6, 2, 2, 64, 16, 3, 1, "SAME"), M.TF32X3, {}),
    "dropped_kblock": ((4, 2, 2, 32, 16, 3, 1, "SAME"), M.F16X3, {}),
    "unwritten_padding_output": ((4, 1, 1, 64, 16, 1, 1, (1, 1, 3, 3)), M.F16X3, {"act": 1}),
}


def _mutant_data(kind):
    shape, impl, opt = MUTANT_LAYERS[kind]
    L = layer(shape)
    rng = np.random.default_rng(len(kind))
    x = rng.standard_normal((L.n, L.h, L.w, L.cin)).astype(F)
    wt = (rng.standard_normal((L.k, L.k, L.cin, L.cout)) * np.sqrt(2.0 / (L.k * L.k * L.cin))).astype(F)
    act = opt.get("act", 0)
    scale = rng.uniform(0.5, 1.5, L.cout).astype(F) if act else None
    shift = rng.standard_normal(L.cout).astype(F) if act else None
    return L, impl, rng, x, wt, scale, shift, act


@pytest.mark.parametrize("kind", list(MUTANT_LAYERS))
def test_stand_in_passes(kind):
    """The device's stand-in passes the comparator on each mistake's layer: clean, and (without an activation) with NaN /
    ±Inf / |x| >= 65536 next to padding and on both sides of every RoI seam; (a) and (b)."""
    L, impl, rng, x, wt, scale, shift, act = _mutant_data(kind)
    r = [check_pad_outputs(stand_in(x, wt, L, impl, scale, shift, act), x, wt, L, impl, crit, scale=scale, shift=shift,
                           act=act) for crit in ("a", "b")]
    if act == 0:
        for bk in ("nan", "inf", "big"):
            xb, bad = place_bad(x, L, range(L.n), bk, impl, rng)
            got = stand_in(xb, wt, L, impl)
            r.append(check_pad_outputs(got, xb, wt, L, impl, "b", bad=bad))
    print("\n[stand-in %s] worst err / (u S) %.2f" % (kind, max(r)))


@pytest.mark.parametrize("kind", list(MUTANT_LAYERS))
def test_padding_mistake_fails_the_comparator(kind):
    L, impl, rng, x, wt, scale, shift, act = _mutant_data(kind)
    xb, bad = (x, None) if act else place_bad(x, L, [0, L.n // 2], "nan", impl, rng)
    fails = []
    for data, b in ((x, None), (xb, bad)):
        got = mutant(kind, data, wt, L, impl, scale, shift, act)
        try:
            check_pad_outputs(got, data, wt, L, impl, "b", bad=b, scale=scale, shift=shift, act=act)
        except AssertionError as e:
            fails.append(str(e)[:110])
        else:
            fails.append(None)
    print("\n[mutant %s] clean: %s | with NaN: %s" % (kind, fails[0], fails[1]))
    assert fails[0] is not None, "%s passes the comparator" % kind
    # every mistake but the clamped edge also moves the non-finite pattern (on this layer NaN reaches every output there)
    assert kind == "clamped_edge" or fails[1] is not None, "%s passes the comparator with NaN inputs" % kind
