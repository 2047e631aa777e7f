"""The conv kernel (`conv_gemm_kernel`) at its padding edges, element by element in all three arithmetic modes.

Padding is not coded in the kernel: TMA zero-fills the part of a tap's A box that lies outside the map.  These tests pin
what any padding optimisation has to keep (tests/test_conv_pad_model.py holds the case list, its geometry predicates and
the comparator, and shows the comparator failing plausible padding mistakes):

1. maps smaller than the filter or the tile (1x1 .. 3x3 maps at 1 / 64 / 300 / 301 RoIs, 1 x 300 and 300 x 1 strips, the
   ResNet head's P = 7 and P = 14 RoI maps);
2. stride-2 padding rules: EXPLICIT (slim conv2d_same) and SAME on even and odd maps, 1x1 .. 3x3 maps, and the ResNet
   block1 / block2 strided convs at 600x1000 and 600x800, each asserting pad_t / pad_l as ops.conv_out_hw gives them;
3. taps straddling k-blocks: cin = 32 / 96 / 160 put a padding tap and a live tap in one 64-wide F16 k-block; cin = 512;
4. split-K where whole splits are padding: block4 conv2 (3x3x512 -> 512) on P = 1 / 2 maps, splits 2 / 3 / 8 and auto;
5. BatchNorm scale / shift + ReLU / ReLU6 on padding-heavy layers; outputs whose receptive field is all padding are
   act(shift) exactly;
6. no reads outside the tensor (the input inside a NaN-filled buffer), no leaks across RoI seams (every other RoI all NaN),
   and NaN / +-Inf / |x| >= 65536 at corners, edges next to padding and on both sides of RoI seams reaching exactly the
   outputs whose receptive field holds one;
7. raster m vs n bit-equal, block_n 64 vs 128 reported, on a padding-heavy RoI layer.

Criteria as in test_conv_gpu.py (u = 2^-24, S = sum |x||w| over the receptive field): (a) |got - model| <= BETA u S in
every mode, (b) |got - ref64| <= ALPHA u S in F16X3 and TF32X3; every output NaN-prefilled between sentinel guard bands,
inputs checked unchanged, two runs bit-equal, and the plan's geometry (frcnn_conv_plan_geometry at the device's SM count)
checked against its case's predicate and the plan's own report.

Observed on an H100 80 GB HBM3 (SXM, 700 W limit), worst err / (u S) over the modes, (a) / (b): small maps 1.02 / 1.21,
stride 2 0.80 / 1.23, straddling k-blocks 0.75 / 1.28, split-K 0.72 / 0.74, epilogue 1.08 / 1.24; NaN bytes around the
input 0.66 / 1.30, NaN RoIs 0.69 / 1.22, non-finite values 0.80 / 1.19, except TF32X3 with |x| up to 1e30 (one term then
dominates S and carries tf32x3's 2^-22 split error): 4.65.  Every all-padding output was exactly act(shift); block_n 64
and 128 gave the same bits on both raster layers.  About 30 seconds."""
import zlib

import numpy as np
import pytest
import torch

import conv_split_model as M
from test_conv_gpu import ALPHA, BETA, MODE_IDS, check_guards, dev, epilogue64, guarded, ratio, sm_count
from test_conv_pad_model import (PAD_CASES, case_ids, check_pad_outputs, layer, place_bad, plan_geometry,
                                 receptive_hits)

pytestmark = pytest.mark.gpu
F = np.float32
NAN_GUARD = 64                  # floats of NaN before and after the input in the out-of-tensor test (256 B: TMA alignment)
WORST = {}


@pytest.fixture(scope="module", autouse=True)
def report_worst():
    yield
    if WORST:
        print("\n[pad edges] worst err / (u S), (a) / (b):")
        for (group, mode), (ra, rb) in sorted(WORST.items()):
            print("  %-12s %-7s a=%.2f b=%s" % (group, mode, ra, "%.2f" % rb if rb is not None else "-"))


def note(group, mode, ra, rb=None):
    a, b = WORST.get((group, mode), (0.0, None))
    WORST[group, mode] = (max(a, ra), rb if b is None else (b if rb is None else max(b, rb)))


def run_pad(x, wt, impl, L, scale=None, shift=None, act=0, block_n=0, split_k=0, runs=2, nan_border=False):
    """One plan over layer L, `runs` runs: (outputs, geometry).  Guard bands, inputs unchanged (with nan_border the input
    sits between NaN-filled bytes, checked unchanged as well), plan report == frcnn_conv_plan_geometry."""
    from tf_faster_rcnn_b200 import ops
    pc = ops.PackedConv(wt, scale, shift, impl=impl)
    if nan_border:
        xbuf = torch.full((x.size + 2 * NAN_GUARD,), float("nan"), dtype=torch.float32, device="cuda")
        xbuf[NAN_GUARD:NAN_GUARD + x.size] = dev(x).view(-1)
        xd = xbuf[NAN_GUARD:NAN_GUARD + x.size].view(x.shape)
        before = xbuf.cpu().numpy().view(np.int32).copy()
    else:
        xd = dev(x)
    buf, out = guarded((L.n, L.ho, L.wo, L.cout))
    plan = ops.ConvPlan(xd, pc, out, L.stride, L.pt, L.pl, act, None, block_n, 0, split_k)
    outs = []
    for _ in range(runs):
        plan.run()
        torch.cuda.synchronize()
        outs.append(out.cpu().numpy().copy())
        check_guards(buf, out.numel())
    assert np.array_equal(xd.cpu().numpy().view(np.int32), x.view(np.int32)), "input modified"
    if nan_border:
        assert np.array_equal(xbuf.cpu().numpy().view(np.int32), before), "input buffer modified"
    for o in outs[1:]:
        assert np.array_equal(o.view(np.int32), outs[0].view(np.int32)), "two runs differ"
    info = plan.info()
    g = plan_geometry(L, impl, sm_count(), block_n, split_k)
    assert (info["block_n"], info["tile_n"], info["tile_h"], info["tile_w"], info["grid_m"], info["grid_n"]) == \
        (g["block_n"], g["tile_n"], g["tile_h"], g["tile_w"], g["m_tiles"], g["n_tiles"]), (info, g)
    assert info["splits"] == (g["splits"] if g["split_tiles"] > 0 else 1), (info, g)
    return outs, g


def data(seed, L):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((L.n, L.h, L.w, L.cin)).astype(F)
    wt = (rng.standard_normal((L.k, L.k, L.cin, L.cout)) * np.sqrt(2.0 / (L.k * L.k * L.cin))).astype(F)
    return rng, x, wt


_REF = {}


def refs(key, x, wt, L):
    """(ref64, S) of a case, computed once for the three modes."""
    if key not in _REF:
        if len(_REF) > 2:
            _REF.clear()
        _REF[key] = (M.conv64(x, wt, L.stride, L.pt, L.pl, L.ho, L.wo),
                     M.conv64(np.abs(x), np.abs(wt), L.stride, L.pt, L.pl, L.ho, L.wo))
    return _REF[key]


@pytest.mark.parametrize("mode", MODE_IDS)
@pytest.mark.parametrize("case", PAD_CASES, ids=case_ids(PAD_CASES))
def test_pad_edges_per_element(cuda, case, mode):
    group, name, shape, opt, covers = case
    impl = M.MODES[mode]
    L = layer(shape)
    rng, x, wt = data(zlib.crc32(name.encode()), L)
    act = opt.get("act", 0)
    scale = rng.uniform(0.5, 1.5, L.cout).astype(F) if "act" in opt else None
    shift = rng.standard_normal(L.cout).astype(F) if "act" in opt else None
    (got, _), g = run_pad(x, wt, impl, L, scale, shift, act, opt.get("block_n", 0), opt.get("split_k", 0))
    assert covers(g, impl, L), "%s no longer covers its path: %s %s" % (name, L, g)
    assert np.isfinite(got).all(), "non-finite output (unwritten rows?) %s" % g
    want64, s = refs(name, x, wt, L)
    mdl, _ = M.model(x, wt, impl, L.stride, L.pt, L.pl, L.ho, L.wo)
    y_m, sc, rnd_m = epilogue64(mdl, scale, shift, None, act)
    ra = ratio(got, y_m, s, sc, rnd_m)
    # (b) through the comparator: finiteness, the bound, all-padding outputs == act(shift) exactly
    rb = check_pad_outputs(got, x, wt, L, impl, "b", scale=scale, shift=shift, act=act, refs=(want64, s),
                           bound=np.inf if mode == "f16x1" else ALPHA)
    line = "[%s %s] a=%.2f b=%.2f geom=%s" % (name, mode, ra, rb, {k: g[k] for k in (
        "block_n", "tile_n", "tile_h", "tile_w", "tiles", "split_tiles", "splits", "kb_per_split", "k_blocks")})
    print("\n" + line)
    note(group, mode, ra, rb if mode != "f16x1" else None)
    assert ra <= BETA, line


# 6. ------------------------------------------------------------------------------------------------------------------
SEAM_LAYERS = [
    # name, (n, h, w, cin, cout, k, stride, pad)
    ("map1x1_n300", (300, 1, 1, 64, 64, 3, 1, "SAME")),
    ("map2x2_n64_cin32", (64, 2, 2, 32, 64, 3, 1, "SAME")),      # F16 k-blocks with one padding and one live tap
    ("map3x3_n64_cin96", (64, 3, 3, 96, 64, 3, 1, "SAME")),
    ("map2x2_n301", (301, 2, 2, 64, 64, 3, 1, "SAME")),           # RoIs straddle M tiles, last tile past the last RoI
    ("s2_even_explicit", (20, 6, 8, 64, 64, 3, 2, "EXPLICIT")),
    ("s2_even_same", (20, 6, 8, 64, 64, 3, 2, "SAME")),
    ("strip_h1_w300", (1, 1, 300, 64, 64, 3, 1, "SAME")),
]


def _crit(mode):
    return ("a", BETA) if mode == "f16x1" else ("b", ALPHA)


@pytest.mark.parametrize("mode", MODE_IDS)
@pytest.mark.parametrize("lay", SEAM_LAYERS, ids=[c[0] for c in SEAM_LAYERS])
def test_no_read_outside_the_tensor(cuda, lay, mode):
    """The input inside a buffer whose bytes before and after it are NaN: a padding tap never reads them."""
    name, shape = lay
    impl = M.MODES[mode]
    L = layer(shape)
    _, x, wt = data(zlib.crc32(("oob" + name).encode()), L)
    (got, _), g = run_pad(x, wt, impl, L, nan_border=True)
    crit, bound = _crit(mode)
    r = check_pad_outputs(got, x, wt, L, impl, crit, bound=bound)
    print("\n[outside %s %s] %s=%.2f" % (name, mode, crit, r))
    note("outside", mode, r if crit == "a" else 0.0, r if crit == "b" else None)


@pytest.mark.parametrize("mode", MODE_IDS)
@pytest.mark.parametrize("lay", SEAM_LAYERS[:5], ids=[c[0] for c in SEAM_LAYERS[:5]])
def test_nan_roi_does_not_leak(cuda, lay, mode):
    """Every pixel of every odd RoI is NaN: the even RoIs, which share M tiles with them, stay finite and in bound."""
    name, shape = lay
    impl = M.MODES[mode]
    L = layer(shape)
    _, x, wt = data(zlib.crc32(("leak" + name).encode()), L)
    g = plan_geometry(L, impl, sm_count())
    assert g["tile_n"] > 1, "RoI k and k + 1 no longer share an M tile: %s" % g
    bad = np.zeros(x.shape, bool)
    bad[1::2] = True
    xb = np.where(bad, F(np.nan), x)
    (got, _), _ = run_pad(xb, wt, impl, L)
    crit, bound = _crit(mode)
    r = check_pad_outputs(got, xb, wt, L, impl, crit, bad=bad, bound=bound)
    assert np.isfinite(got[0::2]).all() and not np.isfinite(got[1::2]).any()
    print("\n[leak %s %s] %s=%.2f" % (name, mode, crit, r))
    note("seams", mode, r if crit == "a" else 0.0, r if crit == "b" else None)


@pytest.mark.parametrize("mode", MODE_IDS)
@pytest.mark.parametrize("kind", ["nan", "inf", "big"])
@pytest.mark.parametrize("lay", SEAM_LAYERS, ids=[c[0] for c in SEAM_LAYERS])
def test_non_finite_next_to_padding_and_seams(cuda, lay, kind, mode):
    """NaN / +-Inf / |x| >= 65536 at map corners, at edge pixels next to padding, on the last pixel of RoI k and the first
    of RoI k + 1 (k inside an M tile and at its last RoI): exactly the outputs whose receptive field holds one are
    non-finite ('big' in TF32X3: finite and in bound), every other output in bound."""
    name, shape = lay
    impl = M.MODES[mode]
    L = layer(shape)
    rng, x, wt = data(zlib.crc32(("bad" + name).encode()), L)
    g = plan_geometry(L, impl, sm_count())
    tn = g["tile_n"]
    rois = sorted({0, min(tn // 2, L.n - 1), min(tn - 1, L.n - 1), L.n - 1})
    xb, bad = place_bad(x, L, rois, kind, impl, rng)
    (got, _), _ = run_pad(xb, wt, impl, L)
    crit, bound = _crit(mode)
    r = check_pad_outputs(got, xb, wt, L, impl, crit, bad=bad, bound=bound)
    hits = 0 if bad is None else int(receptive_hits(bad.any(-1), L).sum())
    print("\n[%s %s %s] non-finite outputs %d (%d pixels), %s=%.2f" % (kind, name, mode, (~np.isfinite(got)).sum(), hits,
                                                                      crit, r))
    assert bad is None or hits > 0
    note("non-finite", mode, r if crit == "a" else 0.0, r if crit == "b" else None)


# 7. ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["f16x3", "tf32x3"])
@pytest.mark.parametrize("shape", [(64, 2, 2, 128, 256, 3, 1, "SAME"), (300, 1, 1, 64, 256, 3, 1, "SAME")],
                         ids=["map2x2_n64", "map1x1_n300"])
def test_raster_order_and_block_n_on_padding_heavy_layers(cuda, shape, mode, monkeypatch):
    """FRCNN_CONV_RASTER m and n give the same bits; block_n 64 vs 128 reported."""
    impl = M.MODES[mode]
    L = layer(shape)
    _, x, wt = data(17, L)
    outs = {}
    for r in ("m", "n"):
        monkeypatch.setenv("FRCNN_CONV_RASTER", r)
        for bn in (64, 128):
            (o, _), g = run_pad(x, wt, impl, L, block_n=bn)
            assert g["n_tiles"] > 1 and g["block_n"] == bn and g["tile_n"] > 1, g
            outs[r, bn] = o
    monkeypatch.delenv("FRCNN_CONV_RASTER")
    for bn in (64, 128):
        assert np.array_equal(outs["m", bn].view(np.int32), outs["n", bn].view(np.int32)), bn
    same = np.array_equal(outs["m", 64].view(np.int32), outs["m", 128].view(np.int32))
    print("\n[%s %s] block_n 64 vs 128 bit-identical: %s (max diff %.3e)" % (
        "x".join(map(str, shape[:3])), mode, same, np.abs(outs["m", 64] - outs["m", 128]).max()))
