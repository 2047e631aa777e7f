"""The conv kernel's two ResNet fusions at their edges (`conv_gemm.cu`: the second A source, the mean epilogue).

Every case runs into a NaN-prefilled output between sentinel guard bands, checks that every input is unchanged and that
two runs are bit-equal.  u = 2^-24; S = sum |h2||W3 s3| + |x||Wsc ssc| per output element (tests/test_conv_fused.py).

* Folded scales: per-channel BatchNorm scales from 2^8 down to 2^-60, one of the two small or both, packed by
  engine.concat_layers.  F16X3 / TF32X3 per channel within the float64 bound of the unfused formula (test_conv_fused.py)
      |got - y64| <= (ALPHA + 2) u S + u |b3 + bsc| + 2 u |pre64|;
  F16X1 within BETA u S of its operand model (fused_ref64.folded_model).
* Second-source operand ranges: h2 and x at independent magnitudes 2^-24 .. 2^15; NaN / Inf / |x| >= 65536 in either
  source or both: exactly those pixel rows non-finite, in every channel (TF32X3: a large finite value stays finite and in
  bound); 65504 <= |x| < 65520 fp32-grade.
* Second-source geometry: seams inside a k-block, on k-block and chunk boundaries, source 2 holding the odd tail, split-K
  (auto on a ragged round, forced with the seam inside and on a split boundary, a short last split), every activation,
  residual with x2, raster order and block_n bit-exact.
* Mean epilogue: bit for bit the op-order model (fused_ref64.mean_model) applied to the same plan's unfused output, and
  within the composite float64 bound (the kernel's per-element bound averaged, plus stage_ref64's spatial-mean bound), over
  mean_hw 1 .. 1000, groups spanning 1 .. 8+ tiles, cout 4 .. 2052, both block_n, every activation, residual and x2 on / off,
  persistent units > grid; non-finite values reach only their group's channels, sums near 3e37 overflow to +Inf, ReLU maps
  NaN to 0.

Observed on an H100 80 GB HBM3 (700 W limit), max err / bound: folded scales 0.19 in each mode, on every channel.  With
the whole-matrix packing this replaced (W' packed as it is, epilogue scale 1), F16X3 failed every channel whose two scales
were both 2^-24 or smaller: 3.9 at 2^-24, 61 at 2^-28, 932 at 2^-32, 1.8e4 at 2^-36, up to 5.9e5; TF32X3 passed.
Magnitudes 0.28 against the model, 0.38 against float64; just below the f16 overflow 0.26; seams 0.28; split-K 0.21;
activations and residual 0.24.  Mean epilogue: bit-equal to the model in every case; composite bound 0.28 (hw 7), 0.058
(hw 49), 0.003 (hw 1000).  About a minute in all."""
import ctypes as C
import zlib

import numpy as np
import pytest
import torch

import conv_split_model as M
import fused_ref64 as R
import stage_ref64 as S

pytestmark = pytest.mark.gpu
F = np.float32
U = M.U
ALPHA = 8.0
BETA = 8.0
BETA_SUBNORMAL = 32.0          # (a) where f16 operands are subnormal (tests/test_conv_gpu.py)
NAN_QUIET, NAN_DEVICE = np.int32(0x7fc00000).view(F), np.int32(0x7fffffff).view(F)


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def run_checked(plan, buf, out, inputs):
    """Two runs: guard bands intact, bit-equal outputs, inputs (device, host) unchanged -> the output."""
    outs = []
    for _ in range(2):
        plan.run()
        torch.cuda.synchronize()
        outs.append(out.cpu().numpy().copy())
        S.check_guarded(buf, out.numel())
    assert np.array_equal(outs[0].view(np.int32), outs[1].view(np.int32)), "two runs differ"
    for d, h in inputs:
        if d is not None:
            assert np.array_equal(d.cpu().numpy().view(np.int32), np.asarray(h, F).view(np.int32)), "input modified"
    return outs[0]


def folded_unit(rng, cin, cin2, cout, s3, ssc):
    """A projection unit's conv3 + shortcut with folded scales s3 / ssc: (packed w, sigma, shift, parts) where parts holds
    the fp32 arrays of the unfused formula (w3, s3, b3, wsc, ssc, bsc)."""
    from tf_faster_rcnn_b200 import engine
    t = R.BNStore()
    R.bn_layer(rng, t, "u/conv3", cin, cout, np.broadcast_to(s3, (cout,)), wstd=np.sqrt(2.0 / cin))
    R.bn_layer(rng, t, "u/shortcut", cin2, cout, np.broadcast_to(ssc, (cout,)), wstd=np.sqrt(2.0 / cin2))
    w, sigma, shift = engine.concat_layers(t, ["u/conv3", "u/shortcut"], 1e-5)
    a3, b3 = t.scale_shift("u/conv3", 1e-5)
    asc, bsc = t.scale_shift("u/shortcut", 1e-5)
    return w, sigma, shift, (t["u/conv3/weights"], a3, b3, t["u/shortcut/weights"], asc, bsc)


def run_concat(h2, x, w, sigma, shift, impl, act=0, res=None, block_n=0, split_k=0, kb_per_chunk=0):
    from tf_faster_rcnn_b200 import ops
    n, h, wd, _ = h2.shape
    cout = w.shape[-1]
    pc = ops.PackedConv(w, sigma, shift, impl=impl)
    hd, xd = dev(h2), dev(x)
    rd = None if res is None else dev(res)
    buf, out = S.guarded_out((n, h, wd, cout))
    plan = ops.ConvPlan(hd, pc, out, 1, 0, 0, act, rd, block_n, kb_per_chunk, split_k, x2=xd)
    got = run_checked(plan, buf, out, [(hd, h2), (xd, x), (rd, res)])
    return got, plan.info()


def act64(v, act):
    return v if act == 0 else np.maximum(v, 0) if act == 1 else np.minimum(np.maximum(v, 0), 6)


def unfused64(h2, x, parts, res=None, act=0):
    """(y64, bound (b), S): the float64 unfused formula act((h2.W3) s3 + b3 + (x.Wsc) ssc + bsc (+ res)) and its bound."""
    w3, a3, b3, wsc, asc, bsc = parts
    n, h, wd, _ = h2.shape
    c64 = lambda a, b: M.conv64(a, b, 1, 0, 0, h, wd)
    d = lambda v: np.asarray(v, np.float64)
    pre = c64(h2, w3) * d(a3) + d(b3) + c64(x, wsc) * d(asc) + d(bsc)
    s = c64(np.abs(d(h2)), np.abs(d(w3) * d(a3))) + c64(np.abs(d(x)), np.abs(d(wsc) * d(asc)))
    c = pre if res is None else pre + d(res)
    bound = (ALPHA + 2) * U * s + U * np.abs(d(b3) + d(bsc)) + 2 * U * (np.abs(pre) + np.abs(c))
    return act64(c, act), bound, s


def model64(h2, x, w, sigma, shift, impl, res=None, act=0, beta=BETA):
    """(y, bound (a)) of the operand model on the packed matrix, with the epilogue's roundings."""
    m, s = R.folded_model(np.concatenate([h2, x], axis=3), w, sigma, impl)
    b = m + shift.astype(np.float64)
    c = b if res is None else b + res.astype(np.float64)
    return act64(c, act), beta * U * s + 2 * U * (np.abs(b) + np.abs(c))


# ---- folded scales ----------------------------------------------------------------------------------------------------
FOLD_EXP = [8, 4, 0, -4, -8, -16, -24, -28, -32, -36, -40, -48, -56, -60]


def fold_scales():
    """(s3, ssc, label) per output channel: both small, conv3's alone, the shortcut's alone."""
    e = np.asarray(FOLD_EXP, np.float64)
    one = np.ones_like(e)
    s3 = np.concatenate([2.0 ** e, 2.0 ** e, one])
    ssc = np.concatenate([2.0 ** e, one, 2.0 ** e])
    labels = ["both 2^%d" % v for v in FOLD_EXP] + ["s3 2^%d" % v for v in FOLD_EXP] + ["ssc 2^%d" % v for v in FOLD_EXP]
    # two more channels at scale 1: cout % 4 == 0, the vectorised epilogue of the production layers
    return np.append(s3, [1, 1]), np.append(ssc, [1, 1]), labels + ["one", "one"]


@pytest.mark.parametrize("mode", ["f16x3", "tf32x3", "f16x1"])
def test_folded_scales_per_channel(cuda, mode):
    """Every channel within its bound; the whole-matrix packing failed F16X3 from both scales 2^-24 on (module docstring:
    the matrix's largest weight sits in the 2^8 channel, so 2^-24 lies 32 binades below it)."""
    impl = M.MODES[mode]
    rng = np.random.default_rng(101)
    s3, ssc, labels = fold_scales()
    cout = len(labels)
    h2 = np.abs(rng.standard_normal((2, 9, 15, 64))).astype(F)
    x = rng.standard_normal((2, 9, 15, 96)).astype(F)
    w, sigma, shift, parts = folded_unit(rng, 64, 96, cout, s3, ssc)
    got, _ = run_concat(h2, x, w, sigma, shift, impl)
    if mode == "f16x1":
        want, bound = model64(h2, x, w, sigma, shift, impl)
    else:
        want, bound, _ = unfused64(h2, x, parts)
    err = np.abs(got.astype(np.float64) - want)
    per = (err / bound).reshape(-1, cout).max(axis=0)
    print("\n[folded %s] err/bound per channel: %s" % (mode, " ".join("%s=%.3g" % (l, v) for l, v in zip(labels, per))))
    bad = [l for l, v in zip(labels, per) if not v <= 1.0]
    assert np.isfinite(got).all() and not bad, "channels outside the bound: %s (max %.3g)" % (bad, per.max())


# ---- second-source operand ranges -------------------------------------------------------------------------------------
MAG_EXP = [-24, -14, 0, 14, 15]


def at_magnitude(rng, shape, e):
    """|v| in [2^e, 2^(e+1)) with random signs, capped at 65504 (the largest finite fp16)."""
    v = np.minimum(2.0 ** e * rng.uniform(1, 2, shape), 65504.0) * np.sign(rng.standard_normal(shape))
    return v.astype(F)


@pytest.mark.parametrize("mode", ["f16x3", "tf32x3", "f16x1"])
def test_second_source_magnitudes(cuda, mode):
    """h2 at 2^e1 and x at 2^e2, independently.  (a) against the model everywhere (BETA_SUBNORMAL where an f16 operand is
    subnormal); (b) against float64 in F16X3 where both lie in [2^-14, 65520), in TF32X3 always."""
    impl = M.MODES[mode]
    rng = np.random.default_rng(103)
    w, sigma, shift, parts = folded_unit(rng, 64, 64, 64, rng.uniform(0.3, 1.5, 64), rng.uniform(0.3, 1.5, 64))
    worst_a = worst_b = 0.0
    for e1 in MAG_EXP:
        for e2 in MAG_EXP:
            h2 = at_magnitude(rng, (1, 8, 16, 64), e1)
            x = at_magnitude(rng, (1, 8, 16, 64), e2)
            got, _ = run_concat(h2, x, w, sigma, shift, impl)
            sub = impl != M.TF32X3 and min(e1, e2) < -14
            want, bound = model64(h2, x, w, sigma, shift, impl, beta=BETA_SUBNORMAL if sub else BETA)
            worst_a = max(worst_a, S.check_bounded(got, want, bound, "(a) %s h2 2^%d x 2^%d" % (mode, e1, e2)))
            if mode == "tf32x3" or (mode == "f16x3" and not sub):
                want, bound, _ = unfused64(h2, x, parts)
                worst_b = max(worst_b, S.check_bounded(got, want, bound, "(b) %s h2 2^%d x 2^%d" % (mode, e1, e2)))
    print("\n[magnitudes %s] max err/bound (a) %.3f (b) %.3f" % (mode, worst_a, worst_b))


BAD = {"nan": [NAN_QUIET, NAN_DEVICE, -NAN_DEVICE], "inf": [np.inf, -np.inf, np.inf], "big": [65536.0, -1e5, 1e30]}


@pytest.mark.parametrize("where", ["src1", "src2", "both"])
@pytest.mark.parametrize("bad", ["nan", "inf", "big"])
@pytest.mark.parametrize("mode", ["f16x3", "tf32x3", "f16x1"])
def test_second_source_non_finite(cuda, mode, bad, where):
    """Bad values at three pixels (first row, a tile seam, the last row) of source 1, source 2, or both at one pixel:
    exactly those pixel rows are non-finite, in every channel; every other row meets (b) ((a) for F16X1).  'big' (finite
    |x| >= 65536) is non-finite in the f16 modes and finite and within (b) in TF32X3."""
    impl = M.MODES[mode]
    rng = np.random.default_rng(zlib.crc32((mode + bad + where).encode()))
    n, h, wd, cin, cin2, cout = 2, 9, 15, 64, 96, 68
    h2 = rng.standard_normal((n, h, wd, cin)).astype(F)
    x = rng.standard_normal((n, h, wd, cin2)).astype(F)
    w, sigma, shift, parts = folded_unit(rng, cin, cin2, cout, rng.uniform(0.3, 1.5, cout), rng.uniform(0.3, 1.5, cout))
    P = n * h * wd
    rows = [0, 128, P - 1] if where != "both" else [131]
    h2f, xf = h2.reshape(P, cin), x.reshape(P, cin2)
    h2c, xc = h2.copy(), x.copy()
    for i, (r, v) in enumerate(zip(rows, BAD[bad])):
        for src, clean, cdim in ((h2f, h2c.reshape(P, cin), cin), (xf, xc.reshape(P, cin2), cin2)):
            if where == "both" or (where == "src1") == (src is h2f):
                c = (7 * i + 3) % cdim
                src[r, c] = F(v)
                clean[r, c] = 0.0
    got, _ = run_concat(h2, x, w, sigma, shift, impl)
    expect = np.zeros(P, bool)
    if not (bad == "big" and mode == "tf32x3"):
        expect[rows] = True
    nonfin = ~np.isfinite(got.reshape(P, cout))
    assert np.array_equal(nonfin, np.repeat(expect[:, None], cout, axis=1)), \
        "non-finite rows %s, want rows %s in every channel" % (np.flatnonzero(nonfin.any(axis=1)), np.flatnonzero(expect))
    keep = ~np.repeat(expect[:, None], cout, axis=1).reshape(got.shape)
    hh, xx = (h2, x) if not expect.any() else (h2c, xc)
    if mode == "f16x1":
        want, bound = model64(hh, xx, w, sigma, shift, impl)
    else:
        want, bound, _ = unfused64(hh, xx, parts)
    S.check_bounded(got[keep], want[keep], bound[keep], "%s %s %s" % (mode, bad, where))


def test_second_source_just_below_f16_overflow(cuda):
    """65504 <= |x| < 65520 rounds to a finite fp16 hi: F16X3 stays within (b) with such values in both sources."""
    rng = np.random.default_rng(107)
    h2 = rng.standard_normal((1, 8, 16, 64)).astype(F)
    x = rng.standard_normal((1, 8, 16, 96)).astype(F)
    h2[0, 3, 3, :8] = F(65519.0) * np.sign(rng.standard_normal(8)).astype(F)
    x[0, 5, 7, :8] = F(65504.0)
    x[0, 3, 3, 8:16] = F(-65519.0)
    w, sigma, shift, parts = folded_unit(rng, 64, 96, 64, rng.uniform(0.3, 1.5, 64), rng.uniform(0.3, 1.5, 64))
    got, _ = run_concat(h2, x, w, sigma, shift, M.F16X3)
    want, bound, _ = unfused64(h2, x, parts)
    print("\n[below overflow] max err/bound %.3f" % S.check_bounded(got, want, bound, "65504..65519"))


# ---- second-source geometry -------------------------------------------------------------------------------------------
KEYS = ["block_n", "tile_n", "tile_h", "tile_w", "m_tiles", "n_tiles", "tiles", "split_tiles", "splits", "kb_per_split",
        "units", "grid", "k_blocks", "kb_per_chunk", "tiles_h", "tiles_w"]


def geom(n, h, w, cin, cout, cin2=0, block_n=0, split_k=0, impl=0, mean_hw=0):
    """frcnn_conv_plan_geometry of a pointwise layer at the device's SM count -> (rc, decomposition)."""
    from tf_faster_rcnn_b200 import _native as N
    d = N.ConvDesc(None, None, None, None, None, None, None, n, h, w, cin, cout, 1, 1, 1, 0, 0, h, w, 0, block_n, 0,
                   split_k, impl, 1.0, None, cin2, None, mean_hw)
    out = (C.c_int * 16)()
    rc = N.lib().frcnn_conv_plan_geometry(C.byref(d), torch.cuda.get_device_properties(0).multi_processor_count, out)
    return rc, dict(zip(KEYS, list(out)))


def concat_case(mode, name, shape, act=0, residual=False, block_n=0, split_k=0, kb_per_chunk=0, seed=None):
    """One fused conv against (b) ((a) for F16X1) -> (got, info, geometry, max err / bound)."""
    impl = M.MODES[mode]
    n, h, wd, cin, cin2, cout = shape
    rng = np.random.default_rng(zlib.crc32(name.encode()) if seed is None else seed)
    h2 = np.abs(rng.standard_normal((n, h, wd, cin))).astype(F)
    x = rng.standard_normal((n, h, wd, cin2)).astype(F)
    res = rng.standard_normal((n, h, wd, cout)).astype(F) * 3 if residual else None
    w, sigma, shift, parts = folded_unit(rng, cin, cin2, cout, rng.uniform(0.3, 1.5, cout), rng.uniform(0.3, 1.5, cout))
    got, info = run_concat(h2, x, w, sigma, shift, impl, act, res, block_n, split_k, kb_per_chunk)
    rc, g = geom(n, h, wd, cin, cout, cin2, block_n, split_k, impl)
    assert rc == 0 and info["block_n"] == g["block_n"] and info["splits"] == (g["splits"] if g["split_tiles"] else 1), (info, g)
    assert g["k_blocks"] == -(-(cin + cin2) // (32 if impl == M.TF32X3 else 64))
    if mode == "f16x1":
        want, bound = model64(h2, x, w, sigma, shift, impl, res, act)
    else:
        want, bound, _ = unfused64(h2, x, parts, res, act)
    r = S.check_bounded(got, want, bound, "%s %s" % (name, mode))
    return got, info, g, r


SEAM_CIN = [32, 64, 96, 512]
SEAM_CIN2 = [32, 96, 1024, 2048]


@pytest.mark.parametrize("mode", ["f16x3", "tf32x3", "f16x1"])
def test_second_source_seams(cuda, mode):
    """cin x cin2: the seam inside a 64-wide k-block (cin 32, 96), on a k-block boundary (64) and on a chunk boundary (512);
    source 2 holds the f16 modes' odd tail when cin2 / 32 is odd; kb_per_chunk 1 / 2 / 8 in turn."""
    worst = 0.0
    for i, cin in enumerate(SEAM_CIN):
        for j, cin2 in enumerate(SEAM_CIN2):
            kpc = (1, 2, 8)[(i + j) % 3]
            _, _, _, r = concat_case(mode, "seam%d_%d" % (cin, cin2), (1, 9, 30, cin, cin2, 64), kb_per_chunk=kpc)
            worst = max(worst, r)
    print("\n[seams %s] max err/bound %.3f" % (mode, worst))


@pytest.mark.parametrize("mode", ["f16x3", "tf32x3", "f16x1"])
def test_second_source_split_k(cuda, mode):
    """Auto split-K of a ragged last round (asserted split), forced splits with the seam (k = 512) on a split boundary
    (3 splits) and inside a split with a short last one (5 splits)."""
    impl = M.MODES[mode]
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    # tiles = m_tiles * 2 just past a multiple of the SM count: a ragged round of 4 tiles
    m_tiles = (sms + 4) // 2 + (sms + 4) % 2
    n = m_tiles * 128 // 64
    _, info, g, r0 = concat_case(mode, "auto_ragged", (n, 8, 8, 512, 1024, 256), block_n=128)
    assert g["split_tiles"] > 0 and g["splits"] > 1 and info["splits"] == g["splits"], (info, g)
    kb = 64 if impl != M.TF32X3 else 32
    _, _, g3, r3 = concat_case(mode, "forced3", (1, 9, 30, 512, 1024, 128), split_k=3)
    assert g3["splits"] == 3 and (g3["kb_per_split"] * kb) == 512, g3                  # seam on the first split boundary
    _, _, g5, r5 = concat_case(mode, "forced5", (1, 9, 30, 512, 1024, 128), split_k=5)
    assert g5["splits"] == 5 and 512 % (g5["kb_per_split"] * kb) != 0, g5              # seam inside a split
    assert g5["k_blocks"] - 4 * g5["kb_per_split"] < g5["kb_per_split"], g5           # a short last split
    print("\n[split %s] auto (%d splits) %.3f, forced 3 %.3f, forced 5 %.3f" % (mode, g["splits"], r0, r3, r5))


@pytest.mark.parametrize("mode", ["f16x3", "tf32x3", "f16x1"])
def test_second_source_epilogues(cuda, mode):
    """ACT_NONE and RELU6, and a residual together with x2 (every activation), at both block_n."""
    worst = 0.0
    for act in (0, 1, 2):
        for residual in (False, True):
            for bn in (64, 128):
                _, info, _, r = concat_case(mode, "epi%d%d%d" % (act, residual, bn), (2, 9, 15, 64, 96, 192), act, residual, bn)
                assert info["block_n"] == bn
                worst = max(worst, r)
    print("\n[epilogues %s] max err/bound %.3f" % (mode, worst))


@pytest.mark.parametrize("mode", ["f16x3", "tf32x3", "f16x1"])
def test_second_source_raster_and_block_n_bit_exact(cuda, mode, monkeypatch):
    """FRCNN_CONV_RASTER m / n and block_n 64 / 128 change the tile walk, not any element's arithmetic: bit-equal outputs."""
    shape = (3, 14, 40, 96, 96, 320)
    outs = {}
    for raster in ("m", "n"):
        monkeypatch.setenv("FRCNN_CONV_RASTER", raster)
        for bn in (64, 128):
            outs[(raster, bn)], _, _, _ = concat_case(mode, "raster", shape, 1, True, bn, split_k=1, seed=109)
    ref = outs[("m", 64)]
    for k, v in outs.items():
        assert np.array_equal(v.view(np.int32), ref.view(np.int32)), "%s differs from raster m, block_n 64" % (k,)


# ---- mean epilogue ----------------------------------------------------------------------------------------------------
def mean_run(x, x2, wt, scale, shift, res, act, impl, block_n):
    """(mean output, unfused output, plan info): the same plan with and without the mean, never split."""
    from tf_faster_rcnn_b200 import ops
    r, side_h, side_w, _ = x.shape
    cout = wt.shape[-1]
    pc = ops.PackedConv(wt, scale, shift, impl=impl)
    xd, rd = dev(x), None if res is None else dev(res)
    x2d = None if x2 is None else dev(x2)
    ins = [(xd, x), (rd, res), (x2d, x2)]
    fbuf, full = S.guarded_out((r, side_h, side_w, cout))
    y = run_checked(ops.ConvPlan(xd, pc, full, 1, 0, 0, act, rd, block_n, 0, 1, x2=x2d), fbuf, full, ins)
    buf, out = S.guarded_out((r, cout))
    plan = ops.ConvPlan(xd, pc, out, 1, 0, 0, act, rd, block_n, 0, 0, x2=x2d, mean=True)
    got = run_checked(plan, buf, out, ins)
    return got, y, plan.info()


def mean_composite64(x, x2, wt, scale, shift, res, act, impl, y_dev):
    """(float64 mean of the whole formula, composite bound): the per-element bound of the conv + epilogue ((b), or (a)
    around the operand model for F16X1) averaged over the group, plus the spatial-mean bound of the summed values."""
    r, sh, sw, _ = x.shape
    hw = sh * sw
    xc = x if x2 is None else np.concatenate([x, x2], axis=3)
    if impl == M.F16X1:
        v, s = M.model(xc, wt, impl, 1, 0, 0, sh, sw)
        k = BETA
    else:
        v = M.conv64(xc, wt.astype(np.float64), 1, 0, 0, sh, sw)
        s = M.conv64(np.abs(xc.astype(np.float64)), np.abs(wt.astype(np.float64)), 1, 0, 0, sh, sw)
        k = ALPHA
    sc = np.abs(scale.astype(np.float64))
    a = v * scale.astype(np.float64)
    b = a + shift.astype(np.float64)
    c = b if res is None else b + res.astype(np.float64)
    elem = k * U * s * sc + 2 * U * (np.abs(a) + np.abs(b) + np.abs(c))
    y64 = act64(c, act)
    m64 = y64.reshape(r, hw, -1).mean(axis=1)
    _, smb = S.spatial_mean_ref(y_dev)
    return m64, smb + elem.reshape(r, hw, -1).mean(axis=1)


# (groups, hw) with the rotating options of each: cout, block_n, act, residual, x2, mode
MEAN_CASES = [
    ((300, 1), [(60, 64, 0, True, False, "f16x3"), (4, 128, 1, False, True, "tf32x3")]),
    ((200, 2), [(68, 128, 2, True, True, "f16x1"), (192, 64, 0, False, False, "f16x3")]),
    ((97, 3), [(192, 128, 1, True, False, "tf32x3"), (60, 64, 2, False, True, "f16x3")]),
    ((61, 7), [(4, 64, 0, True, True, "f16x3"), (68, 128, 1, True, False, "f16x1")]),
    ((300, 49), [(192, 128, 1, True, True, "f16x3"), (68, 64, 0, True, False, "tf32x3"), (60, 128, 2, False, False, "f16x1")]),
    ((5, 49), [(2052, 128, 0, True, True, "f16x3"), (2052, 64, 1, True, False, "tf32x3")]),
    ((2, 64), [(60, 128, 0, False, True, "tf32x3"), (192, 64, 2, True, False, "f16x3")]),
    ((3, 127), [(68, 64, 1, True, True, "f16x3"), (4, 128, 0, True, False, "f16x1")]),
    ((2, 128), [(192, 128, 2, True, False, "f16x3"), (60, 64, 0, False, True, "tf32x3")]),
    ((3, 129), [(4, 64, 1, True, False, "tf32x3"), (68, 128, 0, True, True, "f16x3")]),
    ((5, 196), [(2052, 64, 2, True, True, "f16x3"), (192, 128, 0, True, False, "f16x1")]),
    ((3, 300), [(60, 128, 1, True, True, "f16x3"), (68, 64, 0, True, False, "tf32x3")]),
    ((2, 1000), [(192, 64, 0, True, True, "f16x3"), (4, 128, 1, False, False, "tf32x3")]),
    ((1, 7), [(60, 64, 0, True, True, "f16x3"), (68, 128, 1, False, False, "tf32x3")]),
]


def mean_inputs(rng, g, hw, cout, residual, with_x2, data="normal"):
    x = rng.standard_normal((g, hw, 1, 64)).astype(F)
    x2 = rng.standard_normal((g, hw, 1, 96)).astype(F) if with_x2 else None
    k = 64 + (96 if with_x2 else 0)
    wt = (rng.standard_normal((1, 1, k, cout)) * np.sqrt(2.0 / k)).astype(F)
    scale, shift = rng.uniform(0.5, 1.5, cout).astype(F), rng.standard_normal(cout).astype(F)
    res = None
    if residual:
        res = rng.standard_normal((g, hw, 1, cout))
        if data == "offset":
            res += 1e4
        res = res.astype(F)
    return x, x2, wt, scale, shift, res


@pytest.mark.parametrize("case", MEAN_CASES, ids=["g%d_hw%d" % c[0] for c in MEAN_CASES])
def test_mean_epilogue_bit_exact_with_model(cuda, case):
    """The mean equals fused_ref64.mean_model on the unfused output of the same plan bit for bit, and lies within the
    composite float64 bound; the tile width is the flattened layer's."""
    (g, hw), combos = case
    worst = 0.0
    for i, (cout, bn, act, residual, with_x2, mode) in enumerate(combos):
        impl = M.MODES[mode]
        rng = np.random.default_rng(1000 * g + hw + i)
        x, x2, wt, scale, shift, res = mean_inputs(rng, g, hw, cout, residual, with_x2, "offset" if i % 2 else "normal")
        got, y, info = mean_run(x, x2, wt, scale, shift, res, act, impl, bn)
        tw = R.flat_tile_width(g * hw)
        assert info["block_n"] == bn and info["splits"] == 1 and info["tile_w"] == tw, info
        want = R.mean_model(y.reshape(g * hw, cout), hw, tw)
        S.check_exact(got.view(np.int32), want.view(np.int32), "mean g%d hw%d %s cout%d bn%d act%d res%d x2%d"
                      % (g, hw, mode, cout, bn, act, residual, with_x2))
        m64, bound = mean_composite64(x, x2, wt, scale, shift, res, act, impl, y)
        with np.errstate(invalid="ignore"):
            worst = max(worst, S.check_bounded(got, m64, bound, "mean composite g%d hw%d %s" % (g, hw, mode)))
        if (g, hw) == (300, 49) and i == 0:
            _, pg = geom(g, hw, 1, 64, cout, 96 if with_x2 else 0, bn, 0, impl, mean_hw=hw)
            assert pg["units"] > pg["grid"], pg                          # persistent CTAs walk several tiles
    print("\n[mean g%d hw%d] max err/bound (composite) %.3f" % (g, hw, worst))


@pytest.mark.parametrize("geom_", [(5, 49), (3, 300)], ids=["g5_hw49", "g3_hw300"])
def test_mean_epilogue_non_finite(cuda, geom_):
    """ACT_NONE: a NaN, +Inf, -Inf, and +Inf with -Inf in one group, each in its own (group, channel) through the residual,
    reach exactly that group's channel; a channel of one group near 3e37 overflows to +Inf; all as the model predicts bit
    for bit.  ReLU: the NaN rule (fmaxf) makes every such value 0 or finite, and the mean finite."""
    g, hw = geom_
    cout = 68
    rng = np.random.default_rng(113 + g)
    x, x2, wt, scale, shift, res = mean_inputs(rng, g, hw, cout, True, True)
    rf = res.reshape(g * hw, cout)
    last = g - 1
    marks = {(0, 5): "nan", (last, 6): "+inf", (last, 9): "-inf", (1, 7): "inf-inf", (1, 11): "big"}
    rows = lambda gg: np.arange(gg * hw, gg * hw + hw)
    mid = lambda gg: gg * hw + hw // 2
    rf[mid(0), 5] = NAN_QUIET
    rf[mid(last) + 1, 6] = np.inf
    rf[rows(last)[-1], 9] = -np.inf
    rf[rows(1)[0], 7], rf[rows(1)[-1], 7] = np.inf, -np.inf
    rf[rows(1), 11] = F(3e37)
    for act in (0, 1):
        impl = M.F16X3
        got, y, info = mean_run(x, x2, wt, scale, shift, res, act, impl, 128)
        want = R.mean_model(y.reshape(g * hw, cout), hw, info["tile_w"])
        S.check_exact(got, want, "mean non-finite act%d" % act)
        nonfin = ~np.isfinite(got)
        if act == 0:
            expect = np.zeros_like(nonfin)
            for (gg, c) in marks:
                expect[gg, c] = True
            assert np.array_equal(nonfin, expect), "non-finite at %s" % (np.argwhere(nonfin).tolist(),)
            assert np.isnan(got[0, 5]) and got[last, 6] == np.inf and got[last, 9] == -np.inf and np.isnan(got[1, 7])
            assert got[1, 11] == np.inf and np.isfinite(y.reshape(g * hw, cout)[rows(1), 11]).all()
        else:                                      # -Inf and NaN become 0; +Inf and the overflow stay
            assert np.isfinite(got[0, 5]) and np.isfinite(got[last, 9])
            assert got[last, 6] == np.inf and got[1, 7] == np.inf and got[1, 11] == np.inf
            assert y.reshape(g * hw, cout)[mid(0), 5] == 0                  # fmaxf(NaN, 0) = 0
