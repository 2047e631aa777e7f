"""The models of fused_ref64.py and their comparators have teeth, on the CPU.

* Folded weights: the packing of engine.concat_layers is the restatement of fused_ref64 bit for bit (powers of two,
  w * scale == W'); on the device's operand model the earlier packing (W' whole, scale 1) loses the fp32 grade of channels
  whose two BatchNorm scales are both small, from about 2^-30 on, and the per-column packing keeps it down to 2^-60.
* Mean epilogue: the op-order model lies within stage_ref64's spatial-mean bound, on every geometry of the GPU tests; one
  plausible mistake each fails it -- a group offset by one row, the middle tile of a 3-tile group dropped or added twice,
  division by the tile width, segments counted from the tile's first row, source-2 rows shifted by one pixel, a column
  scale that is not a power of two."""
import numpy as np
import pytest

import conv_split_model as M
import fused_ref64 as R
import stage_ref64 as S

F = np.float32
ALPHA = 8.0           # the kernel's per-element bound against float64, in u S (tests/test_conv_gpu.py)


# ---- folded weights ---------------------------------------------------------------------------------------------------
SCALES = 2.0 ** np.array([8, 4, 0, -4, -12, -24, -28, -32, -36, -48, -60, -100, -126, -140], np.float64)


def test_concat_layers_packs_per_column_powers_of_two():
    """engine.concat_layers == fused_ref64.pack_columns bit for bit, on channels whose scales run from 2^8 to 2^-140
    (subnormal folded weights) plus an all-zero channel; the packing contract holds and the matrix packs at wexp 13."""
    from tf_faster_rcnn_b200 import engine, ops
    rng = np.random.default_rng(5)
    cout = len(SCALES) + 1
    sc = np.append(SCALES, 1.0)
    t = R.BNStore()
    R.bn_layer(rng, t, "u/conv3", 64, cout, sc)
    R.bn_layer(rng, t, "u/shortcut", 96, cout, sc[::-1])
    t["u/conv3/weights"][..., -1] = 0
    t["u/shortcut/weights"][..., -1] = 0
    w, scale, shift = engine.concat_layers(t, ["u/conv3", "u/shortcut"], 1e-5)
    s3, b3 = t.scale_shift("u/conv3", 1e-5)
    ssc, bsc = t.scale_shift("u/shortcut", 1e-5)
    wfold = R.fold(t["u/conv3/weights"], s3, t["u/shortcut/weights"], ssc)
    wp, sp = R.pack_columns(wfold)
    assert w.dtype == F and scale.dtype == F and shift.dtype == F and w.shape == (1, 1, 160, cout)
    assert np.array_equal(w.view(np.int32), wp.view(np.int32)) and np.array_equal(scale.view(np.int32), sp.view(np.int32))
    R.check_packing(w, scale, wfold)
    assert scale[-1] == 1 and not w[..., -1].any()
    assert np.array_equal(shift.view(np.int32), (b3 + bsc).astype(F).view(np.int32))
    assert ops.weight_exponent(w) == 13
    assert np.array_equal(ops.column_scales(wfold), sp)


def test_column_scales_edges():
    """Powers of two exactly, one ulp below a power of two, the largest fp32, the smallest subnormal, zero, Inf and NaN."""
    from tf_faster_rcnn_b200 import ops
    big = np.finfo(F).max
    cols = [F(1), F(2), np.nextafter(F(2), F(0)), F(-0.75), big, F(2.0 ** -149), F(0), F(np.inf), F(np.nan)]
    want = [1, 2, 1, 0.5, 2.0 ** 127, 2.0 ** -149, 1, 1, 1]
    w = np.zeros((1, 1, 3, len(cols)), F)
    w[0, 0, 1] = cols
    got = ops.column_scales(w)
    assert got.dtype == F and np.array_equal(got, np.asarray(want, F)), got


def _fold_case(rng, s3, ssc, cin=64, cin2=64):
    h2 = np.abs(rng.standard_normal((1, 8, 16, cin))).astype(F)          # conv2's ReLU output
    x = rng.standard_normal((1, 8, 16, cin2)).astype(F)
    w3 = (rng.standard_normal((1, 1, cin, len(s3))) * 0.1).astype(F)
    wsc = (rng.standard_normal((1, 1, cin2, len(s3))) * 0.1).astype(F)
    return h2, x, R.fold(w3, np.asarray(s3, F), wsc, np.asarray(ssc, F))


def test_fold_check_whole_matrix_packing_loses_small_channels():
    """Channel c with both BatchNorm scales 2^-4c (c = 0..15).  Earlier packing: within ALPHA u S down to 2^-28, above it from
    2^-32 on.  Per-column packing: within it down to 2^-60.  One scale small and the other 1 passes either way (the small
    part is a vanishing share of S)."""
    rng = np.random.default_rng(7)
    sc = 2.0 ** (-4.0 * np.arange(16))
    h2, x, wf = _fold_case(rng, sc, sc)
    old = R.fold_ratio(h2, x, wf, R.pack_whole)
    new = R.fold_ratio(h2, x, wf, R.pack_columns)
    print("\n[fold] whole-matrix packing err/(u S) by channel:", " ".join("%.3g" % v for v in old))
    print("[fold] per-column packing  err/(u S) by channel:", " ".join("%.3g" % v for v in new))
    assert old[:8].max() <= ALPHA and (old[8:] > ALPHA).all() and old[-1] > 1e4 * ALPHA, old
    assert new.max() <= ALPHA, new
    for a, b in ((sc, np.ones(16)), (np.ones(16), sc)):
        h2, x, wf = _fold_case(rng, a, b)
        for pack in (R.pack_whole, R.pack_columns):
            assert R.fold_ratio(h2, x, wf, pack).max() <= ALPHA
    # TF32X3 carries no weight exponent: both packings are fp32-grade
    h2, x, wf = _fold_case(rng, sc, sc)
    for pack in (R.pack_whole, R.pack_columns):
        assert R.fold_ratio(h2, x, wf, pack, M.TF32X3).max() <= ALPHA


def test_fold_teeth_source2_shifted_and_scale_not_power_of_two():
    rng = np.random.default_rng(9)
    sc = 2.0 ** (-2.0 * np.arange(8))
    h2, x, wf = _fold_case(rng, sc, sc[::-1])
    assert R.fold_ratio(h2, x, wf, R.pack_columns).max() <= ALPHA
    # source-2 rows one pixel late: the model of x's rows shifted against the truth
    xs = np.roll(x.reshape(-1, x.shape[-1]), 1, axis=0).reshape(x.shape)
    xc, xsc = np.concatenate([h2, x], axis=3), np.concatenate([h2, xs], axis=3)
    wp, sp = R.pack_columns(wf)
    mdl, s = R.folded_model(xsc, wp, sp, M.F16X3)
    ref = M.conv64(xc, wf.astype(np.float64), 1, 0, 0, 8, 16)
    assert (np.abs(mdl - ref) / (M.U * s)).max() > 1e3 * ALPHA
    # a scale that is not a power of two (the column maximum itself): the product no longer gives W' back
    m = np.abs(wf).reshape(-1, wf.shape[-1]).max(axis=0)
    bad = (wf / m).astype(F)
    with pytest.raises(AssertionError, match="power of two"):
        R.check_packing(bad, m, wf)
    assert not np.array_equal((bad * m).astype(F), wf)
    R.check_packing(wp, sp, wf)


# ---- mean epilogue ----------------------------------------------------------------------------------------------------
# (groups, hw) of the GPU tests' mean geometries, and the tile width of the flattened layer
MEAN_GEOMS = [(300, 1), (200, 2), (97, 3), (61, 7), (300, 49), (5, 49), (2, 64), (3, 127), (2, 128), (3, 129), (5, 196),
              (3, 300), (2, 1000), (1, 7)]


def _mean_data(rng, g, hw, c, kind):
    y = rng.standard_normal((g * hw, c))
    if kind == "offset":
        y += 1e4
    elif kind == "cancel":
        y += np.where((np.arange(g * hw) % hw < hw // 2)[:, None], 1e4, -1e4)
    elif kind == "relu":
        y = np.maximum(y, 0)
    return y.astype(F)


@pytest.mark.parametrize("kind", ["normal", "offset", "cancel", "relu"])
def test_mean_model_within_spatial_mean_bound(kind):
    rng = np.random.default_rng(13)
    for g, hw in MEAN_GEOMS:
        y = _mean_data(rng, g, hw, 12, kind)
        tw = R.flat_tile_width(g * hw)
        got = R.mean_model(y, hw, tw)
        m64, bound = S.spatial_mean_ref(y.reshape(g, hw, 1, -1))
        with np.errstate(invalid="ignore"):
            S.check_bounded(got, m64, bound, "mean model g%d hw%d %s" % (g, hw, kind))
        if hw == 1:                                      # one row per group: the value itself (-0 aside)
            assert np.array_equal(got, y + F(0))


def test_mean_model_geometry_coverage():
    """The geometries reach every shape of the group/tile overlap: many start offsets in a tile, groups spanning 1, 2, 3 and
    >= 8 tiles, layers of fewer rows than one tile."""
    offsets, spans, short = set(), set(), False
    for g, hw in MEAN_GEOMS:
        P = g * hw
        tw = R.flat_tile_width(P)
        short |= P < 128
        for k in range(g):
            offsets.add((k * hw) % tw)
            spans.add((k * hw + hw - 1) // tw - (k * hw) // tw + 1)
    assert len(offsets) >= 100 and {1, 2, 3} <= spans and max(spans) >= 8 and short, (len(offsets), spans)


# mutant -> (groups, hw) where it must show
MUTANT_CASES = {"group_offset": (5, 49), "drop_mid_tile": (3, 300), "double_mid_tile": (3, 300),
                "divide_by_tile": (300, 49), "segments_from_tile_row": (5, 49)}


@pytest.mark.parametrize("mutant", R.MUTANTS)
def test_mean_model_mutants_fail(mutant):
    rng = np.random.default_rng(17)
    g, hw = MUTANT_CASES[mutant]
    y = _mean_data(rng, g, hw, 12, "offset")
    y[np.arange(g * hw) % hw == 0] += 5e3                 # a group's first row stands out: an offset by one row shows
    tw = R.flat_tile_width(g * hw)
    m64, bound = S.spatial_mean_ref(y.reshape(g, hw, 1, -1))
    S.check_bounded(R.mean_model(y, hw, tw), m64, bound)
    with pytest.raises(AssertionError, match="err/bound"):
        S.check_bounded(R.mean_model(y, hw, tw, mutant), m64, bound, mutant)
