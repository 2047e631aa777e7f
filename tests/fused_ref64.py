"""CPU models of the conv kernel's two ResNet fusions (`conv_gemm.cu`), used by `test_fused_ref64.py` (their teeth, on the
CPU) and `test_conv_fused_edges_gpu.py` (the device against them).

* Folded weights.  A projection unit's conv3 runs against W' = [W3 diag(s3) ; Wsc diag(ssc)] (fp32 products).  The
  device multiplies the f16 split of the PACKED matrix (one weight exponent for all of it, ops.weight_exponent) and the
  epilogue multiplies by the packed scale.  `pack_columns` restates engine.concat_layers' packing: each column divided by
  the power of two sigma_c that puts its largest |w| in [1, 2), scale = sigma; `pack_whole` is the earlier packing
  (W' as it is, scale 1).  `folded_model` is conv_split_model.model on the packed matrix, times the scale.
* Mean epilogue.  `mean_model` restates epilogue_mean + mean_finish_kernel on the values they sum -- the activated output
  of the same plan without the mean, flattened to [pixels, cout] -- in their exact fp32 order:
    tile mt holds rows [mt tw, mt tw + nrows); group g's rows in it are rs..re (tile-local), rs = max(g hw - w0, 0),
    re = min((g + 1) hw - w0, nrows); the tile partial is  a0 = row rs, a1 = a2 = a3 = 0, then rows rs+1.. four at a time
    into a1, a2, a3, a0, the tail (< 4 rows) into a1, and (a0 + a1) + (a2 + a3);  the group's mean is its tile partials
    added in tile order, divided once (fp32, round to nearest) by hw.
  Every add is one fp32 rounding, as numpy's float32 add, so the model is bit-exact wherever the device is deterministic
  (NaN payloads aside: compare NaN as NaN)."""
import numpy as np

import conv_split_model as M

F = np.float32
U = M.U


# ---- folded weights ---------------------------------------------------------------------------------------------------
def sigma_pow2(w):
    """The power of two per output column that puts the column's largest |w| in [1, 2); 1 for an all-zero column."""
    w = np.asarray(w, F)
    m = np.abs(w).reshape(-1, w.shape[-1]).max(axis=0).astype(np.float64)
    e = np.floor(np.log2(np.where(m > 0, m, 1.0)))
    return np.where(m > 0, 2.0 ** e, 1.0).astype(F)


def pack_columns(wfold):
    """(packed w, epilogue scale) of engine.concat_layers: w / sigma, sigma."""
    sigma = sigma_pow2(wfold)
    return (np.asarray(wfold, F) / sigma).astype(F), sigma


def pack_whole(wfold):
    """(packed w, epilogue scale) of the earlier packing: the folded matrix itself, scale 1."""
    return np.asarray(wfold, F), np.ones(wfold.shape[-1], F)


def check_packing(wpack, scale, wfold):
    """The packing contract: every scale a power of two; w packed * scale == W' bit for bit wherever the quotient W' / scale
    is a normal fp32 (a weight more than 126 binades below its column's largest becomes a subnormal quotient and may lose
    its low bits: at most half its last place, far below the 2^-35 of the column's largest the f16 split keeps); each
    non-zero column's largest |w packed| in [1, 2)."""
    frac, _ = np.frexp(np.asarray(scale, F))
    assert (frac == 0.5).all(), "a column scale is not a power of two"
    wfold = np.asarray(wfold, F)
    back = (wpack * scale).astype(F)
    normal = np.abs(wpack) >= np.finfo(F).tiny
    assert np.array_equal(back[normal].view(np.int32), wfold[normal].view(np.int32)), "w packed * scale != W'"
    assert (np.abs(back.astype(np.float64) - wfold)[~normal] <= (2.0 ** -150 * scale.astype(np.float64) * ~normal)[~normal]).all(), \
        "a subnormal quotient off by more than half its last place"
    m = np.abs(wpack).reshape(-1, wpack.shape[-1]).max(axis=0)
    assert ((m == 0) | ((m >= 1) & (m < 2))).all(), "a column's largest weight outside [1, 2)"


class BNStore(dict):
    """TF-variable-name -> array store with engine.Weights.scale_shift: enough for engine.concat_layers."""

    def scale_shift(self, name, bn_eps):
        from tf_faster_rcnn_b200 import engine
        p = name + "/BatchNorm/"
        return engine.bn_fold(self[p + "gamma"], self[p + "beta"], self[p + "moving_mean"], self[p + "moving_variance"], bn_eps)


def bn_layer(rng, store, name, cin, cout, scale, wstd=0.1):
    """Put a 1x1 layer with BatchNorm into `store`: N(0, wstd^2) weights, and gamma / beta chosen so that the folded scale
    is `scale` per output channel (up to its fp32 roundings) and the folded shift about N(0, scale^2)."""
    var = rng.uniform(0.5, 2.0, cout)
    store[name + "/weights"] = (rng.standard_normal((1, 1, cin, cout)) * wstd).astype(F)
    store[name + "/BatchNorm/gamma"] = (scale * np.sqrt(var + 1e-5)).astype(F)
    store[name + "/BatchNorm/beta"] = (rng.standard_normal(cout) * scale).astype(F)
    store[name + "/BatchNorm/moving_mean"] = (rng.standard_normal(cout) * 0.1).astype(F)
    store[name + "/BatchNorm/moving_variance"] = var.astype(F)


def fold(w3, s3, wsc, ssc):
    """W' = [W3 diag(s3) ; Wsc diag(ssc)]: fp32 products (HWIO [1, 1, cin + cin2, cout])."""
    return np.concatenate([(w3 * s3).astype(F), (wsc * ssc).astype(F)], axis=2)


def folded_model(xc, wpack, scale, mode):
    """(model, S) of a 1x1 layer against the packed matrix: conv_split_model's operand model times the epilogue scale
    (exact: a power of two), and S = sum |x| |w packed * scale|."""
    n, h, w, _ = xc.shape
    m, s = M.model(xc, wpack, mode, 1, 0, 0, h, w)
    return m * scale.astype(np.float64), s * np.abs(scale.astype(np.float64))


def fold_ratio(h2, x, wfold, pack, mode=M.F16X3):
    """Per output channel: max |folded model - float64| / (u S), S = sum |x||W'|, for the packing `pack`."""
    xc = np.concatenate([h2, x], axis=3)
    wp, sc = pack(wfold)
    mdl, _ = folded_model(xc, wp, sc, mode)
    n, h, w, _ = xc.shape
    ref = M.conv64(xc, wfold.astype(np.float64), 1, 0, 0, h, w)
    s = M.conv64(np.abs(xc.astype(np.float64)), np.abs(wfold.astype(np.float64)), 1, 0, 0, h, w)
    with np.errstate(invalid="ignore", divide="ignore"):
        r = np.where(s > 0, np.abs(mdl - ref) / (U * s), 0.0)
    return r.reshape(-1, wfold.shape[-1]).max(axis=0)


# ---- mean epilogue ----------------------------------------------------------------------------------------------------
MUTANTS = ("group_offset", "drop_mid_tile", "double_mid_tile", "divide_by_tile", "segments_from_tile_row")


def _sum4(rows):
    """epilogue_mean's sum of one group's rows of one tile (fp32 [L, C], L >= 1)."""
    z = np.zeros(rows.shape[1], F)
    a0, a1, a2, a3 = rows[0].copy(), z.copy(), z.copy(), z.copy()
    n = rows.shape[0]
    r = 1
    with np.errstate(over="ignore", invalid="ignore"):
        while r + 3 < n:
            a1 = a1 + rows[r]
            a2 = a2 + rows[r + 1]
            a3 = a3 + rows[r + 2]
            a0 = a0 + rows[r + 3]
            r += 4
        while r < n:
            a1 = a1 + rows[r]
            r += 1
        return (a0 + a1) + (a2 + a3)


def tile_partials(y, hw, tw, mutant=None):
    """{(tile, group): fp32 [C]} of epilogue_mean over y fp32 [pixels, C] in tiles of tw rows."""
    P = y.shape[0]
    parts = {}
    for mt in range(-(-P // tw)):
        w0 = mt * tw
        nrows = min(tw, P - w0)
        g0 = w0 // hw
        nseg = (w0 + nrows - 1) // hw - g0 + 1
        buf = y[w0:w0 + nrows]
        for s in range(nseg):
            g = g0 + s
            if mutant == "segments_from_tile_row":          # groups cut at multiples of hw from the tile's first row
                rs, re = s * hw, min((s + 1) * hw, nrows)
            else:
                rs, re = max(g * hw - w0, 0), min((g + 1) * hw - w0, nrows)
            if mutant == "group_offset":
                rs, re = min(rs + 1, nrows - 1), min(re + 1, nrows)
            if rs >= re:
                continue
            parts[(mt, g)] = _sum4(buf[rs:re])
    return parts


def mean_model(y, hw, tw, mutant=None):
    """fp32 [pixels / hw, C]: the mean epilogue's result on the unfused activated output y fp32 [pixels, C] (tile width tw =
    the plan's tile_w).  `mutant` (one of MUTANTS) restates one plausible mistake, for the comparators' teeth."""
    y = np.ascontiguousarray(y, F)
    P, C = y.shape
    assert P % hw == 0
    parts = tile_partials(y, hw, tw, mutant)
    out = np.empty((P // hw, C), F)
    with np.errstate(over="ignore", invalid="ignore"):
        for g in range(P // hw):
            m0, m1 = (g * hw) // tw, (g * hw + hw - 1) // tw
            tiles = list(range(m0, m1 + 1))
            if mutant == "drop_mid_tile" and len(tiles) >= 3:
                tiles.pop(1)
            elif mutant == "double_mid_tile" and len(tiles) >= 3:
                tiles.insert(1, tiles[1])
            acc = parts[(tiles[0], g)].copy()
            for m in tiles[1:]:
                acc = acc + parts[(m, g)]
            out[g] = acc / F(tw if mutant == "divide_by_tile" else hw)
    return out


def flat_tile_width(pixels):
    """The plan's tile width of a flattened pointwise layer of `pixels` rows (conv_gemm.cu choose_tile on one row of
    pixels: the fewest 128-row tiles, then the narrowest width giving that count)."""
    tiles = -(-pixels // 128)
    return -(-pixels // tiles)
