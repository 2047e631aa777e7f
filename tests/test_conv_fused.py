"""The conv kernel's two fusions of the ResNet bottleneck, element by element.

* Second A source: a projection-shortcut unit's conv3 reads its own input h2 (cin channels) and the unit input x (cin2
  channels) in one K loop against [W3 diag(s3) ; Wsc diag(ssc)] (engine.concat_layers), shift b3 + bsc.  Held to a float64
  bound of the unfused formula relu((h2.W3) s3 + b3 + (x.Wsc) ssc + bsc), with u = 2^-24 and S = sum |h2||W3 s3| + |x||Wsc ssc|:
      |got - y64| <= (ALPHA + 2) u S + u |b3 + bsc| + 2 u |pre64|
  ALPHA u S is the kernel's bound against float64 (tests/test_conv_gpu.py); folding a scale into a weight rounds it once
  (u S); the fp32 shift sum rounds once (u |b3 + bsc|); the epilogue's add rounds once (u |pre|, doubled for the error
  already in pre).  F16X1 is not fp32-grade: it is held to its operand model (tests/conv_split_model.py) with BETA instead.
* Mean epilogue: the last conv of the head writes each RoI's spatial mean, not the map.  Its per-element values are those of
  the same plan without the mean (same block_n, never split), so the mean is held to the spatial-mean bound of
  tests/stage_ref64.py around the float64 mean of that unfused output.
The CPU tests pin the weight folding against numpy and the decomposition the two options give.

Observed on an H100 80 GB HBM3 (700 W limit), max err / bound: concatenated conv 0.24 (F16X3), 0.20 (TF32X3), 0.29 (F16X1,
against its model); mean epilogue 0.074 (F16X3, TF32X3), 0.058 (F16X1)."""
import ctypes as C
import zlib

import numpy as np
import pytest
import torch

import conv_split_model as M
import fused_ref64 as R
import stage_ref64 as S

F = np.float32
U = M.U
ALPHA = 8.0           # as tests/test_conv_gpu.py
BETA = 8.0
KEYS = ["block_n", "tile_n", "tile_h", "tile_w", "m_tiles", "n_tiles", "tiles", "split_tiles", "splits", "kb_per_split",
        "units", "grid", "k_blocks", "kb_per_chunk", "tiles_h", "tiles_w"]


def geom(n, h, w, cin, cout, cin2=0, mean_hw=0, block_n=0, split_k=0, impl=0, k=1, sms=132):
    from tf_faster_rcnn_b200 import _native as N
    d = N.ConvDesc(None, None, None, None, None, None, None, n, h, w, cin, cout, k, k, 1, k // 2, k // 2, h, w, 0, block_n, 0,
                   split_k, impl, 1.0, None, cin2, None, mean_hw)
    out = (C.c_int * 16)()
    rc = N.lib().frcnn_conv_plan_geometry(C.byref(d), sms, out)
    return rc, dict(zip(KEYS, list(out)))


# ---- CPU: weight folding and decomposition ------------------------------------------------------------------------------
class _W(dict):
    def scale_shift(self, name, bn_eps):
        from tf_faster_rcnn_b200 import engine
        p = name + "/BatchNorm/"
        return engine.bn_fold(self[p + "gamma"], self[p + "beta"], self[p + "moving_mean"], self[p + "moving_variance"], bn_eps)


def test_concat_layers_folds_scales_in_fp32_per_column_pow2():
    """The BatchNorm scales are folded into the weights in fp32 (w * sigma == the numpy fp32 products, bit for bit), each
    output column packed by a power of two sigma that returns as the epilogue scale, and the shifts summed in fp32."""
    from tf_faster_rcnn_b200 import engine, ops
    rng = np.random.default_rng(11)
    t = _W()
    for nm, cin in (("a/conv3", 64), ("a/shortcut", 96)):
        t[nm + "/weights"] = (rng.standard_normal((1, 1, cin, 256)) * 0.05).astype(F)
        for k, v in (("gamma", rng.uniform(0.3, 0.7, 256)), ("beta", rng.standard_normal(256)),
                     ("moving_mean", rng.standard_normal(256)), ("moving_variance", rng.uniform(0.5, 2, 256))):
            t[nm + "/BatchNorm/" + k] = v.astype(F)
    w, sc, sh = engine.concat_layers(t, ["a/conv3", "a/shortcut"], 1e-5)
    s3, b3 = t.scale_shift("a/conv3", 1e-5)
    ssc, bsc = t.scale_shift("a/shortcut", 1e-5)
    assert sc.dtype == F and w.dtype == F and sh.dtype == F and w.shape == (1, 1, 160, 256) and sc.shape == (256,)
    want = np.concatenate([t["a/conv3/weights"] * s3, t["a/shortcut/weights"] * ssc], axis=2).astype(F)   # fp32 products
    # packed per output column: W' / sigma with sigma a power of two, so w * sigma gives the fp32 products back exactly
    assert (np.frexp(sc)[0] == 0.5).all()
    assert np.array_equal((w * sc).astype(F).view(np.int32), want.view(np.int32))
    m = np.abs(w).reshape(-1, 256).max(axis=0)
    assert ((m >= 1) & (m < 2)).all()
    assert np.array_equal(sh.view(np.int32), (b3 + bsc).astype(F).view(np.int32))
    # one weight exponent for the whole matrix, and every column reaches its top binade
    assert ops.weight_exponent(w) == 13
    # no scale: the weights pass unchanged
    assert np.array_equal(ops.concat_scaled_weights([w[:, :, :64], w[:, :, 64:]], [None, None]), w)


def test_second_source_adds_its_k_blocks_and_keeps_the_tiles():
    for impl, ks in ((0, 2), (1, 1)):
        rc, g1 = geom(4, 38, 50, 64, 256, impl=impl)
        rc2, g2 = geom(4, 38, 50, 64, 256, cin2=96, impl=impl)
        assert rc == rc2 == 0
        assert g2["k_blocks"] == -(-(64 + 96) // (32 * ks))
        assert {k: g1[k] for k in ("block_n", "tile_w", "m_tiles", "n_tiles")} == {k: g2[k] for k in ("block_n", "tile_w", "m_tiles", "n_tiles")}
    rc, g = geom(1, 38, 50, 256, 128, cin2=512, split_k=3)
    assert rc == 0 and g["splits"] == 3 and g["split_tiles"] == g["tiles"]


def test_mean_epilogue_is_never_split():
    rc, g = geom(300, 7, 7, 2048, 512)                     # the head 1x1 splits its ragged round without the mean ...
    assert rc == 0 and g["split_tiles"] > 0
    rc, g = geom(300, 7, 7, 2048, 512, mean_hw=49)          # ... and not with it
    assert rc == 0 and g["split_tiles"] == 0 and g["splits"] == 1 and g["units"] == g["tiles"]


@pytest.mark.parametrize("bad", ["cin2_3x3", "cin2_odd", "mean_3x3", "mean_hw", "mean_split"])
def test_refused_descriptors(bad):
    from tf_faster_rcnn_b200 import _native as N
    args = {"cin2_3x3": dict(cin2=64, k=3), "cin2_odd": dict(cin2=48), "mean_3x3": dict(mean_hw=49, k=3),
            "mean_hw": dict(mean_hw=48), "mean_split": dict(mean_hw=49, split_k=2)}[bad]
    rc, _ = geom(300, 7, 7, 64, 128, **args)
    assert rc == -2 and N.last_error()


# ---- GPU: the concatenated conv --------------------------------------------------------------------------------------
def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


# name, (n, h, w, cin, cin2, cout), split_k
CONCAT_CASES = [
    ("block1_unit1", (2, 19, 25, 64, 64, 256), 0),        # ResNet block1 unit 1: 64 + 64 channels
    ("cin2_96", (1, 20, 30, 64, 96, 128), 0),             # 5 boxes of 32 channels: the f16 modes' odd tail lies in source 2
    ("cin_96", (1, 20, 30, 96, 64, 64), 0),               # a 64-wide k-block straddles the two sources
    ("split3", (1, 38, 50, 256, 512, 128), 3),            # forced split-K over both sources
]


@pytest.mark.gpu
@pytest.mark.parametrize("block_n", [64, 128])
@pytest.mark.parametrize("mode", ["f16x3", "tf32x3", "f16x1"])
@pytest.mark.parametrize("case", CONCAT_CASES, ids=[c[0] for c in CONCAT_CASES])
def test_concat_conv_within_bound_of_unfused(cuda, case, mode, block_n):
    from tf_faster_rcnn_b200 import _native as N, ops
    name, (n, h, w, cin, cin2, cout), split_k = case
    impl = M.MODES[mode]
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    h2 = rng.standard_normal((n, h, w, cin)).astype(F)
    x = rng.standard_normal((n, h, w, cin2)).astype(F)
    w3 = (rng.standard_normal((1, 1, cin, cout)) * np.sqrt(2.0 / cin)).astype(F)
    wsc = (rng.standard_normal((1, 1, cin2, cout)) * np.sqrt(2.0 / cin2)).astype(F)
    s3, ssc = rng.uniform(0.3, 1.5, cout).astype(F), rng.uniform(0.3, 1.5, cout).astype(F)
    b3, bsc = rng.standard_normal(cout).astype(F), rng.standard_normal(cout).astype(F)
    wcat = ops.concat_scaled_weights([w3, wsc], [s3, ssc])
    wpack, sigma = R.pack_columns(wcat)                   # engine.concat_layers' packing
    shift = (b3 + bsc).astype(F)
    pc = ops.PackedConv(wpack, sigma, shift, impl=impl)
    hd, xd = dev(h2), dev(x)
    buf, out = S.guarded_out((n, h, w, cout))
    plan = ops.ConvPlan(hd, pc, out, 1, 0, 0, N.ACT_RELU, None, block_n, 0, split_k, x2=xd)
    outs = []
    for _ in range(2):
        plan.run()
        torch.cuda.synchronize()
        outs.append(out.cpu().numpy().copy())
        S.check_guarded(buf, out.numel())
    got = outs[0]
    assert np.array_equal(outs[0].view(np.int32), outs[1].view(np.int32)), "two runs differ"
    assert np.array_equal(hd.cpu().numpy(), h2) and np.array_equal(xd.cpu().numpy(), x), "input modified"
    info = plan.info()
    assert info["block_n"] == block_n and (not split_k or info["splits"] == split_k), info
    _, g = geom(n, h, w, cin, cout, cin2=cin2, block_n=block_n, split_k=split_k, impl=impl,
                sms=torch.cuda.get_device_properties(0).multi_processor_count)
    assert g["k_blocks"] == -(-(cin + cin2) // (32 if impl == M.TF32X3 else 64))
    c64 = lambda a, b: M.conv64(a, b, 1, 0, 0, h, w)
    if mode != "f16x1":
        pre64 = (c64(h2, w3) * s3.astype(np.float64) + b3.astype(np.float64) + c64(x, wsc) * ssc.astype(np.float64)
                 + bsc.astype(np.float64))
        s = c64(np.abs(h2), np.abs(w3.astype(np.float64) * s3)) + c64(np.abs(x), np.abs(wsc.astype(np.float64) * ssc))
        bound = (ALPHA + 2) * U * s + U * np.abs(b3.astype(np.float64) + bsc) + 2 * U * np.abs(pre64)
        alpha_s = ALPHA
    else:
        m, s = R.folded_model(np.concatenate([h2, x], axis=3), wpack, sigma, impl)
        pre64 = m + shift.astype(np.float64)
        bound = BETA * U * s + 2 * U * np.abs(pre64)
        alpha_s = BETA
    y64 = np.maximum(pre64, 0)
    r = S.check_bounded(got, y64, bound, "concat conv %s %s bn%d" % (name, mode, block_n))
    err = np.abs(got - y64)
    print("\n[concat %s %s bn%d] max err/bound %.3f  max err/(u S) %.2f (bound's kernel share %.0f)"
          % (name, mode, block_n, r, float((err / (U * s)).max()), alpha_s))


# ---- GPU: the mean epilogue --------------------------------------------------------------------------------------------
# name, (rois, side, cin, cin2, cout), the tiles of 128 rows (or fewer) the flattened rows fill
MEAN_CASES = [
    ("r2_1tile", (2, 7, 64, 0, 256), 1),                  # 98 rows: both RoIs in one tile
    ("r5_2tiles", (5, 7, 64, 0, 256), 2),                 # 245 rows: a RoI straddles the tile boundary
    ("r7_3tiles", (7, 7, 64, 0, 128), 3),
    ("r10_4tiles", (10, 7, 64, 0, 192), 4),               # 490 rows; cout 192: a partial last N tile at block_n 128
    ("r300_hw49", (300, 7, 64, 0, 512), 115),             # the head's 300 RoIs
    ("r300_hw1", (300, 1, 64, 0, 256), 3),                # hw = 1: every row is its own group
    ("r5_x2", (5, 7, 64, 96, 256), 2),                    # with a second A source (a one-unit block)
]


@pytest.mark.gpu
@pytest.mark.parametrize("data", ["normal", "offset", "cancel"])
@pytest.mark.parametrize("block_n", [64, 128])
@pytest.mark.parametrize("mode", ["f16x3", "tf32x3", "f16x1"])
@pytest.mark.parametrize("case", MEAN_CASES, ids=[c[0] for c in MEAN_CASES])
def test_mean_epilogue_within_spatial_mean_bound(cuda, case, mode, block_n, data):
    """normal: ReLU'd conv + residual; offset / cancel: no activation, the residual carries stage_ref64's data (1e4 + N(0,1);
    +1e4 over the first half of each RoI's positions, -1e4 over the rest)."""
    from tf_faster_rcnn_b200 import _native as N, ops
    name, (r, side, cin, cin2, cout), tiles = case
    impl = M.MODES[mode]
    rng = np.random.default_rng(zlib.crc32((name + data).encode()))
    x = rng.standard_normal((r, side, side, cin)).astype(F)
    x2 = rng.standard_normal((r, side, side, cin2)).astype(F) if cin2 else None
    wt = (rng.standard_normal((1, 1, cin + cin2, cout)) * np.sqrt(2.0 / (cin + cin2))).astype(F)
    scale, shift = rng.uniform(0.5, 1.5, cout).astype(F), rng.standard_normal(cout).astype(F)
    res = rng.standard_normal((r, side, side, cout))
    if data == "offset":
        res += 1e4
    elif data == "cancel":
        res += np.where(np.arange(side * side).reshape(1, side, side, 1) < side * side // 2, 1e4, -1e4)
    res = res.astype(F)
    act = N.ACT_RELU if data == "normal" else N.ACT_NONE
    pc = ops.PackedConv(wt, scale, shift, impl=impl)
    xd, rd = dev(x), dev(res)
    x2d = None if x2 is None else dev(x2)
    full = torch.empty((r, side, side, cout), dtype=torch.float32, device="cuda")
    ops.ConvPlan(xd, pc, full, 1, 0, 0, act, rd, block_n, 0, 1, x2=x2d).run()          # the same plan, unfused and unsplit
    buf, out = S.guarded_out((r, cout))
    plan = ops.ConvPlan(xd, pc, out, 1, 0, 0, act, rd, block_n, 0, 0, x2=x2d, mean=True)
    outs = []
    for _ in range(2):
        plan.run()
        torch.cuda.synchronize()
        outs.append(out.cpu().numpy().copy())
        S.check_guarded(buf, out.numel())
    assert np.array_equal(outs[0].view(np.int32), outs[1].view(np.int32)), "two runs differ"
    assert np.array_equal(rd.cpu().numpy(), res), "residual modified"
    info = plan.info()
    assert info["block_n"] == block_n and info["splits"] == 1 and info["grid_m"] == tiles, info
    y = full.cpu().numpy()
    m64, bound = S.spatial_mean_ref(y)
    with np.errstate(invalid="ignore"):                  # 0 / 0 where a ReLU'd mean is exactly 0 (bound 0, err 0)
        ratio = S.check_bounded(outs[0], m64, bound, "mean epilogue %s %s bn%d %s" % (name, mode, block_n, data))
    print("\n[mean %s %s bn%d %s] max err/bound %.3f" % (name, mode, block_n, data, ratio))
