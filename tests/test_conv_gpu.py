"""The wgmma implicit-GEMM conv/FC kernel (`conv_gemm_kernel`) in all three arithmetic modes, element by element.

With u = 2^-24, S_i = sum |x||w| over output i's receptive field (tests/conv_split_model.py) and act = NONE:
  (a) accumulation  |got - model| <= BETA * u * S_i   every mode, every operand range: the model holds the device's operand
                    roundings, so only summation error remains; a dropped, doubled, mis-scaled or mis-swizzled term is
                    orders of magnitude above it.
  (b) fp32 grade    |got - ref64| <= ALPHA * u * S_i  F16X3 and TF32X3 inside the documented operand range (float64 truth);
                    F16X1 fails it by >= 100x.
With an epilogue the reference is the float64 epilogue of the model / of ref64, and the bound gains |scale| and the
roundings of the epilogue's three fp32 operations.  Every path case asserts the plan took the path it exists for
(frcnn_conv_plan_geometry at the device's SM count, cross-checked against the plan's own report), runs its output into a
NaN-prefilled view between sentinel guard bands, and checks that input and residual are untouched.

Calibration (H100 80 GB HBM3, 400 W): ALPHA = BETA = 8; the observed maxima of err / (u S) per mode are listed at their
definition (largest: 1.97 for (a), 6.22 for (b); F16X1 misses (b) by 636x on its demonstration case).
The older tests further down keep their max-norm bound (4e-6 of max|ref|)."""
import ctypes as C
import zlib

import numpy as np
import pytest
import torch

import conv_split_model as M
from oracle import layers as L

pytestmark = pytest.mark.gpu
F = np.float32


def ref64(x, w, stride, pad_t, pad_l, ho, wo):
    return M.conv64(x, w, stride, pad_t, pad_l, ho, wo)


def run_conv(x, w, stride, mode, scale=None, shift=None, residual=None, act=0, block_n=0, kb_per_chunk=0, time_it=False, split_k=0):
    from tf_faster_rcnn_b200 import ops
    n, h, wd, cin = x.shape
    k = w.shape[0]
    ho, wo, pt, pl = ops.conv_out_hw(h, wd, k, stride, mode)
    pc = ops.PackedConv(w, scale, shift)
    xd = torch.from_numpy(x).cuda()
    out = torch.full((n, ho, wo, w.shape[3]), float("nan"), dtype=torch.float32, device="cuda")
    rd = None if residual is None else torch.from_numpy(residual).cuda()
    plan = ops.ConvPlan(xd, pc, out, stride, pt, pl, act, rd, block_n, kb_per_chunk, split_k)
    plan.run()
    torch.cuda.synchronize()
    info = plan.info()
    if time_it:
        for _ in range(3):
            plan.run()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(20):
            plan.run()
        e1.record()
        torch.cuda.synchronize()
        info["us"] = e0.elapsed_time(e1) * 1000 / 20
        info["tflops"] = 2.0 * n * ho * wo * w.shape[3] * k * k * cin / (info["us"] * 1e-6) / 1e12
    return out.cpu().numpy(), info, (ho, wo, pt, pl)


CASES = [
    # name, n, h, w, cin, cout, k, stride, mode, block_n
    ("fc_small", 1, 1, 300, 64, 64, 1, 1, "SAME", 0),
    ("pw_1900_bn64", 1, 38, 50, 256, 256, 1, 1, "SAME", 64),
    ("pw_1900_bn128", 1, 38, 50, 1024, 256, 1, 1, "SAME", 128),
    ("c3_s1_64", 1, 38, 50, 64, 64, 3, 1, "SAME", 0),
    ("c3_s1_odd_cout", 1, 20, 30, 128, 96, 3, 1, "SAME", 0),
    ("c3_s1_big", 1, 75, 100, 64, 128, 3, 1, "SAME", 0),
    ("c3_s2_explicit", 1, 75, 100, 64, 64, 3, 2, "EXPLICIT", 0),
    ("c3_s2_odd", 1, 38, 51, 32, 64, 3, 2, "EXPLICIT", 0),
    ("head_c3_rois", 20, 7, 7, 64, 64, 3, 1, "SAME", 0),
    ("head_pw_rois", 20, 7, 7, 128, 64, 1, 1, "SAME", 0),
    ("fc_k3136", 1, 1, 300, 3136, 128, 1, 1, "SAME", 0),
    ("fc_cout405", 1, 1, 300, 256, 405, 1, 1, "SAME", 0),
    ("rpn_cout72", 1, 38, 50, 512, 72, 1, 1, "SAME", 0),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_conv_matches_oracle(cuda, case):
    name, n, h, w, cin, cout, k, stride, mode, bn = case
    rng = np.random.default_rng(abs(hash(name)) % (2 ** 31))
    x = rng.standard_normal((n, h, w, cin)).astype(F)
    wt = (rng.standard_normal((k, k, cin, cout)) * np.sqrt(2.0 / (k * k * cin))).astype(F)
    got, info, (ho, wo, pt, pl) = run_conv(x, wt, stride, mode, block_n=bn)
    want64 = ref64(x, wt, stride, pt, pl, ho, wo)
    want32 = L.conv2d(x, wt, stride, "SAME") if mode == "SAME" else L.conv2d_same(x, wt, stride)
    assert got.shape == want32.shape
    assert np.isfinite(got).all(), "%s: non-finite output (unwritten rows?) plan=%s" % (name, info)
    scale = np.abs(want64).max()
    e_gpu = np.abs(got - want64).max() / scale
    e_cpu = np.abs(want32 - want64).max() / scale
    print("\n[%s] plan=%s err_gpu_vs_f64=%.2e err_oracle_vs_f64=%.2e gpu_vs_oracle=%.2e" %
          (name, info, e_gpu, e_cpu, np.abs(got - want32).max() / scale))
    assert e_gpu < 4e-6, (name, e_gpu, info)


def test_conv_epilogue_bn_residual_relu(cuda):
    rng = np.random.default_rng(5)
    x = rng.standard_normal((1, 38, 50, 64)).astype(F)
    wt = (rng.standard_normal((1, 1, 64, 256)) * 0.2).astype(F)
    gamma, beta = rng.uniform(0.5, 1.5, 256).astype(F), rng.standard_normal(256).astype(F)
    mean, var = rng.standard_normal(256).astype(F), rng.uniform(0.5, 1.5, 256).astype(F)
    res = rng.standard_normal((1, 38, 50, 256)).astype(F)
    conv = L.conv2d(x, wt, 1, "SAME")
    bn, inv, shift = L.batch_norm(conv, gamma, beta, mean, var, 1e-5)
    want = L.relu(res + bn)
    got, info, _ = run_conv(x, wt, 1, "SAME", scale=inv, shift=shift, residual=res, act=1)
    err = np.abs(got - want).max()
    print("\n[epilogue] plan=%s max abs err=%.2e" % (info, err))
    assert err < 2e-5
    got6, _, _ = run_conv(x, wt, 1, "SAME", scale=None, shift=beta, act=2)
    assert np.abs(got6 - L.relu6(conv + beta)).max() < 2e-5


@pytest.mark.parametrize("shape", [("k3136_fc", 1, 1, 300, 3136, 128, 1), ("vgg_conv5", 1, 38, 50, 512, 512, 3),
                                   ("vgg_conv3", 1, 150, 200, 256, 256, 3), ("res_head_pw", 300, 7, 7, 2048, 512, 1),
                                   ("res_head_c3", 300, 7, 7, 512, 512, 3), ("res_b3_pw", 1, 38, 50, 1024, 256, 1)])
def test_accumulation_chunk_sweep(cuda, shape):
    """Accuracy and speed over the kb_per_chunk settings a plan accepts (the sm_90a kernel promotes every k-block)."""
    name, n, h, w, cin, cout, k = shape
    rng = np.random.default_rng(1)
    x = np.maximum(rng.standard_normal((n, h, w, cin)), 0).astype(F)      # post-ReLU-like
    wt = (rng.standard_normal((k, k, cin, cout)) * np.sqrt(2.0 / (k * k * cin))).astype(F)
    want64 = None
    for kpc in (2, 4, 8, 12, 16, 100000):
        for bn in ((0,) if kpc != 8 else (0, 64)):
            got, info, (ho, wo, pt, pl) = run_conv(x, wt, 1, "SAME", block_n=bn, kb_per_chunk=kpc, time_it=True)
            if want64 is None:
                want64 = ref64(x, wt, 1, pt, pl, ho, wo)
                want32 = L.conv2d(x, wt, 1, "SAME")
                print("\n[%s] oracle fp32 vs f64: %.2e" % (name, np.abs(want32 - want64).max() / np.abs(want64).max()))
            e = np.abs(got - want64).max() / np.abs(want64).max()
            print("[%s] kb_per_chunk=%d bn=%d grid=%dx%d tile=%dx%dx%d  err=%.2e  %.1f us  %.1f TFLOP/s" %
                  (name, kpc, info["block_n"], info["grid_m"], info["grid_n"], info["tile_n"], info["tile_h"], info["tile_w"],
                   e, info["us"], info["tflops"]))
            if kpc <= 8:
                assert e < 4e-6


@pytest.mark.parametrize("shape", [("b3_conv1", 1, 38, 50, 1024, 256, 1), ("b3_conv2", 1, 38, 50, 256, 256, 3), ("vgg_conv5", 1, 38, 50, 512, 512, 3),
                                   ("fc6_like", 1, 1, 300, 25088, 256, 1)])
def test_split_k(cuda, shape):
    """split-K (two-pass, deterministic) matches the unsplit kernel's accuracy, incl. BN + residual + ReLU epilogue."""
    name, n, h, w, cin, cout, k = shape
    rng = np.random.default_rng(3)
    x = np.maximum(rng.standard_normal((n, h, w, cin)), 0).astype(F)
    wt = (rng.standard_normal((k, k, cin, cout)) * np.sqrt(2.0 / (k * k * cin))).astype(F)
    scale = rng.uniform(0.5, 1.5, cout).astype(F); shift = rng.standard_normal(cout).astype(F)
    res = rng.standard_normal((n, h, w, cout)).astype(F)
    want = L.relu(L.conv2d(x, wt, 1, "SAME") * scale + shift + res)
    for sk in (1, 0, 2, 3, 8):
        got, info, _ = run_conv(x, wt, 1, "SAME", scale=scale, shift=shift, residual=res, act=1, split_k=sk, time_it=True)
        got2, _, _ = run_conv(x, wt, 1, "SAME", scale=scale, shift=shift, residual=res, act=1, split_k=sk)
        e = np.abs(got - want).max() / np.abs(want).max()
        print("\n[%s] split_k=%d -> splits=%d grid=%dx%d bn=%d  err vs oracle %.2e  %.1f us" %
              (name, sk, info["splits"], info["grid_m"], info["grid_n"], info["block_n"], e, info["us"]))
        assert e < 5e-6
        assert np.array_equal(got, got2), "split-K must be run-to-run deterministic"


def test_throughput_mode_f16x1(cuda):
    """FRCNN_CONV_F16X1 (opt-in, NOT fp32-grade): plain fp16 operands, one MMA per product, fp32 accumulation -- error of a few
    1e-4 of the output range, three orders above the default FP16x3 path on the same packed weights."""
    from tf_faster_rcnn_b200 import ops, _native as N
    rng = np.random.default_rng(12)
    for (n, h, w, cin, cout, k) in [(1, 38, 50, 256, 256, 3), (20, 7, 7, 512, 512, 1), (1, 1, 300, 3136, 128, 1)]:
        x = np.maximum(rng.standard_normal((n, h, w, cin)), 0).astype(np.float32)
        wt = (rng.standard_normal((k, k, cin, cout)) * np.sqrt(2.0 / (k * k * cin))).astype(np.float32)
        ho, wo, pt, pl = ops.conv_out_hw(h, w, k, 1, "SAME")
        errs = {}
        for impl in (N.CONV_F16X3, N.CONV_F16X1):
            pc = ops.PackedConv(wt, impl=impl)
            out = torch.full((n, ho, wo, cout), float("nan"), dtype=torch.float32, device="cuda")
            ops.ConvPlan(torch.from_numpy(x).cuda(), pc, out, 1, pt, pl, 0, None).run()
            torch.cuda.synchronize()
            errs[impl] = out.cpu().numpy()
        scale = np.abs(errs[N.CONV_F16X3]).max()
        dev = np.abs(errs[N.CONV_F16X1] - errs[N.CONV_F16X3]).max() / scale
        assert not np.isnan(errs[N.CONV_F16X1]).any()
        assert 1e-6 < dev < 3e-3, dev


# ---------------------------------------------------------------------------------------------------------------------
# Per-element bounds in all three modes
#
# Observed on an H100 80 GB HBM3 (400 W limit), max over elements of err / (u S):
#   (a) vs the model, path cases:        F16X3 1.79, TF32X3 1.97, F16X1 1.88 (all three on long_fc6_pos, K = 25088, x, w >= 0)
#   (b) vs float64, path cases:          F16X3 1.82, TF32X3 1.98; the all-positive demo of test_f16x1_fails_...: F16X3 6.22
#       F16X1:                           189 (long_fc6_pos) .. 6176 (tail_pw_cin32); 5088 on the demo (>= 100 x ALPHA)
#       the fp32 CPU oracle L.conv2d:    3.1 .. 9.4, and 65 on long_c3_512_pos
#   TF32X3 activation sweep 2^-100 .. 2^100: (a) <= 0.90, (b) <= 0.97; weight channel spread / layer scales: <= 1.1
#   F16X3 activation sweep 2^-20 .. 65504: (a) <= 0.88, (b) <= 1.01 from 2^-14 up; layer scales 1e-6 / 300 / 1e-20: <= 0.90
#   deep fp16-subnormal operands: (a) 12.4 for activations at 2^-24 (F16X3 and F16X1; 0.69 at 2^-20 and 2^-16) and 18.0 over
#   the channels 2^-28 .. 2^-40 below the layer max.  The model multiplies the subnormal fp16
#   values exactly; the tensor core's sums of such products are off by a further ~2^-20 of S.  Not modelled: asserted
#   against BETA_SUBNORMAL, which applies only there.
U = M.U
ALPHA = 8.0           # (b): F16X3 / TF32X3 vs float64 (2^-21 of S)
BETA = 8.0            # (a): every mode vs the operand model
BETA_SUBNORMAL = 32.0 # (a) where fp16 operands are subnormal (see above)
MODE_IDS = ["f16x3", "tf32x3", "f16x1"]
GEOM_KEYS = ["block_n", "tile_n", "tile_h", "tile_w", "m_tiles", "n_tiles", "tiles", "split_tiles", "splits", "kb_per_split",
             "units", "grid", "k_blocks", "kb_per_chunk", "tiles_h", "tiles_w"]
GUARD = 64                              # floats of sentinel before and after every output: 256 B keeps float4 stores aligned
SENTINEL = np.int32(0x7fa5a5a5)         # a NaN payload no kernel produces


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def geometry(x_shape, cout, k, stride, pt, pl, ho, wo, impl, block_n=0, split_k=0):
    """frcnn_conv_plan_geometry at the device's SM count: the decomposition the plan chooses."""
    from tf_faster_rcnn_b200 import _native as N
    n, h, w, cin = x_shape
    d = N.ConvDesc(None, None, None, None, None, None, None, n, h, w, cin, cout, k, k, stride, pt, pl, ho, wo, 0, block_n, 0,
                   split_k, impl, 1.0)
    out = (C.c_int * 16)()
    N.check(N.lib().frcnn_conv_plan_geometry(C.byref(d), sm_count(), out), "geometry")
    return dict(zip(GEOM_KEYS, list(out)))


def guarded(shape):
    """(whole buffer, NaN-prefilled output view): sentinels before and after the view, offset a multiple of 16 bytes."""
    numel = int(np.prod(shape))
    buf = torch.full((numel + 2 * GUARD,), int(SENTINEL), dtype=torch.int32, device="cuda")
    out = buf.view(torch.float32)[GUARD:GUARD + numel].view(shape)
    out.fill_(float("nan"))
    return buf, out


def check_guards(buf, numel):
    b = buf.cpu().numpy()
    assert (b[:GUARD] == SENTINEL).all() and (b[GUARD + numel:] == SENTINEL).all(), "store outside the output"


def conv_run(x, w, impl, stride=1, pad="SAME", scale=None, shift=None, residual=None, act=0, block_n=0, split_k=0, runs=1):
    """One plan, `runs` runs; returns (outputs of every run, plan info, geometry, (ho, wo, pt, pl))."""
    from tf_faster_rcnn_b200 import ops
    n, h, wd, cin = x.shape
    k, cout = w.shape[0], w.shape[3]
    ho, wo, pt, pl = ops.conv_out_hw(h, wd, k, stride, pad)
    pc = ops.PackedConv(w, scale, shift, impl=impl)
    xd = dev(x)
    rd = None if residual is None else dev(residual)
    buf, out = guarded((n, ho, wo, cout))
    plan = ops.ConvPlan(xd, pc, out, stride, pt, pl, act, rd, block_n, 0, split_k)
    outs = []
    for _ in range(runs):
        plan.run()
        torch.cuda.synchronize()
        outs.append(out.cpu().numpy().copy())
        check_guards(buf, out.numel())
    assert np.array_equal(xd.cpu().numpy().view(np.int32), x.view(np.int32)), "input modified"
    if residual is not None:
        assert np.array_equal(rd.cpu().numpy().view(np.int32), residual.view(np.int32)), "residual modified"
    info = plan.info()
    g = geometry(x.shape, cout, k, stride, pt, pl, ho, wo, impl, block_n, split_k)
    assert (info["block_n"], info["tile_n"], info["tile_h"], info["tile_w"], info["grid_m"], info["grid_n"]) == \
        (g["block_n"], g["tile_n"], g["tile_h"], g["tile_w"], g["m_tiles"], g["n_tiles"]), (info, g)
    assert info["splits"] == (g["splits"] if g["split_tiles"] > 0 else 1), (info, g)
    return outs, info, g, (ho, wo, pt, pl)


def epilogue64(v, scale, shift, residual, act):
    """float64 epilogue of the kernel's order: v*scale + shift (+ residual), then the activation; and the magnitudes its
    three fp32 roundings act on."""
    sc = np.ones(v.shape[-1]) if scale is None else scale.astype(np.float64)
    sh = np.zeros(v.shape[-1]) if shift is None else shift.astype(np.float64)
    a = v * sc
    b = a + sh
    c = b if residual is None else b + residual.astype(np.float64)
    y = np.maximum(c, 0) if act == 1 else np.minimum(np.maximum(c, 0), 6) if act == 2 else c
    return y, np.abs(sc), np.abs(a) + np.abs(b) + np.abs(c)


def ratio(got, want, s, sc=1.0, rnd=0.0):
    """max over elements of |got - want| / (u S |scale|), after taking the epilogue's roundings (2u per op) out."""
    err = np.maximum(np.abs(got.astype(np.float64) - want) - 2 * U * rnd, 0)
    den = U * s * sc
    with np.errstate(invalid="ignore", divide="ignore"):
        r = np.where(den > 0, err / np.where(den > 0, den, 1), np.where(err > 0, np.inf, 0))
    return float(r.max()) if r.size else 0.0


_REF = {}


def reference(key, x, w, stride, pt, pl, ho, wo):
    """(ref64, S) of a case, computed once for all three modes."""
    if key not in _REF:
        if len(_REF) > 2:
            _REF.clear()
        _REF[key] = (ref64(x, w, stride, pt, pl, ho, wo),
                     M.conv64(np.abs(x), np.abs(w), stride, pt, pl, ho, wo))
    return _REF[key]


def make_data(seed, n, h, w, cin, cout, k, positive=False):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((n, h, w, cin))
    wt = rng.standard_normal((k, k, cin, cout)) * np.sqrt(2.0 / (k * k * cin))
    if positive:
        x, wt = np.abs(x), np.abs(wt)
    return rng, x.astype(F), wt.astype(F)


def flattened(g, n, h, w):
    return g["tile_n"] == 1 and g["tile_h"] == 1 and g["tiles_h"] == 1 and g["tile_w"] * g["tiles_w"] >= n * h * w


def odd_tail(g, k, cin, impl):
    return impl != M.TF32X3 and (k * k * cin // 32) % 2 == 1


# name, (n, h, w, cin, cout, k, stride, pad), options, what the case exists to cover (asserted on the geometry g)
PATH_CASES = [
    ("pw_flat_1ntile", (2, 19, 25, 64, 64, 1, 1, "SAME"), {},
     lambda g, i: flattened(g, 2, 19, 25) and g["n_tiles"] == 1),                   # 1x1 flattened to one row, one N tile
    ("pw_flat_2ntiles", (2, 19, 25, 128, 256, 1, 1, "SAME"), {},
     lambda g, i: flattened(g, 2, 19, 25) and g["n_tiles"] == 2),                   # ... two N tiles
    ("c3_s1_tile_n1", (1, 38, 50, 64, 64, 3, 1, "SAME"), {},
     lambda g, i: g["tile_n"] == 1 and g["tile_h"] > 1),                            # 3x3 stride 1, spatial tiles of one image
    ("roi_c3_n20", (20, 7, 7, 64, 64, 3, 1, "SAME"), {},
     lambda g, i: g["tile_n"] > 1),                                                 # RoI head, several RoIs per tile (2 x 7 x 7)
    ("roi_c3_n300", (300, 7, 7, 64, 64, 3, 1, "SAME"), {},
     lambda g, i: g["tile_n"] > 1 and 300 % g["tile_n"] != 0),                      # 300 RoIs: the last tile runs past RoI 300
    ("c3_s2_same_odd", (1, 37, 51, 64, 64, 3, 2, "SAME"), {},
     lambda g, i: True),                                                            # stride 2 SAME, odd h / w
    ("c3_s2_explicit_odd", (1, 37, 51, 64, 64, 3, 2, "EXPLICIT"), {},
     lambda g, i: True),                                                            # stride 2 EXPLICIT (conv2d_same), odd h / w
    ("pw_s2", (1, 37, 51, 64, 128, 1, 2, "SAME"), {},
     lambda g, i: not flattened(g, 1, 19, 26) and g["tiles_w"] * g["tile_w"] < 128),  # 1x1 stride 2: NOT flattened
    ("c3_s4", (1, 41, 53, 64, 64, 3, 4, "SAME"), {},
     lambda g, i: True),                                                            # stride 4 (the plan takes up to 8)
    ("tail_pw_cin32", (1, 38, 50, 32, 64, 1, 1, "SAME"), {},
     lambda g, i: i == M.TF32X3 or odd_tail(g, 1, 32, i)),                          # MobileNet's first pointwise: one box + empty
    ("tail_c3_cin32", (1, 38, 50, 32, 64, 3, 1, "SAME"), {},
     lambda g, i: i == M.TF32X3 or odd_tail(g, 3, 32, i)),                          # 9 boxes: odd tail
    ("tail_c3_cin96", (1, 20, 30, 96, 64, 3, 1, "SAME"), {},
     lambda g, i: i == M.TF32X3 or odd_tail(g, 3, 96, i)),                          # 27 boxes: odd tail
    ("long_fc6_pos", (1, 1, 300, 25088, 128, 1, 1, "SAME"), {"positive": True},
     lambda g, i: g["k_blocks"] == (784 if i == M.TF32X3 else 392)),                # VGG fc6 K = 25088, x, w >= 0
    ("long_c3_512_pos", (1, 19, 25, 512, 128, 3, 1, "SAME"), {"positive": True},
     lambda g, i: g["k_blocks"] == (144 if i == M.TF32X3 else 72)),                 # 3x3x512, x, w >= 0
    ("cout24", (1, 38, 50, 64, 24, 1, 1, "SAME"), {},
     lambda g, i: g["block_n"] > 24 and g["n_tiles"] == 1),                         # cout below block_n
    ("cout36", (1, 20, 30, 64, 36, 3, 1, "SAME"), {},
     lambda g, i: g["block_n"] > 36 and g["n_tiles"] == 1),
    ("cout72", (1, 38, 50, 512, 72, 1, 1, "SAME"), {},
     lambda g, i: g["n_tiles"] * g["block_n"] > 72),                                # RPN head width
    ("cout405_res_relu6", (1, 1, 300, 256, 405, 1, 1, "SAME"), {"epi": 2},
     lambda g, i: g["split_tiles"] == 0),                                           # generic epilogue + residual + ReLU6
    ("cout105_res_relu6", (1, 19, 25, 64, 105, 3, 1, "SAME"), {"epi": 2},
     lambda g, i: g["split_tiles"] == 0),
    ("cout2048", (1, 19, 25, 256, 2048, 1, 1, "SAME"), {},
     lambda g, i: g["n_tiles"] == 16),
    ("bn64", (1, 38, 50, 128, 256, 3, 1, "SAME"), {"block_n": 64},
     lambda g, i: g["block_n"] == 64),                                              # forced block_n, same layer as below
    ("bn128", (1, 38, 50, 128, 256, 3, 1, "SAME"), {"block_n": 128},
     lambda g, i: g["block_n"] == 128),
    ("split_auto_small", (1, 38, 50, 256, 256, 3, 1, "SAME"), {},
     lambda g, i: g["split_tiles"] == g["tiles"] and g["splits"] >= 2),             # too small to fill the GPU: all split
    ("split_auto_ragged", (1, 128, 140, 1536, 64, 1, 1, "SAME"), {},
     lambda g, i: 0 < g["split_tiles"] < g["tiles"] and g["splits"] >= 2),          # ragged last round split
    ("split2_short_epi", (1, 38, 50, 160, 128, 3, 1, "SAME"), {"split_k": 2, "epi": 1},
     lambda g, i: g["splits"] == 2 and g["k_blocks"] % g["kb_per_split"] != 0),     # forced, last split short, tail_reduce epilogue
    ("split3_epi", (1, 38, 50, 160, 128, 3, 1, "SAME"), {"split_k": 3, "epi": 1},
     lambda g, i: g["splits"] == 3 and g["split_tiles"] == g["tiles"]),
    ("split8_short", (1, 38, 50, 160, 128, 3, 1, "SAME"), {"split_k": 8},
     lambda g, i: g["splits"] == 8 and g["k_blocks"] % g["kb_per_split"] != 0),
    ("units_gt_grid", (1, 150, 200, 64, 64, 3, 1, "SAME"), {},
     lambda g, i: g["units"] > g["grid"]),                                          # persistent CTAs walk several units
    ("whole_tile_epi", (1, 38, 50, 64, 256, 1, 1, "SAME"), {"epi": 1},
     lambda g, i: g["split_tiles"] == 0),                                           # vectorised whole-tile epilogue, BN+res+ReLU
]


@pytest.mark.parametrize("mode", MODE_IDS)
@pytest.mark.parametrize("case", PATH_CASES, ids=[c[0] for c in PATH_CASES])
def test_conv_per_element_bounds(cuda, case, mode):
    name, (n, h, w, cin, cout, k, stride, pad), opt, covers = case
    impl = M.MODES[mode]
    from tf_faster_rcnn_b200 import ops
    rng, x, wt = make_data(zlib.crc32(name.encode()), n, h, w, cin, cout, k, opt.get("positive", False))
    epi = opt.get("epi", 0)
    scale = shift = res = None
    if epi:
        ho, wo, _, _ = ops.conv_out_hw(h, w, k, stride, pad)
        scale = rng.uniform(0.5, 1.5, cout).astype(F)
        shift = rng.standard_normal(cout).astype(F)
        res = rng.standard_normal((n, ho, wo, cout)).astype(F)
    (got, got2), info, g, (ho, wo, pt, pl) = conv_run(x, wt, impl, stride, pad, scale, shift, res, epi,
                                                       opt.get("block_n", 0), opt.get("split_k", 0), runs=2)
    assert covers(g, impl), "%s no longer covers its path: %s" % (name, g)
    assert np.array_equal(got.view(np.int32), got2.view(np.int32)), "two runs differ"
    assert np.isfinite(got).all(), "non-finite output (unwritten rows?) %s" % g
    want64, s = reference(name, x, wt, stride, pt, pl, ho, wo)
    mdl, _ = M.model(x, wt, impl, stride, pt, pl, ho, wo)
    y_m, sc, rnd_m = epilogue64(mdl, scale, shift, res, epi)
    y_r, _, rnd_r = epilogue64(want64, scale, shift, res, epi)
    ra = ratio(got, y_m, s, sc, rnd_m)
    rb = ratio(got, y_r, s, sc, rnd_r)
    line = "[%s %s] a=%.2f b=%.2f" % (name, mode, ra, rb)
    if not epi and mode == "f16x3":
        o32 = L.conv2d(x, wt, stride, "SAME") if pad == "SAME" else L.conv2d_same(x, wt, stride)
        line += " oracle_fp32=%.2f" % ratio(o32, want64, s)
    print("\n" + line + " geom=%s" % {kk: g[kk] for kk in ("block_n", "tile_n", "tile_h", "tile_w", "tiles", "split_tiles",
                                                              "splits", "kb_per_split", "units", "grid", "k_blocks")})
    assert ra <= BETA, line
    if mode != "f16x1":
        assert rb <= ALPHA, line
    # the older max-norm criterion, kept
    if mode != "f16x1":
        assert np.abs(got - y_r).max() / np.abs(y_r).max() < 4e-6, line


@pytest.mark.parametrize("mode", ["f16x3", "tf32x3"])
def test_conv_raster_order_and_block_n_are_bit_exact(cuda, mode, monkeypatch):
    """FRCNN_CONV_RASTER (read by decide_geometry at plan creation) only reorders the tiles: m and n give the same bits.
    block_n 64 vs 128 on one layer: reported, and asserted equal only as far as it was measured to hold."""
    impl = M.MODES[mode]
    _, x, wt = make_data(7, 1, 38, 50, 128, 256, 3)
    outs = {}
    for r in ("m", "n"):
        monkeypatch.setenv("FRCNN_CONV_RASTER", r)
        for bn in (64, 128):
            (o,), info, g, _ = conv_run(x, wt, impl, block_n=bn)
            assert g["n_tiles"] > 1 and g["block_n"] == bn
            outs[r, bn] = o
    monkeypatch.delenv("FRCNN_CONV_RASTER")
    for bn in (64, 128):
        assert np.array_equal(outs["m", bn].view(np.int32), outs["n", bn].view(np.int32)), bn
    same = np.array_equal(outs["m", 64].view(np.int32), outs["m", 128].view(np.int32))
    print("\n[%s] block_n 64 vs 128 bit-identical: %s (max diff %.3e)" % (mode, same, np.abs(outs["m", 64] - outs["m", 128]).max()))


def test_f16x1_fails_the_fp32_grade_bound(cuda):
    """Criterion (b) tells fp32-grade from plain fp16: activations sitting 3/8 of an fp16 ulp above an fp16 value, all
    weights positive.  F16X1 drops that 3/8 ulp from every product: >= 100 x ALPHA; F16X3 on the same data meets (b)."""
    rng = np.random.default_rng(11)
    base = rng.uniform(1.0, 1.99, (1, 19, 25, 64)).astype(np.float16).astype(F)
    x = (base + F(0.375 * 2.0 ** -10)).astype(F)
    wt = np.abs(rng.standard_normal((3, 3, 64, 64)) * 0.06).astype(F)
    r = {}
    for mode in ("f16x3", "f16x1"):
        (got,), _, _, (ho, wo, pt, pl) = conv_run(x, wt, M.MODES[mode])
        want, s = reference("f16x1_demo", x, wt, 1, pt, pl, ho, wo)
        r[mode] = ratio(got, want, s)
    print("\n[f16x1 demo] b ratio f16x3=%.2f f16x1=%.1f" % (r["f16x3"], r["f16x1"]))
    assert r["f16x3"] <= ALPHA and r["f16x1"] >= 100 * ALPHA, r


# ---------------------------------------------------------------------------------------------------------------------
# Operand range and non-finite inputs
RANGE_LAYER = (2, 13, 17, 64, 32, 3)          # n, h, w, cin, cout, k: two images, odd map, 3x3 SAME


def _range_run(x, wt, mode):
    impl = M.MODES[mode]
    (got,), _, _, (ho, wo, pt, pl) = conv_run(x, wt, impl)
    want = ref64(x, wt, 1, pt, pl, ho, wo)
    mdl, s = M.model(x, wt, impl, 1, pt, pl, ho, wo)
    return got, want, mdl, s


@pytest.mark.parametrize("mode", ["f16x3", "tf32x3", "f16x1"])
def test_activation_scale_sweep(cuda, mode):
    """|x| drawn from [2^e, 2^(e+1)) with random signs.  (a) everywhere; (b) where the mode carries the operands to 2^-22
    (F16X3: 2^-14 <= |x| < 65520, TF32X3: the whole sweep, 2^-100 .. 2^100); below F16X3's range the model states the
    loss: |model - ref64| <= (2^(-36-e) + 2^-22) * S."""
    n, h, w, cin, cout, k = RANGE_LAYER
    rng, _, wt = make_data(21, n, h, w, cin, cout, k)
    exps = [-24, -20, -16, -14, -10, 0, 10, 14, 15] if mode != "tf32x3" else [-100, -60, -24, -14, 0, 14, 15, 60, 100]
    res = {}
    for e in exps:
        mag = rng.uniform(1.0, 2.0, (n, h, w, cin)) * 2.0 ** e
        if e == 15 and mode != "tf32x3":
            mag = rng.uniform(2.0 ** 15, 65503.0, (n, h, w, cin))
            mag.flat[rng.integers(mag.size)] = 65503.99
        x = (mag * rng.choice([-1.0, 1.0], mag.shape)).astype(F)
        got, want, mdl, s = _range_run(x, wt, mode)
        assert np.isfinite(got).all(), e
        res[e] = (ratio(got, mdl, s), ratio(got, want, s), float(np.max(np.abs(mdl - want) / s / 2.0 ** (-36 - e))))
        print("\n[sweep %s 2^%d] a=%.2f b=%.2f" % (mode, e, res[e][0], res[e][1]))
    for e, (ra, rb, loss) in res.items():
        subnormal = mode != "tf32x3" and e < -14
        assert ra <= (BETA_SUBNORMAL if subnormal else BETA), (e, ra)
        if mode == "tf32x3" or (mode == "f16x3" and e >= -14):
            assert rb <= ALPHA, (e, rb)
        elif mode == "f16x3":
            assert loss <= 1.0 + 2.0 ** (e + 14), (e, loss)      # |model - ref64| <= (2^(-36-e) + 2^-22) S


@pytest.mark.parametrize("mode", ["f16x3", "tf32x3"])
def test_weight_channel_spread_and_layer_scale(cuda, mode):
    """Channel c scaled by 2^-c (c = 0..40, each channel's max |w| normalised first), one layer exponent for all: (b) for
    channels within 2^-27 of the layer max, (a) for all.  The whole layer scaled by 1e-6, 300 and 1e-20: (a) and (b)."""
    impl = M.MODES[mode]
    rng = np.random.default_rng(31)
    x = rng.standard_normal((1, 13, 17, 64)).astype(F)
    wt = rng.standard_normal((3, 3, 64, 41))
    wt = (wt / np.abs(wt).max(axis=(0, 1, 2)) * 2.0 ** -np.arange(41)).astype(F)
    got, want, mdl, s = _range_run(x, wt, mode)
    ra = [ratio(got[..., c], mdl[..., c], s[..., c]) for c in range(41)]
    rb = [ratio(got[..., c], want[..., c], s[..., c]) for c in range(41)]
    print("\n[channel spread %s] a max %.2f; b by channel %s" % (mode, max(ra), " ".join("%.1f" % v for v in rb)))
    assert max(ra[:28]) <= BETA, ra
    assert max(ra[28:]) <= (BETA_SUBNORMAL if mode == "f16x3" else BETA), ra     # f16: hi plane subnormal from 2^-28 on
    assert max(rb[:28]) <= ALPHA, rb
    for f in (1e-6, 300.0, 1e-20):
        w2 = (rng.standard_normal((3, 3, 64, 32)) * 0.06 * f).astype(F)
        got, want, mdl, s = _range_run(x, w2, mode)
        ra, rb = ratio(got, mdl, s), ratio(got, want, s)
        print("[layer scale %s %g] a=%.2f b=%.2f" % (mode, f, ra, rb))
        assert ra <= BETA and rb <= ALPHA, (f, ra, rb)


def test_weight_exponent_beyond_100_is_refused(cuda):
    """max|w| = 1e-30 needs wexp = 113: PackedConv raises frcnn_pack_conv_weights' argument error before any launch."""
    from tf_faster_rcnn_b200 import ops, _native as N
    w = np.full((3, 3, 32, 8), 1e-30, F)
    with pytest.raises(RuntimeError, match="wexp=113 out of range"):
        ops.PackedConv(w, impl=N.CONV_F16X3)


NAN_QUIET, NAN_DEVICE = np.int32(0x7fc00000).view(F), np.int32(0x7fffffff).view(F)   # numpy's NaN, the device's own


@pytest.mark.parametrize("mode", ["f16x3", "tf32x3", "f16x1"])
@pytest.mark.parametrize("bad", ["nan", "inf", "big"])
def test_non_finite_activations(cuda, mode, bad):
    """Non-finite (or, in the f16 modes, out-of-range) activations at known pixels: exactly the outputs whose receptive field
    holds one are non-finite, and every other output still meets (b) ((a) for F16X1) -- nothing leaks into other tiles.
    'big' = finite |x| >= 65536: non-finite in F16X3 / F16X1 (never a finite wrong value), plain (b) in TF32X3."""
    n, h, w, cin, cout, k = RANGE_LAYER
    rng, x, wt = make_data(41, n, h, w, cin, cout, k)
    vals = {"nan": [NAN_QUIET, NAN_DEVICE, -NAN_DEVICE], "inf": [np.inf, -np.inf, np.inf],
            "big": [65536.0, -1e5, 3.0e38]}[bad]
    places = [(0, 0, 0, 5), (0, 6, 9, 63), (1, 12, 16, 0)]                  # corner, interior, opposite corner of image 1
    xc = x.copy()
    for (b, i, j, c), v in zip(places, vals):
        x[b, i, j, c] = F(v)
        xc[b, i, j, c] = 0.0
    impl = M.MODES[mode]
    (got,), _, _, (ho, wo, pt, pl) = conv_run(x, wt, impl)
    ind = np.zeros((n, h, w, 1))
    for b, i, j, _ in places:
        ind[b, i, j, 0] = 1.0
    hit = ref64(ind, np.ones((k, k, 1, 1)), 1, pt, pl, ho, wo)[..., 0] > 0       # receptive field holds a bad pixel
    hit = np.repeat(hit[..., None], cout, axis=-1)
    expect_nonfinite = hit if (bad != "big" or mode != "tf32x3") else np.zeros_like(hit)
    print("\n[%s %s] non-finite outputs %d, expected %d" % (bad, mode, (~np.isfinite(got)).sum(), expect_nonfinite.sum()))
    assert np.array_equal(~np.isfinite(got), expect_nonfinite), "finite/non-finite pattern differs from the receptive fields"
    want, s = (ref64(x, wt, 1, pt, pl, ho, wo), M.conv64(np.abs(x), np.abs(wt), 1, pt, pl, ho, wo)) if not \
        expect_nonfinite.any() else (ref64(xc, wt, 1, pt, pl, ho, wo), M.conv64(np.abs(xc), np.abs(wt), 1, pt, pl, ho, wo))
    keep = ~expect_nonfinite
    if mode == "f16x1":
        mdl, s = M.model(xc, wt, impl, 1, pt, pl, ho, wo)
        assert ratio(got[keep], mdl[keep], s[keep]) <= BETA
    else:
        assert ratio(got[keep], want[keep], s[keep]) <= ALPHA


def test_f16_edge_just_below_overflow(cuda):
    """65504 <= |x| < 65520 still rounds to a finite fp16 hi: F16X3 stays fp32-grade there."""
    n, h, w, cin, cout, k = RANGE_LAYER
    rng, x, wt = make_data(43, n, h, w, cin, cout, k)
    x[0, 3, 3, :8] = F(65519.0) * np.sign(rng.standard_normal(8)).astype(F)
    x[1, 5, 7, :8] = F(65504.0)
    got, want, mdl, s = _range_run(x, wt, "f16x3")
    assert np.isfinite(got).all() and ratio(got, want, s) <= ALPHA
