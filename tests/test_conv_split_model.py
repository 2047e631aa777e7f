"""The documented operand ranges of the dense kernel's three arithmetic modes, pinned on the CPU model of its operand split
(tests/conv_split_model.py: every rounding the device makes, nothing else).  The GPU tests (test_conv_gpu.py) then hold the
kernel to this model element by element."""
import ctypes as C

import numpy as np
import pytest

import conv_split_model as M
from tf_faster_rcnn_b200 import _native as N


def binade(e, step=1, sign=1.0):
    """Every fp32 value (or every `step`-th) in [2^e, 2^(e+1))."""
    m = np.arange(0, 1 << 23, step, dtype=np.uint32)
    x = ((np.uint32(e + 127) << np.uint32(23)) | m).view(np.float32)
    return x if sign > 0 else -x


def worst(x, mode, saturate=False):
    r = M.activation_error(x, mode, saturate)
    assert np.isfinite(r).all()
    return float(r.max())


def lg(v):
    """log2 to 2 decimals: a worst case of 2^-25 / (2^-14 * (1 + 2^-23)) reads as -22"""
    return round(float(np.log2(v)), 2)


def test_f16x3_activations_keep_2m22_over_the_documented_range():
    """Every fp32 activation with 2^-14 <= |x| <= 65504 is carried to <= 2^-22 relative (every positive value; the
    negative ones sampled: round-to-nearest-even is symmetric); from 2^-13 up the worst case is 2^-23.
    65504 < |x| < 65520 still rounds to a finite hi and is exact to 2^-23 as well."""
    for e in range(-14, 16):
        x = binade(e)
        if e == 15:
            x = x[x <= 65504.0]
        for xs in (x, -x[::97]):
            w = worst(xs, M.F16X3)
            assert w <= 2.0 ** -22, (e, w)
            assert lg(w) == (-22 if e == -14 else -23), (e, np.log2(w))
    x = np.float32([65504.0, 65505.0, 65519.99])
    assert worst(x, M.F16X3) <= 2.0 ** -23


def test_f16x3_activation_loss_below_2m14():
    """Below 2^-14 the hi plane is subnormal: the worst relative error of binade [2^e, 2^(e+1)) is exactly 2^(-36-e), until
    the lo plane underflows too (the measured curve; a change to the split moves it)."""
    curve = {}
    for e in range(-26, -13):
        curve[e] = worst(binade(e, step=3), M.F16X3)
    for e, w in curve.items():
        assert lg(w) == -36 - e, (e, np.log2(w))
    # the table of DESIGN §4.1
    assert [lg(curve[e]) for e in (-14, -16, -20, -24)] == [-22, -20, -16, -12]
    x = np.float32([2.0 ** -36, 2.0 ** -40, 1e-45])                   # below 2^-35 the lo plane is zero too: x is lost
    assert (M.activation_error(x, M.F16X3) == 1.0).all()


def test_f16_activations_out_of_range_are_infinite_not_clamped():
    """|x| >= 65520 and +-Inf: the conversion overflows to Inf (hi = +-Inf, lo = -+Inf or NaN), so every product with it is
    non-finite.  The earlier saturating conversion turned all of them into the finite +-65535.98."""
    x = np.float32([65520.0, 65536.0, 1e5, 3e38, np.inf, -65520.0, -1e6, -np.inf])
    for mode in (M.F16X3, M.F16X1):
        hi, lo = M.split_activations(x, mode)
        assert np.isinf(hi).all() and (np.sign(hi) == np.sign(x)).all()
    hi, lo = M.split_activations(x, M.F16X3, saturate=True)
    assert np.isfinite(hi + lo).all()
    big = np.abs(x) >= 65536.0
    assert (np.abs(hi + lo)[big] == 65504.0 + 65504.0 / 2048.0).all()              # 65535.98, whatever x was
    hi, lo = M.split_activations(np.float32([np.nan]), M.F16X3)
    assert np.isnan(hi).all()


def test_tf32x3_activations_keep_2m22_over_the_fp32_range():
    """TF32X3: <= 2^-22 relative from 2^-115 up to the tf32 overflow threshold (2^-23 from 2^-113; both signs, every binade
    sampled, two binades exhaustive).  Below that the lo plane is subnormal: the worst case of binade e is 2^(-137-e), 2^-11
    at 2^-126.  From (2 - 2^-11) * 2^127 on, hi rounds to Inf."""
    for e in (-3, 40):
        assert lg(worst(binade(e), M.TF32X3)) == -23
    for e in range(-115, 128):
        x = binade(e, step=1021)
        x = np.concatenate([x, -x, binade(e)[-3:]])
        if e == 127:
            x = x[np.abs(x) < np.float32(2.0 ** 127 * (2.0 - 2.0 ** -11))]
        w = worst(x, M.TF32X3)
        assert w <= 2.0 ** -22 and (e < -113 or lg(w) == -23), (e, np.log2(w))
    for e in range(-126, -113):
        assert lg(worst(binade(e, step=7), M.TF32X3)) == -137 - e, e
    hi, _ = M.split_activations(np.float32([2.0 ** 127 * (2.0 - 2.0 ** -11), np.finfo(np.float32).max]), M.TF32X3)
    assert np.isinf(hi).all()


def test_f16x1_is_fp16_grade():
    """F16X1 keeps the hi plane only: 2^-11 worst, about 2^-12 on average, over the normal fp16 range."""
    for e in (-14, 0, 14):
        r = M.activation_error(binade(e), M.F16X1)
        assert lg(r.max()) == -11 and 2.0 ** -13 < r.mean() < 2.0 ** -12, (e, r.max(), r.mean())


@pytest.mark.parametrize("layer_max", [1.0, 3.7e-5, 812.0, 2.0 ** -60])
def test_weight_channels_27_binades_below_the_layer_max(layer_max):
    """ops.weight_exponent puts max|w| in [2^13, 2^14): weights down to 2^-27 below the layer's largest keep 2^-22 relative
    (the F16X3 planes, scaling undone exactly); one binade further a power-of-two layer max already loses a bit."""
    lm = np.float32(layer_max)
    for b in range(0, 28):
        w = (binade(0, step=257) * np.float32(lm) * np.float32(2.0 ** -(b + 1))).astype(np.float32)
        w = np.concatenate([[lm], w, -w]).astype(np.float32)
        hi, lo = M.split_weights(w, M.F16X3)
        r = np.abs(w.astype(np.float64) - (hi + lo)) / np.abs(w.astype(np.float64))
        keep = np.abs(w) >= lm * 2.0 ** -27
        assert r[keep].max() <= 2.0 ** -22, (layer_max, b, np.log2(r[keep].max()))
    w = np.concatenate([[lm], binade(0, step=257) * np.float32(lm) * np.float32(2.0 ** -28)]).astype(np.float32)
    hi, lo = M.split_weights(w, M.F16X3)
    r = np.abs(w.astype(np.float64) - (hi + lo)) / np.abs(w.astype(np.float64))
    if layer_max in (1.0, 2.0 ** -60):              # power-of-two max: 2^-28 below it is v in [2^-15, 2^-14)
        assert lg(r.max()) == -21


def test_weight_exponent_out_of_range_is_rejected_before_any_launch():
    """A layer whose max|w| needs wexp > 100 (max|w| = 1e-30 -> 113) is refused by frcnn_pack_conv_weights' argument check,
    which runs before any CUDA call (dummy pointers here: nothing is dereferenced)."""
    w = np.full((3, 3, 32, 8), 1e-30, np.float32)
    e = M.weight_exponent(w)
    assert e == 113
    p = C.c_void_p(16)
    rc = N.lib().frcnn_pack_conv_weights(p, p, p, 3, 3, 32, 8, e, None)
    assert rc != 0 and "wexp=113 out of range" in N.last_error()
    assert M.weight_exponent(np.full((1, 1, 32, 8), 1e-20, np.float32)) <= 100


def test_model_reproduces_a_hand_computed_dot_product():
    """The model's convolution on a 1x1 layer equals sum(hi*hi + lo*hi + hi*lo) computed by hand, and S = sum|x||w|."""
    rng = np.random.default_rng(0)
    x = rng.standard_normal((1, 1, 1, 64)).astype(np.float32)
    w = rng.standard_normal((1, 1, 64, 3)).astype(np.float32)
    for mode in (M.F16X3, M.TF32X3, M.F16X1):
        m, s = M.model(x, w, mode, 1, 0, 0, 1, 1)
        xh, xl = M.split_activations(x[0, 0, 0], mode)
        wh, wl = M.split_weights(w[0, 0], mode)
        want = xh @ wh + xl @ wh + xh @ wl
        assert np.allclose(m[0, 0, 0], want, rtol=1e-14, atol=0)
        assert np.allclose(s[0, 0, 0], np.abs(x[0, 0, 0]).astype(np.float64) @ np.abs(w[0, 0]).astype(np.float64), rtol=1e-14)
        exact = x[0, 0, 0].astype(np.float64) @ w[0, 0].astype(np.float64)
        bound = {M.F16X3: 2.0 ** -21, M.TF32X3: 2.0 ** -21, M.F16X1: 2.0 ** -10}[mode]
        assert (np.abs(m[0, 0, 0] - exact) <= bound * s[0, 0, 0]).all()
