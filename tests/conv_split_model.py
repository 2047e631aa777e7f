"""CPU model of the operand split of `conv_gemm_kernel` (plain numpy + float64 torch convolutions, no GPU).

Every operand is rounded exactly as the device rounds it; products and sums are then taken in float64, so the model is
the kernel's result without its fp32 summation error:

    model(x, w) = sum a_hi*b_hi + (a_lo*b_hi + a_hi*b_lo)          (lo planes unscaled: LO_SCALE folded in)
    S(x, w)     = sum |x|*|w|                                      (per output element; the scale of every error bound)

  F16X3  weights     v = w * 2^e (fp32, e = ops.weight_exponent), hi = RN_f16(v), lo = RN_f16((v - hi) * 2^11)
                     (pack_weights_f16_kernel), undone by out_mult = 2^-e
         activations hi = RN_f16(x), lo = RN_f16((x - hi) * 2^11) in fp32 arithmetic (conv_gemm.cu, pack_f16x2_rn); the
                     conversion does not saturate, so |x| >= 65520 and +-Inf give an infinite hi.  `saturate=True` models the
                     earlier cvt.rn.satfinite conversion, which clamped both planes to +-65504.
  TF32X3 both        hi = RNA_tf32(x), lo = RNA_tf32(x - hi): nearest, ties away from zero, 10 explicit mantissa bits
                     (to_tf32 / cvt.rna; the formula of tools/numerics_split_schemes.round_mantissa)
  F16X1  both        the F16X3 hi planes only
"""
import numpy as np
import torch

F16X3, TF32X3, F16X1 = 0, 1, 2          # frcnn_b200.h FRCNN_CONV_*
MODES = {"f16x3": F16X3, "tf32x3": TF32X3, "f16x1": F16X1}
U = 2.0 ** -24                           # fp32 unit roundoff
LO_SCALE = 2.0 ** -11                    # the fp16 lo planes are stored scaled by 2^11


def weight_exponent(w):
    from tf_faster_rcnn_b200 import ops
    return ops.weight_exponent(w)


def rna_tf32(x):
    """fp32 -> tf32 (10 explicit mantissa bits), nearest, ties away from zero, on the bit pattern; a NaN stays a NaN (as
    through cvt.rna: the bit arithmetic alone would carry a NaN with a full payload, such as 0x7fffffff, to -0.0)."""
    x = np.asarray(x, np.float32)
    u = x.view(np.uint32).astype(np.uint64)
    r = ((((u + (1 << 12)) >> 13) << 13).astype(np.uint32)).view(np.float32)
    return np.where(np.isnan(x), x, r)


def rn_f16(x, saturate=False):
    """fp32 -> fp16 value (as fp32), round to nearest even; IEEE overflow to +-Inf unless `saturate` (satfinite: +-65504)."""
    with np.errstate(over="ignore", invalid="ignore"):
        h = np.asarray(x, np.float32).astype(np.float16).astype(np.float32)
    if saturate:
        h = np.where(np.isinf(h), np.copysign(np.float32(65504.0), h), h).astype(np.float32)
    return h


def split_activations(x, mode, saturate=False):
    """(hi, lo) as float64 with x ~= hi + lo, exactly the values the kernel multiplies (lo unscaled)."""
    x = np.asarray(x, np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        if mode == TF32X3:
            hi = rna_tf32(x)
            lo = rna_tf32(np.float32(x - hi))
            return hi.astype(np.float64), lo.astype(np.float64)
        hi = rn_f16(x, saturate)
        if mode == F16X1:
            return hi.astype(np.float64), np.zeros(x.shape, np.float64)
        lo = rn_f16(np.float32(np.float32(x - hi) * np.float32(2048.0)), saturate)
        return hi.astype(np.float64), lo.astype(np.float64) * LO_SCALE


def split_weights(w, mode):
    """(hi, lo) as float64 with w ~= hi + lo: the packed planes with the layer scaling 2^e undone."""
    w = np.asarray(w, np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        if mode == TF32X3:
            hi = rna_tf32(w)
            lo = rna_tf32(np.float32(w - hi))
            return hi.astype(np.float64), lo.astype(np.float64)
        e = weight_exponent(w)
        v = np.float32(w * np.float32(np.ldexp(1.0, e)))         # frcnn_pack_conv_weights accepts |e| <= 100
        hi = rn_f16(v)
        lo = rn_f16(np.float32(np.float32(v - hi) * np.float32(2048.0)))
        un = 2.0 ** -e
        if mode == F16X1:
            return hi.astype(np.float64) * un, np.zeros(w.shape, np.float64)
        return hi.astype(np.float64) * un, lo.astype(np.float64) * (LO_SCALE * un)


def conv64(x, w, stride, pad_t, pad_l, ho, wo):
    """float64 convolution of NHWC x with HWIO w; zero padding pad_t / pad_l before, whatever is needed after."""
    xt = torch.from_numpy(np.ascontiguousarray(x, np.float64)).permute(0, 3, 1, 2)
    wt = torch.from_numpy(np.ascontiguousarray(w, np.float64)).permute(3, 2, 0, 1)
    kh, kw = w.shape[:2]
    h, wd = x.shape[1:3]
    pb = max((ho - 1) * stride + kh - h - pad_t, 0)
    pr = max((wo - 1) * stride + kw - wd - pad_l, 0)
    xt = torch.nn.functional.pad(xt, (pad_l, pr, pad_t, pb))
    y = torch.nn.functional.conv2d(xt, wt, None, stride=stride)
    return y.permute(0, 2, 3, 1).numpy()[:, :ho, :wo]


def model(x, w, mode, stride, pad_t, pad_l, ho, wo, saturate=False):
    """(model output, S): the kernel's operands, exact products, float64 sums."""
    xh, xl = split_activations(x, mode, saturate)
    wh, wl = split_weights(w, mode)
    g = lambda a, b: conv64(a, b, stride, pad_t, pad_l, ho, wo)
    m = g(xh, wh)
    if mode != F16X1:
        m = m + g(xl, wh) + g(xh, wl)
    s = g(np.abs(x.astype(np.float64)), np.abs(w.astype(np.float64)))
    return m, s


def activation_error(x, mode, saturate=False):
    """|x - (hi + lo)| / |x| per element (float64)."""
    hi, lo = split_activations(x, mode, saturate)
    x64 = np.asarray(x, np.float64)
    with np.errstate(invalid="ignore"):
        return np.abs(x64 - (hi + lo)) / np.abs(x64)
