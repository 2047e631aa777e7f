"""The models and references of front_ref64.py agree with the oracle and with float64 truth, each plausible kernel mistake
below fails its comparator, and every NMS case forces the path it names.  CPU only."""
import numpy as np
import pytest

import front_ref64 as R
from stage_ref64 import check_exact

F = np.float32
MEANS = (102.9801, 115.9465, 122.7717)       # cfg.PIXEL_MEANS (BGR)


def within(got, truth, bound):
    return bool((np.abs(np.asarray(got, np.float64) - truth) <= bound).all())


# ---- greedy NMS -----------------------------------------------------------------------------------------------------------
NMS_CASES = {c[0]: c[1:] for c in R.nms_cases()}


@pytest.mark.parametrize("mode", sorted(R.MODES))
@pytest.mark.parametrize("name", sorted(NMS_CASES))
def test_nms_model_matches_oracle_and_forces_its_path(name, mode):
    boxes, thr, max_out, expect = NMS_CASES[name]
    flags = R.MODES[mode]
    kept, st = R.greedy_nms_model(boxes, thr, flags, max_out)
    want = R.oracle_keep(boxes, np.full(boxes.shape[0], 0.5, F), thr, flags, max_out)
    check_exact(kept, want, "%s %s survivors" % (name, mode))
    R.check_path(st, kept, expect, "%s %s" % (name, mode))


def test_nms_cases_cover_every_path():
    st = [R.greedy_nms_model(b, thr, R.MODES["tf"], mo)[1] for b, thr, mo, _ in NMS_CASES.values()]
    assert sum(s["cuts"] for s in st) >= 3                        # the 256-survivor cut
    assert all(s["tpc4"] >= 1 for s in st)                        # 4 threads per candidate (every first round)
    assert sum(s["tpc1"] for s in st) >= 4                        # 1 thread per candidate
    assert sum(s["maxout_mid_chunk"] for s in st) >= 1            # max_out inside a chunk
    assert max(s["rounds"] for s in st) >= 6                      # the kept set grows across rounds


@pytest.mark.parametrize("mode", sorted(R.MODES))
def test_nms_exact_threshold(mode):
    thr, cases = R.exact_threshold_cases()
    boxes, survivors = cases[mode]
    kept, _ = R.greedy_nms_model(boxes, thr, R.MODES[mode], 10)
    assert list(kept) == survivors
    assert list(R.oracle_keep(boxes, np.asarray([0.9, 0.8], F), thr, R.MODES[mode], 10)) == survivors


@pytest.mark.parametrize("mutant,cases,mode", [
    ("resolve_suppressed", ("chain_cut_256", "chain_cut_255"), "gpu_nms"),
    ("cut_skip", ("cut",), "cpu_nms"),
    ("cut_repeat", ("point",), "tf")])
def test_nms_mutants_fail(mutant, cases, mode):
    flags = R.MODES[mode]
    for name in cases:
        boxes, thr, max_out = (R.point_cut_case(), 0.5, 1024) if name == "point" else NMS_CASES[name][:3]
        want = R.oracle_keep(boxes, np.full(boxes.shape[0], 0.5, F), thr, flags, max_out)
        assert np.array_equal(R.greedy_nms_model(boxes, thr, flags, max_out)[0], want)
        with pytest.raises(AssertionError):
            check_exact(R.greedy_nms_model(boxes, thr, flags, max_out, mutant=mutant)[0], want, mutant)


# ---- score sort -----------------------------------------------------------------------------------------------------------
def sort_key_sets():
    rng = np.random.default_rng(4)
    sets = {"special": R.special_keys(rng, 5000), "equal": np.full(3000, 0.25, F)}
    for byte in range(4):
        sets["byte%d" % byte] = R.one_byte_keys(rng, 3000, byte)
    return sets


def test_sort_reference_order_of_specials():
    bits = np.array([0x3f800000, 0x7f800000, 0x7fc00000, 0xff800000, 0xffc00000, 0x00000000, 0x80000000, 0x00000001,
                     0x80000001, 0x3f800000], np.uint32)
    keys = bits.view(F)                  # 1, +Inf, +NaN, -Inf, -NaN, +0, -0, +min subnormal, -min subnormal, 1 (tie)
    order, sk = R.sort_ref(keys)
    assert list(order) == [2, 1, 0, 9, 7, 5, 6, 8, 3, 4]
    assert np.array_equal(sk.view(np.uint32), bits[order])
    assert np.array_equal(R.from_bits(R.desc_bits(keys)).view(np.uint32), bits)


@pytest.mark.parametrize("name", sorted(sort_key_sets()))
def test_radix_model_matches_reference(name):
    keys = sort_key_sets()[name]
    check_exact(R.radix_model(keys), R.sort_ref(keys)[0], name)


@pytest.mark.parametrize("mutant", ["ties_reversed", "shift"])
def test_sort_mutants_fail(mutant):
    failed = []
    for name, keys in sort_key_sets().items():
        failed.append(not np.array_equal(R.radix_model(keys, mutant), R.sort_ref(keys)[0]))
    assert any(failed), mutant


# ---- preprocess -------------------------------------------------------------------------------------------------------------
GEOMS = {g[0]: g[1:] for g in R.preprocess_geometries() + R.tta_geometries()}
CV2_MAX_DIFF = 2 * 2.0 ** -16     # 2 ulp of |pixel - mean| in [128, 256): the largest |cv2 - model| over these geometries


@pytest.mark.parametrize("hflip", [False, True])
@pytest.mark.parametrize("name", sorted(GEOMS))
def test_preprocess_model_and_cv2_within_bound(name, hflip):
    cv2 = pytest.importorskip("cv2")
    h0, w0, fx, fy, H, W = GEOMS[name]
    im = R.edge_image(np.random.default_rng(h0 * 7 + w0), h0, w0)
    model = R.preprocess_model(im, MEANS, fx, fy, H, W, hflip)
    truth, bound = R.preprocess_truth(im, MEANS, fx, fy, H, W, hflip)
    assert within(model, truth, bound), "max err/bound %.3g" % (np.abs(model - truth) / bound).max()
    px = (im[:, ::-1] if hflip else im).astype(F)
    px -= np.asarray(MEANS)                                      # the host path: float32 -= float64, rounded once
    host = cv2.resize(px, None, None, fx=fx, fy=fy, interpolation=cv2.INTER_LINEAR).reshape(H, W, 3)
    assert within(host, truth, bound), "cv2: max err/bound %.3g" % (np.abs(host - truth) / bound).max()
    assert np.abs(host - model).max() <= CV2_MAX_DIFF


@pytest.mark.parametrize("mutant,name,fails", [
    ("frac32", "fx!=fy", "bound"), ("frac32", "aspect", "bound"), ("fma", "x2", "exact"),
    ("right_keeps_frac", "3x1", "exact"), ("right_keeps_frac", "1x1", "exact"), ("flip_off", "x1", "bound")])
def test_preprocess_mutants_fail(mutant, name, fails):
    h0, w0, fx, fy, H, W = GEOMS[name]
    im = R.edge_image(np.random.default_rng(h0 * 7 + w0), h0, w0)
    hflip = mutant == "flip_off"
    model = R.preprocess_model(im, MEANS, fx, fy, H, W, hflip)
    bad = R.preprocess_model(im, MEANS, fx, fy, H, W, hflip, **{mutant: 1 if mutant == "flip_off" else True})
    if fails == "exact":
        with pytest.raises(AssertionError):
            check_exact(bad, model, mutant)
    else:
        truth, bound = R.preprocess_truth(im, MEANS, fx, fy, H, W, hflip)
        assert within(model, truth, bound) and not within(bad, truth, bound)


# ---- SIMT convolutions and max pool -----------------------------------------------------------------------------------------
def test_conv_first_bound_rejects_shifted_padding():
    rng = np.random.default_rng(8)
    x = (rng.standard_normal((1, 23, 37, 3)) * 50).astype(F)
    w = (rng.standard_normal((7, 7, 3, 64)) * 0.01).astype(F).transpose(3, 2, 0, 1)
    ho, wo, pt, pl = 12, 19, 3, 3                                 # ResNet conv1: 7x7/2, explicit pad 3
    y, bound = R.fma_chain_ref(x, w, 2, pt, pl, ho, wo, 147, None, None, 1)
    assert within(y.astype(F), y, bound)
    shifted = np.maximum(R.conv64_nhwc(x, w, 2, pt + 1, pl, ho, wo), 0).astype(F)
    assert not within(shifted, y, bound)


@pytest.mark.parametrize("mode,k,s", [("SAME", 2, 2), ("ZEROPAD1", 3, 2), ("VALID", 1, 2)])
def test_max_pool_model_matches_oracle(mode, k, s):
    rng = np.random.default_rng(k)
    x = -np.abs(rng.standard_normal((3, 7, 9, 8))).astype(F) - F(0.5)        # all negative: the ZEROPAD1 zeros win at the border
    x[0, 0, 0, :2] = [np.inf, -np.inf]
    x[2, 6, 8, 4:6] = [-np.inf, np.inf]
    ho, wo, pt, pl, neg = R.pool_geometry(7, 9, k, s, mode)
    want = R.pool_oracle(x, k, s, mode)
    check_exact(R.max_pool_model(x, k, s, pt, pl, ho, wo, neg), want, mode)
    if mode == "ZEROPAD1":
        with pytest.raises(AssertionError):
            check_exact(R.max_pool_model(x, k, s, pt, pl, ho, wo, neg, zeros_as_ninf=True), want, "pad zeros as -Inf")


def test_max_pool_nan_rule_differs_from_oracle():
    """fmaxf drops a NaN from the window; the oracle (torch max_pool2d) propagates it."""
    x = np.arange(16, dtype=F).reshape(1, 2, 2, 4)
    x[0, 1, 1, 0] = np.nan
    model = R.max_pool_model(x, 2, 2, 0, 0, 1, 1, True)
    assert model[0, 0, 0, 0] == 8.0
    assert np.isnan(R.pool_oracle(x, 2, 2, "SAME")[0, 0, 0, 0])
