"""The Soft-NMS definition against a float64 restatement of Detectron's cpu_soft_nms (post_ref64.py): the C oracle and the numpy
model of the kernel lie within the float64 comparator on the random families and on every edge case, and equal each other bit
for bit, NaN and +Inf scores included; one deliberate mistake each in the oracle fails the comparator; the features gather
reference on hand cases."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import post_ref64 as R  # noqa: E402
import soft_nms_model as SM  # noqa: E402
import soft_nms_oracle as SO  # noqa: E402
from test_soft_nms import PARAMS, make_set, same  # noqa: E402

F = np.float32


def check_both(d, params, what):
    """Oracle == model bit for bit, and both within the float64 comparator -> the reference."""
    want = SO.soft_nms_c(d, *params)
    assert same(want, SM.soft_nms_model(d, *params)), "%s: oracle and model differ" % what
    ref = R.soft_nms64(d, *params)
    R.check_soft64(*want, d, ref, what)
    return ref


def test_nan_head_rule():
    """The four rows of the NaN finding: oracle, model and float64 restatement all take [0, 3, 2, 1]."""
    for name, fn in (("oracle", SO.soft_nms_c), ("model", SM.soft_nms_model)):
        rows, keep = fn(R.NAN_ROWS, "linear", 0.5, 0.3, 0.001)
        assert keep.tolist() == R.NAN_KEEP, name
        assert rows.tobytes() == R.NAN_ROWS[R.NAN_KEEP].tobytes(), name
    assert R.soft_nms64(R.NAN_ROWS, "linear", 0.5, 0.3, 0.001).keep.tolist() == R.NAN_KEEP


def test_random_families_within_float64():
    rng = np.random.default_rng(64)
    families = ("clustered", "tied", "duplicates", "degenerate", "mixed")
    settled = total = 0
    worst = 0.0
    for it in range(72):
        n = int(rng.integers(1, 121))
        d = make_set(rng, n, families[it % len(families)])
        params = PARAMS[it % len(PARAMS)]
        want = SO.soft_nms_c(d, *params)
        assert same(want, SM.soft_nms_model(d, *params)), (it, params)
        ref = R.soft_nms64(d, *params)
        worst = max(worst, R.check_soft64(*want, d, ref, "set %d %s" % (it, params)))
        settled += ref.settled
        total += want[1].shape[0]
    print("\n[soft-NMS random families] %d of %d selections settled; max |s32 - s64| / bound %.3f" % (settled, total, worst))
    assert settled > 0.8 * total                     # the comparison is not vacuous


@pytest.mark.parametrize("edge", sorted(R.EDGES))
@pytest.mark.parametrize("n", [1, 2, 96, 301])
def test_edges_within_float64(edge, n):
    rng = np.random.default_rng(n)
    d, params = R.EDGES[edge](rng, n)
    assert d.shape == (n, 5) and d.dtype == F
    ref = check_both(d, params, "%s n=%d" % (edge, n))
    if edge not in R.NONFINITE:
        assert ref.complete, (edge, ref.settled, ref.margins)       # exact inputs: every decision decided


def test_edges_take_their_path():
    """Each generator reaches the edge it names."""
    rng = np.random.default_rng(0)
    run = lambda name, n=96: SO.soft_nms_c(*((lambda d, p: (d,) + p)(*R.EDGES[name](rng, n))))  # noqa: E731
    rows, keep = run("iou_at_nt")
    b1 = keep % 3 == 1
    assert b1.sum() == 32 and (rows[b1, 4] == R.iou_at_nt(rng, 96)[0][keep[b1], 4]).all()          # IoU = nt: untouched
    rows, keep = run("decay_to_thresh")
    assert (keep % 3 != 2).all() and (rows[keep % 3 == 1, 4] == F(0.125)).all()
    assert run("all_pruned_first")[1].shape == (1,)
    d, params = R.hole_table(rng, 1024)
    want = SO.soft_nms_c(d, *params)
    assert want[1].shape[0] == 513 and want[1][:3].tolist() == [0, 1023, 1022]       # 511 holes filled from the top down
    rows, keep = run("no_overlap")
    assert keep.shape[0] == 96 and (rows[:, 4] < F(0.001)).sum() == 20
    rows, keep = run("signed_zeros")
    assert (np.signbit(rows[:, 4]) & (rows[:, 4] == 0)).any()
    d, params = R.sigma_huge(rng, 96)
    assert SO.soft_nms_c(d, *params)[0][:, 4].tolist() == sorted(d[:, 4].tolist(), reverse=True)
    d, params = R.inf_hard(rng, 96)
    assert np.isnan(SO.soft_nms_c(d, *params)[0][:, 4]).any()


@pytest.mark.parametrize("edge", R.NONFINITE)
def test_oracle_equals_model_on_nonfinite_scores(edge):
    """NaN and +Inf inputs, and NaN made mid-run: the scan rule makes the oracle and the model agree."""
    for seed in range(40):
        rng = np.random.default_rng(seed)
        d, params = R.EDGES[edge](rng, int(rng.integers(2, 200)))
        for method in ("linear", "gaussian", "hard"):
            p = (method,) + params[1:]
            assert same(SO.soft_nms_c(d, *p), SM.soft_nms_model(d, *p)), (edge, seed, method)


def gaussian_clusters(rng, n):
    return R.clustered_int(rng, n), ("gaussian", 0.5, 0.3, 0.001)


MUTANTS = [(SO.GE_NT, "iou_at_nt"), (SO.NO_PLUS_ONE, "iou_at_nt"), (SO.PRUNE_UNTOUCHED, "no_overlap"), (SO.TIES_HIGH, "all_tied"),
           (SO.STABLE_COMPACT, "hole_table"), (SO.GAUSS_NO_SQUARE, "gaussian")]


@pytest.mark.parametrize("variant,edge", MUTANTS, ids=["ge_nt", "no_plus_one", "prune_untouched", "ties_high", "stable_compaction",
                                                       "gaussian_unsquared"])
def test_each_oracle_mistake_fails_the_comparator(variant, edge):
    rng = np.random.default_rng(variant)
    if edge == "gaussian":
        boxes, params = gaussian_clusters(rng, 96)
        d = R._rows(boxes, R.quantised_scores(rng, 96))
    else:
        d, params = R.EDGES[edge](rng, 96)
    ref = R.soft_nms64(d, *params)
    R.check_soft64(*SO.soft_nms_c(d, *params), d, ref, "definition")
    with pytest.raises(AssertionError):
        R.check_soft64(*SO.soft_nms_c(d, *params, variant=variant), d, ref, "mutant")


def test_features_ref_hand_case():
    keep = np.full((2, 4, 5), -1, np.int32)
    cnt = np.zeros((2, 4), np.int32)
    keep[0, 1, :2], cnt[0, 1] = [3, 1], 2
    keep[0, 3, :1], cnt[0, 3] = [4], 1
    keep[0, 0, :1], cnt[0, 0] = [0], 1                # class 0 never emits
    keep[1, 2, :3], cnt[1, 2] = [2, 0, 1], 3
    fc7 = np.arange(10 * 4, dtype=F).reshape(10, 4)
    feat, roi = R.features_ref(keep, cnt, fc7, 2)
    assert roi.tolist() == [[3, 1], [2, 0]]
    assert np.array_equal(feat[0], fc7[[3, 1]]) and np.array_equal(feat[1], fc7[[7, 5]])
    feat, roi = R.features_ref(keep, cnt, fc7, 4)
    assert roi.tolist() == [[3, 1, 4, -1], [2, 0, 1, -1]] and not feat[:, 3].any()


@pytest.mark.parametrize("C", [2, 1024])
def test_features_model_and_off_by_one_mutant(C):
    """On the device test's cases the kernel's slot lookup equals the gather reference at every max_det, and reading one entry
    past the last count (slot <= total) does not: the cases have totals strictly inside (0, max_det)."""
    rng = np.random.default_rng(C)
    keep, cnt = R.features_case(rng, C)
    fc7 = rng.standard_normal((keep.shape[0] * keep.shape[2], 4)).astype(F)
    totals = cnt[:, 1:].sum(1)
    assert (totals == 5).any() and (totals == 12).any()
    caught = 0
    for max_det in (1, 7, 8, 9, 100):
        wf, wr = R.features_ref(keep, cnt, fc7, max_det)
        mf, mr = R.features_model(keep, cnt, fc7, max_det)
        assert np.array_equal(mr, wr) and np.array_equal(mf, wf), max_det
        assert ((wr == -1).sum(1) == np.maximum(max_det - totals, 0)).all()
        caught += not np.array_equal(R.features_model(keep, cnt, fc7, max_det, inclusive=True)[1], wr)
    assert caught >= 4                                # every max_det above 1 has an image whose count ends before it
