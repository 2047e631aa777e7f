"""POOLING_MODE 'align' / 'pool' without a GPU: the numpy models (tests/roi_pool_oracle.py) against torchvision's CPU ops bit
for bit, the align model against its float64 bound, the plausible mistakes each comparator catches, the configuration keys and
their refusals, the caller-box bound, and the ptxas report of the two kernels."""
import os
import re
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import roi_pool_oracle as RP  # noqa: E402

F = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
torch = pytest.importorskip("torch")
tvops = pytest.importorskip("torchvision.ops")


def tv_align(feat, rois, pooled, sr, aligned):
    x = torch.from_numpy(np.ascontiguousarray(feat.transpose(0, 3, 1, 2)))
    y = tvops.roi_align(x, torch.from_numpy(rois), pooled, spatial_scale=1.0 / 16, sampling_ratio=sr, aligned=aligned)
    return y.numpy().transpose(0, 2, 3, 1)


def tv_pool(feat, rois, pooled):
    x = torch.from_numpy(np.ascontiguousarray(feat.transpose(0, 3, 1, 2)))
    return tvops.roi_pool(x, torch.from_numpy(rois), pooled, spatial_scale=1.0 / 16).numpy().transpose(0, 2, 3, 1)


def rand_feat(rng, b, h, w, c):
    return rng.standard_normal((b, h, w, c)).astype(F)


MAPS = [(1, 1), (2, 3), (38, 50)]


@pytest.mark.parametrize("hw", MAPS, ids=["1x1", "2x3", "38x50"])
@pytest.mark.parametrize("pooled", [1, 2, 7, 14, 16])
def test_align_model_equals_torchvision(hw, pooled):
    rng = np.random.default_rng(hw[0] * 100 + pooled)
    feat = rand_feat(rng, 1, hw[0], hw[1], 8 if hw[0] > 30 else 12)
    rois = RP.edge_rois(*hw, rng, n_random=30 if hw[0] > 30 else 60)
    for sr in (0, 1, 2, 4):
        for aligned in (False, True):
            got = RP.roi_align_model(feat, rois, pooled, sr, aligned)
            want = tv_align(feat, rois, pooled, sr, aligned)
            assert got.tobytes() == want.tobytes(), (sr, aligned)


@pytest.mark.parametrize("hw", MAPS, ids=["1x1", "2x3", "38x50"])
@pytest.mark.parametrize("pooled", [1, 2, 7, 14, 16])
def test_pool_model_equals_torchvision(hw, pooled):
    rng = np.random.default_rng(7 + hw[1] * 100 + pooled)
    feat = rand_feat(rng, 1, hw[0], hw[1], 8)
    rois = RP.edge_rois(*hw, rng)
    assert RP.roi_pool_model(feat, rois, pooled).tobytes() == tv_pool(feat, rois, pooled).tobytes()


def test_pool_model_half_corners_equal_torchvision():
    rng = np.random.default_rng(3)
    feat = rand_feat(rng, 1, 9, 13, 8)
    rois = RP.half_rois(rng, 9, 13)
    for pooled in (1, 2, 7):
        assert RP.roi_pool_model(feat, rois, pooled).tobytes() == tv_pool(feat, rois, pooled).tobytes(), pooled


def test_batch_index_is_clamped():
    rng = np.random.default_rng(11)
    feat = rand_feat(rng, 3, 9, 13, 8)
    rois = RP.edge_rois(9, 13, rng, 20)
    for idx, img in ((-1, 0), (5, 2), (1, 1)):
        r = rois.copy(); r[:, 0] = idx
        r0 = rois.copy(); r0[:, 0] = img
        assert RP.roi_align_model(feat, r, 7, 2, False).tobytes() == tv_align(feat, r0, 7, 2, False).tobytes()
        assert RP.roi_pool_model(feat, r, 7).tobytes() == tv_pool(feat, r0, 7).tobytes()


@pytest.mark.parametrize("sr,aligned", [(0, False), (0, True), (2, False), (4, True)])
def test_align_model_within_float64_bound(sr, aligned):
    rng = np.random.default_rng(20 + sr)
    feat = rand_feat(rng, 1, 38, 50, 8) * F(100)
    rois = RP.edge_rois(38, 50, rng, 40)
    got = RP.roi_align_model(feat, rois, 7, sr, aligned)
    exact, bound = RP.roi_align_ref64(feat, rois, 7, sr, aligned)
    err = np.abs(got.astype(np.float64) - exact)
    assert (err <= bound).all(), float((err - bound).max())
    assert float(bound.max()) < 1e-4 * float(np.abs(feat).max())        # the bound says something
    assert err.max() > 0                                                  # and the fp32 path does round


def nan_cell_feat(rng):
    feat = rand_feat(rng, 1, 9, 13, 8)
    feat[0, 0, 0, :4] = [np.nan, np.inf, -np.inf, np.nan]
    return feat


def test_nan_rule_out_of_range_sample_is_not_read():
    """torchvision adds 0 * feat[b, 0, 0] for a sample outside [-1, dim]; the kernel (and the model) does not read it.  With
    that cell non-finite the two differ exactly in the bins that have such a sample and do not sample the cell otherwise: there
    torchvision gives NaN and the model a finite mean.  Everywhere else they are equal bit for bit."""
    rng = np.random.default_rng(5)
    feat = nan_cell_feat(rng)
    rois = np.array([[0, 60, 40, 150, 120],            # inside: no out-of-range sample, cell (0,0) not sampled
                     [0, -100, 40, 60, 120],            # partly left of the map: out-of-range samples
                     [0, 40, -90, 150, 60]], F)         # partly above
    got = RP.roi_align_model(feat, rois, 7, 2, False)
    want = tv_align(feat, rois, 7, 2, False)
    same = (got == want) | (np.isnan(got) & np.isnan(want))
    differ = ~same
    assert not differ[0].any()
    assert differ[1:].any()
    assert np.isnan(want[differ]).all() and np.isfinite(got[differ]).all()
    assert (differ[..., 4:] == False).all()             # noqa: E712  finite channels of the cell: no difference


def test_nan_rule_pool_max_skips_nan():
    """RoIPool's '>' from -FLT_MAX: a NaN never wins, an all-NaN bin gives -FLT_MAX (torchvision's own result)."""
    feat = np.zeros((1, 4, 4, 4), F)
    feat[..., 0] = np.nan
    feat[0, 1, 1, 1] = np.nan; feat[0, 2, 2, 1] = -3
    rois = np.array([[0, 0, 0, 63, 63]], F)
    got = RP.roi_pool_model(feat, rois, 2)
    assert got.tobytes() == tv_pool(feat, rois, 2).tobytes()
    assert (got[..., 0] == -np.finfo(F).max).all() and not np.isnan(got).any()


@pytest.mark.parametrize("bug,kw", [
    ("no_offset", dict(aligned=True)),
    ("no_min_size", dict(aligned=False)),
    ("no_min_count", dict(aligned=True)),
    ("le_minus_one", dict(aligned=False)),
    ("no_top_clamp", dict(aligned=False)),
])
def test_align_comparator_catches_mistake(bug, kw):
    rng = np.random.default_rng(9)
    feat = rand_feat(rng, 1, 9, 13, 8)
    rois = RP.edge_rois(9, 13, rng, 40)
    for sr in (0, 1, 2):
        want = tv_align(feat, rois, 7 if sr else 2, sr, kw["aligned"])
        good = RP.roi_align_model(feat, rois, 7 if sr else 2, sr, kw["aligned"])
        assert good.tobytes() == want.tobytes()
    caught = []
    for sr in (0, 1, 2):
        p = 7 if sr else 2
        with np.errstate(invalid="ignore", divide="ignore"):
            bad = RP.roi_align_model(feat, rois, p, sr, kw["aligned"], _bug=bug)
        caught.append(bad.tobytes() != tv_align(feat, rois, p, sr, kw["aligned"]).tobytes())
    assert any(caught), bug


def test_pool_comparator_catches_half_even():
    rng = np.random.default_rng(4)
    feat = rand_feat(rng, 1, 9, 13, 8)
    rois = RP.half_rois(rng, 9, 13)
    assert RP.roi_pool_model(feat, rois, 7, _bug="half_even").tobytes() != tv_pool(feat, rois, 7).tobytes()


# ---- configuration --------------------------------------------------------------------------------------------------------
@pytest.fixture
def pool_cfg():
    from model.config import cfg
    saved = (cfg.POOLING_MODE, cfg.POOLING_SIZE, dict(cfg.ROI_ALIGN))
    yield cfg
    cfg.POOLING_MODE, cfg.POOLING_SIZE = saved[:2]
    cfg.ROI_ALIGN.update(saved[2])


def make_net():
    from nets.resnet_v1 import resnetv1
    return resnetv1(num_layers=50)


def test_config_defaults(pool_cfg):
    assert pool_cfg.POOLING_MODE == "crop" and pool_cfg.POOLING_SIZE == 7
    assert pool_cfg.ROI_ALIGN == {"SAMPLING_RATIO": 0, "ALIGNED": False}
    net = make_net()
    net.create_architecture("TEST", 21, tag="default")
    assert net.options["pooling_mode"] == "crop" and net.options["roi_align"] is None


def test_config_yaml_and_set_reach_the_options(pool_cfg, tmp_path):
    from model.config import cfg_from_file, cfg_from_list
    p = tmp_path / "align.yml"
    p.write_text("POOLING_MODE: align\nROI_ALIGN:\n  SAMPLING_RATIO: 2\n  ALIGNED: true\n")
    cfg_from_file(str(p))
    net = make_net()
    net.create_architecture("TEST", 21, tag="default")
    assert net.options["pooling_mode"] == "align" and net.options["roi_align"] == (2, True)
    cfg_from_list(["POOLING_MODE", "pool", "POOLING_SIZE", "14", "ROI_ALIGN.SAMPLING_RATIO", "0", "ROI_ALIGN.ALIGNED", "False"])
    assert pool_cfg.ROI_ALIGN == {"SAMPLING_RATIO": 0, "ALIGNED": False}
    net.create_architecture("TEST", 21, tag="default")
    assert net.options["pooling_mode"] == "pool" and net.options["pooling_size"] == 14 and net.options["roi_align"] is None
    cfg_from_list(["POOLING_MODE", "align", "ROI_ALIGN.SAMPLING_RATIO", "16"])
    net.create_architecture("TEST", 21, tag="default")
    assert net.options["roi_align"] == (16, False)
    with pytest.raises(AssertionError):
        cfg_from_list(["ROI_ALIGN.ALIGNED", "1"])          # the strict merge keeps the bool type


@pytest.mark.parametrize("update,exc", [
    (dict(POOLING_MODE="max"), NotImplementedError),
    (dict(POOLING_MODE="ALIGN"), NotImplementedError),
    (dict(POOLING_MODE="align", SAMPLING_RATIO=-1), ValueError),
    (dict(POOLING_MODE="align", SAMPLING_RATIO=17), ValueError),
    (dict(POOLING_MODE="align", SAMPLING_RATIO=2.0), ValueError),
    (dict(POOLING_MODE="align", SAMPLING_RATIO=True), ValueError),
    (dict(POOLING_MODE="align", ALIGNED=1), ValueError),
    (dict(POOLING_MODE="align", ALIGNED="yes"), ValueError),
    (dict(POOLING_MODE="align", POOLING_SIZE=0), ValueError),
    (dict(POOLING_MODE="pool", POOLING_SIZE=17), ValueError),
    (dict(POOLING_MODE="pool", POOLING_SIZE=7.0), ValueError),
])
def test_invalid_values_raise_before_device_work(pool_cfg, monkeypatch, update, exc):
    from tf_faster_rcnn_b200 import _native
    monkeypatch.setattr(_native, "lib", lambda: pytest.fail("device work before the refusal"))
    pool_cfg.POOLING_MODE = update.get("POOLING_MODE", "crop")
    if "POOLING_SIZE" in update:
        pool_cfg.POOLING_SIZE = update["POOLING_SIZE"]
    for k in ("SAMPLING_RATIO", "ALIGNED"):
        if k in update:
            pool_cfg.ROI_ALIGN[k] = update[k]
    with pytest.raises(exc):
        make_net().create_architecture("TEST", 21, tag="default")


def test_align_keys_are_not_read_outside_align_mode(pool_cfg):
    pool_cfg.ROI_ALIGN.SAMPLING_RATIO = -5
    for mode in ("crop", "pool"):
        pool_cfg.POOLING_MODE = mode
        net = make_net()
        net.create_architecture("TEST", 21, tag="default")
        assert net.options["roi_align"] is None


def test_caller_box_bound():
    from tf_faster_rcnn_b200 import engine
    ok = [np.array([[-600, -400, 1200, 800], [0, 0, 10, 10]], F)]          # within [-W, 2W] x [-H, 2H] of a 400x600 blob
    for mode in ("align", "pool", "crop"):
        engine.check_pool_boxes(mode, ok, [1.0], (400, 600))
    bad = [np.array([[-601, 0, 10, 10]], F), np.array([[0, 0, 1201, 10]], F), np.array([[0, -401, 10, 10]], F),
           np.array([[0, 0, 10, 801]], F), np.array([[0, 0, np.nan, 10]], F), np.array([[0, np.inf, 10, 10]], F)]
    for b in bad:
        for mode in ("align", "pool"):
            with pytest.raises(ValueError):
                engine.check_pool_boxes(mode, [b], [1.0], (400, 600))
        engine.check_pool_boxes("crop", [b], [1.0], (400, 600))              # crop mode accepts what it accepts today
    # the bound applies to the box scaled into the blob
    engine.check_pool_boxes("align", [np.array([[0, 0, 500, 350]], F)], [2.0], (400, 600))
    with pytest.raises(ValueError):
        engine.check_pool_boxes("align", [np.array([[0, 0, 700, 350]], F)], [2.0], (400, 600))


def test_score_boxes_refuses_before_device_work(pool_cfg, monkeypatch):
    """Network.score_boxes in align / pool mode refuses an out-of-bound or non-finite box before any device work."""
    from tf_faster_rcnn_b200 import engine
    for mode in ("align", "pool"):
        pool_cfg.POOLING_MODE = mode
        net = make_net()
        net.create_architecture("TEST", 21, tag="default")
        monkeypatch.setattr(net, "_batch_plan", lambda *a, **k: pytest.fail("device work before the refusal"))
        for b in (np.array([[0, 0, 5000, 10]], F), np.array([[0, np.nan, 10, 10]], F)):
            with pytest.raises(ValueError):
                net.score_boxes(np.zeros((1, 400, 600, 3), F), [1.0], [(400, 600)], [b])
    assert engine.POOLING_MODES == ("crop", "align", "pool")


@pytest.mark.parametrize("kernel", ["roi_align_kernel", "roi_pool_kernel"])
def test_new_kernels_do_not_spill(kernel):
    """ptxas -v output written by the build."""
    log = open(os.path.join(ROOT, "tf_faster_rcnn_b200", "csrc", "_obj", "simt_ops.o.log")).read()
    found = re.findall(r"Function properties for \S*%s\S*\s*\n([^\n]*)" % kernel, log)
    assert len(found) == 1, "ptxas reports for %s: %d" % (kernel, len(found))
    assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in found[0], found[0]


def test_abi_refuses_bad_arguments_without_a_device():
    import ctypes
    from tf_faster_rcnn_b200 import _native
    L = _native.lib()
    p = ctypes.c_void_p(64)
    good = dict(batch=1, fh=4, fw=4, c=8, r=3, pooled=7, scale=0.0625, sr=0)
    for bad in (dict(c=6), dict(c=0), dict(pooled=0), dict(pooled=17), dict(batch=0), dict(fh=0), dict(r=-1), dict(scale=0.0),
                dict(sr=-1), dict(sr=17)):
        a = dict(good, **bad)
        assert L.frcnn_roi_align(p, a["batch"], a["fh"], a["fw"], a["c"], p, a["r"], a["pooled"], a["scale"], a["sr"], 0, p, None) == -2, bad
        assert _native.last_error()
        if "sr" not in bad:
            assert L.frcnn_roi_pool(p, a["batch"], a["fh"], a["fw"], a["c"], p, a["r"], a["pooled"], a["scale"], p, None) == -2, bad
