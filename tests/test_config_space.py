"""The architecture and pooling options of test_config_audit_gpu.py without a GPU: the refusals of create_architecture (before
any device work), the zero-padded depths of a depth-multiplied MobileNet, VGG16's fc6 at every POOLING_SIZE, the launch list
`net_ref64.walk` gives for each option, and the work decomposition (frcnn_conv_plan_geometry, 132 SMs) of the layers each GPU
config exists for."""
import numpy as np
import pytest

import net_ref64 as R
from test_config_audit_gpu import CONFIGS
from test_plan_geometry import geom
from tf_faster_rcnn_b200 import _native as N
from tf_faster_rcnn_b200 import synth

F = np.float32


@pytest.fixture
def no_device(monkeypatch):
    """Any call into the C library fails the test: a refusal must come before device work."""
    def lib():
        raise AssertionError("device work before the refusal")
    monkeypatch.setattr(N, "lib", lib)


@pytest.fixture
def cfg():
    """The cfg, restored afterwards, and the network registry too: a network whose create_architecture was refused must not
    stay where the tensorflow shim's Saver.restore looks for networks."""
    from model.config import cfg as c
    from nets import network
    saved = (c.POOLING_MODE, c.POOLING_SIZE, c.MOBILENET.DEPTH_MULTIPLIER, c.RPN_CHANNELS)
    registry = list(network._REGISTRY)
    yield c
    c.POOLING_MODE, c.POOLING_SIZE, c.MOBILENET.DEPTH_MULTIPLIER, c.RPN_CHANNELS = saved
    network._REGISTRY[:] = registry


def make_net(net_name):
    from nets.vgg16 import vgg16
    from nets.resnet_v1 import resnetv1
    from nets.mobilenet_v1 import mobilenetv1
    return vgg16() if net_name == "vgg16" else mobilenetv1() if net_name == "mobile" else resnetv1(num_layers=int(net_name[3:]))


# ---- refusals ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mult", [0.3, 0.1, 2.25, 3.0, 0.0, -0.5, float("nan"), float("inf"), True, "0.5"])
def test_unsupported_depth_multiplier_is_refused(cfg, no_device, mult):
    """0.3: Conv2d_0 depth 9; 0.1: depth 25 (6.4 -> min_depth 8, then 12, 25); 2.25 / 3.0: Conv2d_0 depth 72 / 96 past what
    conv_first takes; the rest are not positive finite numbers."""
    cfg.MOBILENET.DEPTH_MULTIPLIER = mult
    net = make_net("mobile")
    with pytest.raises(ValueError, match="DEPTH_MULTIPLIER"):
        net.create_architecture("TEST", 21, tag="default")


@pytest.mark.parametrize("mode,size", [("crop", 1), ("crop", 17), ("crop", 0), ("crop", 7.0), ("crop", "7")])
def test_unsupported_crop_pooling_size_is_refused(cfg, no_device, mode, size):
    cfg.POOLING_MODE, cfg.POOLING_SIZE = mode, size
    for net_name in ("res101", "vgg16", "mobile"):
        with pytest.raises(ValueError, match="POOLING_SIZE"):
            make_net(net_name).create_architecture("TEST", 21, tag="default")


@pytest.mark.parametrize("channels", [100, 0, -32, 256.0, "512"])
def test_unsupported_rpn_channels_are_refused(cfg, no_device, channels):
    cfg.RPN_CHANNELS = channels
    with pytest.raises(ValueError, match="RPN_CHANNELS"):
        make_net("res50").create_architecture("TEST", 21, tag="default")


@pytest.mark.parametrize("mode,size", [("crop", 2), ("crop", 16), ("align", 1), ("pool", 16)])
def test_supported_pooling_sizes_are_accepted(cfg, no_device, mode, size):
    cfg.POOLING_MODE, cfg.POOLING_SIZE = mode, size
    make_net("res101").create_architecture("TEST", 21, tag="default")


# ---- depth multipliers ---------------------------------------------------------------------------------------------------------
MULTS = [0.25, 0.5, 0.75, 1.0, 1.25, 1.5, 1.75, 2.0, 0.375, 0.625]


@pytest.mark.parametrize("mult", MULTS)
def test_depth_multiplier_runs_padded_layers(cfg, mult):
    """Every accepted multiplier: the padded checkpoint matches the network layer by layer, Conv2d_0's padded depth is one
    conv_first takes, every pointwise layer's plan geometry accepts its padded K, the pad is zeros (variance 1) and the real
    channels are the checkpoint's."""
    from nets.mobilenet_v1 import FIRST_COUTS, check_depth_multiplier, pad_depths, padded_depth
    d = check_depth_multiplier(mult)
    w = synth.make("mobile", 21, 9, depth_multiplier=mult)
    wp = pad_depths(w)
    sc = "MobilenetV1/Conv2d_%d"
    assert wp[sc % 0 + "/weights"].shape == (3, 3, 3, padded_depth(d[0])) and padded_depth(d[0]) in FIRST_COUTS
    cin = padded_depth(d[0])
    for i in range(1, 14):
        pw = wp[sc % i + "_pointwise/weights"]
        assert pw.shape == (1, 1, cin, padded_depth(d[i])) and wp[sc % i + "_depthwise/depthwise_weights"].shape[2] == cin
        geom(1, 19, 25, cin, pw.shape[3], 1)                          # raises when the conv kernel refuses the layer
        real = w[sc % i + "_pointwise/weights"]
        assert np.array_equal(pw[:, :, :real.shape[2], :real.shape[3]], real)
        assert not pw[:, :, real.shape[2]:].any() and not pw[..., real.shape[3]:].any()
        bn = sc % i + "_pointwise/BatchNorm/"
        assert not wp[bn + "gamma"][d[i]:].any() and (wp[bn + "moving_variance"][d[i]:] == 1).all()
        cin = pw.shape[3]
    assert cin == d[13] == synth.mobilenet_depth(1024, mult)           # the head's feature width is not padded
    if all(v % 32 == 0 for v in d):
        assert wp is w


def test_padding_leaves_the_real_channels_unchanged():
    """The oracle's MobileNet body on the padded checkpoint equals the unpadded one on the real channels (float32, 64 x 96)."""
    from nets.mobilenet_v1 import pad_depths
    from oracle import nets as ON
    w = synth.make("mobile", 21, 9, depth_multiplier=0.25)
    blob = synth.synthetic_blob(64, 96)
    a = ON.image_to_head("mobile", w, blob)
    b = ON.image_to_head("mobile", pad_depths(w), blob)
    assert a.shape == b.shape
    np.testing.assert_allclose(b, a, rtol=1e-5, atol=1e-6)


# ---- synth: VGG16 fc6 at every POOLING_SIZE -----------------------------------------------------------------------------------
@pytest.mark.parametrize("P,rows", [(1, 512), (7, 25088), (14, 100352)])
def test_vgg_fc6_rows_follow_the_pooling_size(P, rows):
    assert synth.spec("vgg16", 21, 9, pooling_size=P)["vgg_16/fc6/weights"] == (rows, 4096)


def test_vgg_fc6_draw_follows_the_pooling_size():
    assert synth.make("vgg16", 21, 9, pooling_size=1)["vgg_16/fc6/weights"].shape == (512, 4096)


def shaped(spec):
    """Zero-stride stand-ins with the shapes of `spec` (check_variables reads only shapes)."""
    return {k: np.broadcast_to(F(0), s) for k, s in spec.items()}


def test_check_variables_reads_the_pooling_size(cfg):
    cfg.POOLING_MODE, cfg.POOLING_SIZE = "align", 14
    net = make_net("vgg16")
    net.create_architecture("TEST", 21, tag="default")
    assert net.check_variables(shaped(synth.spec("vgg16", 21, 9, pooling_size=14))) == []
    msgs = net.check_variables(shaped(synth.spec("vgg16", 21, 9)))
    assert len(msgs) == 1 and "vgg_16/fc6/weights" in msgs[0], msgs


# ---- the walk --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("A,dcol,ld", [(1, 4, 8), (9, 20, 56), (25, 52, 152)])
def test_walk_anchor_layout(A, dcol, ld):
    L = {l.key: l for l in R.walk("res101", A, 81)}
    assert L["resnet_v1_101/rpn_heads"].p["cout"] == ld
    assert L["rpn_decode"].p == dict(A=A, dcol=dcol)
    assert L["resnet_v1_101/rpn_heads"].p["fused"] == [("resnet_v1_101/rpn_cls_score", 0, 2 * A),
                                                      ("resnet_v1_101/rpn_bbox_pred", dcol, 4 * A)]


def test_walk_pooling_options():
    base = [l.label for l in R.walk("res101", 12, 81)]
    for pooling, label in (("crop", "crop_pool"), ("align", "roi_align"), ("pool", "roi_pool")):
        for mp in (False, True):
            L = R.walk("res101", 12, 81, pooling, mp)
            assert [l.label for l in L] == [label if x == "crop_pool" else x for x in base]
            assert [l for l in L if l.key == "pool5"][0].p == dict(mode=pooling, pre_pool=mp)
    assert [l for l in R.walk("vgg16", 9, 21) if l.key == "pool5"][0].p["pre_pool"]
    assert [l.label for l in R.walk("mobile", 9, 21)] == [l.label for l in R.walk("mobile", 25, 21)]


# ---- the paths the GPU configs claim ---------------------------------------------------------------------------------------------
def rows(g):
    return g["tile_n"] * g["tile_h"] * g["tile_w"]


# config id -> the layer the path is on (n, h, w, cin, cout, k), what the decomposition must show
GEOMETRY = {
    "mobile_dm025": ((1, 300, 400, 32, 32, 1), lambda g: g["k_blocks"] == 1),                    # Conv2d_1_pointwise, K 32
    "mobile_dm075": ((1, 76, 100, 64, 96, 1), lambda g: g["k_blocks"] == 1 and g["n_tiles"] == 1),
    "mobile_dm125": ((1, 152, 200, 64, 96, 1), lambda g: g["k_blocks"] == 1),
    "res50_rpn256": ((1, 19, 25, 256, 72, 1), lambda g: g["k_blocks"] == 4),          # rpn_heads (A = 12), K = 256
    "vgg16_rpn128": ((1, 19, 25, 128, 56, 1), lambda g: g["k_blocks"] == 2),
    "res101_a1": ((1, 19, 25, 1024, 8, 1), lambda g: g["block_n"] == 64 and g["n_tiles"] == 1),
    "res101_a25": ((1, 38, 50, 1024, 152, 1), lambda g: g["block_n"] == 128 and g["n_tiles"] == 2),
    "res101_crop14": ((300, 14, 14, 1024, 512, 1), lambda g: rows(g) == 128 and g["m_tiles"] == 460),     # 196 rows per RoI
    "res101_crop2": ((300, 2, 2, 512, 512, 3), lambda g: g["tile_n"] == 30 and (g["tile_h"], g["tile_w"]) == (2, 2)),
    "res101_align1": ((300, 1, 1, 512, 512, 3), lambda g: g["tile_n"] == 100 and g["splits"] > 1),
    "res101_pool16": ((300, 16, 16, 1024, 512, 1), lambda g: rows(g) == 128 and g["m_tiles"] == 600),    # two tiles per RoI
    "vgg16_align14": ((1, 1, 300, 100352, 4096, 1), lambda g: g["k_blocks"] == 1568 and g["splits"] == 1),
    "vgg16_crop4": ((1, 1, 300, 8192, 4096, 1), lambda g: g["k_blocks"] == 128),
}


def test_every_gpu_config_is_listed_once():
    ids = [c[0] for c in CONFIGS]
    assert len(ids) == len(set(ids)) == 16
    assert set(GEOMETRY) <= set(ids)


@pytest.mark.parametrize("cid", sorted(GEOMETRY))
def test_gpu_config_covers_its_path(cid):
    shape, covers = GEOMETRY[cid]
    g = geom(*shape)
    assert covers(g), "%s no longer covers its path: %s" % (cid, g)


def test_crop14_mean_groups_span_tiles():
    """The ResNet head's last conv3 at P = 14 reduces 196 rows per RoI in its epilogue, over 128-row tiles."""
    g = geom(300, 14, 14, 512, 2048, 1)
    assert rows(g) == 128 and 196 % rows(g) != 0
