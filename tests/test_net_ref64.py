"""The per-layer comparator of `net_ref64.py` has teeth (CPU only).

A stand-in for the device -- every tensor-core conv is `conv_split_model.model` with an fp32 epilogue, the SIMT convs the
float64 conv with an fp32 epilogue, max pool its model -- runs the ResNet-50 backbone and RPN convolutions of `synth.make`
weights on a small blob.  Its outputs pass the audit in the three arithmetic modes; each wiring fault below fails it, and
the failure names the faulty layer."""
import numpy as np
import pytest

import conv_split_model as M
import net_ref64 as R
from tf_faster_rcnn_b200 import synth

SC = "resnet_v1_50"
B1 = SC + "/block1/unit_%d/bottleneck_v1"
HW = (64, 96)
TILE = (4, 8)


@pytest.fixture(scope="module")
def net():
    w = synth.make("res50", 21, 9)
    layers = R.walk("res50", 9, 21, head=False)
    layers = [l for l in layers if l.kind in ("conv", "conv_first", "max_pool")]
    return w, layers, synth.synthetic_blob(*HW)


def run(net, mode=M.F16X3, mutant=None):
    w, layers, blob = net
    bufs = R.standin(layers, w, blob, mode, mutant, TILE)
    plans = {l.key: dict(tile=TILE) for l in layers}
    return R.audit(layers, w, bufs, mode, plans, n_random=64)


def test_walk_restates_the_oracle():
    layers = R.walk("res101", 12, 81)
    labels = [l.label for l in layers]
    assert labels[:2] == ["conv_first:resnet_v1_101/conv1", "max_pool"]
    convs = [l for l in layers if l.kind == "conv" and "/bottleneck_v1/" in l.key]
    assert len(convs) == 3 * (3 + 4 + 23 + 3)
    proj = [l.key for l in layers if l.kind == "conv" and len(l.p["parts"]) == 2]
    assert proj == ["resnet_v1_101/block%d/unit_1/bottleneck_v1/conv3" % b for b in (1, 2, 3, 4)]
    assert sum(1 for l in layers if l.key.endswith("/shortcut_pool")) == 2
    assert [l.key for l in layers if l.p.get("mean")] == ["resnet_v1_101/block4/unit_3/bottleneck_v1/conv3"]
    assert labels[-4:] == ["conv:resnet_v1_101/cls_bbox", "cls_finish", "bbox_decode", "detect_post"]
    assert labels.index("crop_pool") == labels.index("proposals") + 1
    mob = R.walk("mobile", 12, 81)
    assert {l.p["eps"] for l in mob if l.kind in ("conv_first", "depthwise") or "pointwise" in l.key} == {1e-3}
    assert sum(1 for l in mob if l.kind == "depthwise") == 13 and mob[-5].label == "spatial_mean"
    vgg = R.walk("vgg16", 9, 21, pooling="align")
    assert [l.label for l in vgg].count("max_pool") == 4 and "roi_align" in [l.label for l in vgg]
    assert vgg[-6].p["fc"] and vgg[-6].key == "vgg_16/fc6"


@pytest.mark.parametrize("mode", ["f16x3", "tf32x3", "f16x1"])
def test_standin_passes(net, mode):
    rows = run(net, M.MODES[mode])
    assert len(rows) == len(net[1])
    worst = max(rows, key=lambda r: r.ratio)
    print("\n[%s] worst err/bound %.3f at %s %s" % (mode, worst.ratio, worst.label, worst.at))
    assert worst.ratio <= 1


MUTANTS = [
    ("eps", B1 % 2 + "/conv2"),                    # BatchNorm eps 1e-3 instead of 1e-5
    ("residual", SC + "/block2/unit_3/bottleneck_v1/conv3"),  # the residual of unit 1 instead of unit 2
    ("swap", B1 % 1 + "/conv3"),                   # the projection unit's two A sources swapped
    ("pad", B1 % 2 + "/conv2"),                    # SAME padding shifted by one
    ("kblock", SC + "/block2/unit_2/bottleneck_v1/conv1"),   # one input channel's contribution lost
    ("shift", SC + "/block3/unit_4/bottleneck_v1/conv3"),    # the shift missing on one output channel
    ("cols+4", SC + "/rpn_heads"),                 # the RPN bbox columns written at dcol + 4
    ("cols-4", SC + "/rpn_heads"),                 # ... at dcol - 4, over the cls columns' zero pad
    ("seam", B1 % 2 + "/conv3"),                   # one output 1 % off at a tile seam
]


@pytest.mark.parametrize("mutant", MUTANTS, ids=[m[0] for m in MUTANTS])
def test_mutant_fails_naming_its_layer(net, mutant):
    with pytest.raises(R.Finding) as e:
        run(net, M.F16X3, mutant)
    assert str(e.value).startswith("conv:" + mutant[1] + ":"), str(e.value)
