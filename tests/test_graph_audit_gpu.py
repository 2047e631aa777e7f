"""Every step of the detection graph at production shapes, each against float64 (or its exact model) on its own device inputs.

Per config: a first `detect` call on other images builds the plan (eager warm-up, graph capture, one replay); then every tape
buffer and record buffer except the post step's scratch workspace is filled with 0xff bytes (NaN as fp32, -1 as int32) and a
second call on the audited images is a pure replay of the cached graph.  The tape's step labels must match `net_ref64.walk`
one for one (so no step goes unaudited), and every step is audited (`net_ref64.audit`, fed the device outputs of the steps the
oracle says feed it).  Then the same steps run eagerly, one at a time with a synchronise between them, each step's declared
outputs poisoned the same way before it runs: each step's outputs equal the replay's bit for bit, and no step changes a tape
buffer it does not declare as its output.

What the ordering check covers: a step missing from the graph, or one that in this replay read a buffer before its producer
wrote it (a missing or misplaced PDL wait or stream dependency), reads poison or the wrong images' values instead of the
warm-up's, and fails its audit or the eager comparison.  It cannot prove a race absent: a premature read that happens to land
after the producer's store in this replay passes.

Observed on an H100 80 GB HBM3 (700 W limit), worst err / bound over all steps: ResNet-101 0.40 (batch 4: 0.40, align mode: 0.40),
VGG16 0.35, MobileNet-v1 0.77 (a head depthwise conv), ResNet-152 at 1000 RoIs 0.38, ResNet-50 TF32X3 0.34, F16X1 0.34 (against
its operand model); the module runs in about 4 minutes."""

import numpy as np
import pytest
import torch

import conv_split_model as M
import net_ref64 as R
from graph_audit import build, run_audit

pytestmark = pytest.mark.gpu
F = np.float32

# (id, net, classes, anchor scales, blob H x W, batch, cfg updates, FRCNN_CONV_IMPL)
CONFIGS = [
    ("res101", "res101", 81, (4, 8, 16, 32), (600, 800), 1, {}, None),
    ("vgg16", "vgg16", 21, (8, 16, 32), (600, 800), 1, {}, None),
    ("mobile", "mobile", 81, (4, 8, 16, 32), (600, 800), 1, {}, None),
    ("res152_1000", "res152", 81, (2, 4, 8, 16, 32), (800, 1067), 1, {"TEST.RPN_POST_NMS_TOP_N": 1000}, None),
    ("res101_b4", "res101", 81, (4, 8, 16, 32), (600, 800), 4, {}, None),
    ("res101_align", "res101", 81, (4, 8, 16, 32), (600, 800), 1, {"POOLING_MODE": "align"}, None),
    ("res50_tf32", "res50", 21, (8, 16, 32), (600, 800), 1, {}, "tf32"),
    ("res50_f16x1", "res50", 21, (8, 16, 32), (600, 800), 1, {}, "f16x1"),
]
@pytest.mark.parametrize("cid,net_name,C,scales,hw,B,cfg_updates,impl", CONFIGS, ids=[c[0] for c in CONFIGS])
def test_graph_audit(cuda, monkeypatch, cid, net_name, C, scales, hw, B, cfg_updates, impl):
    net, w, rec = build(monkeypatch, net_name, C, scales, cfg_updates, impl)
    mode = M.MODES[{"tf32": "tf32x3", "f16x1": "f16x1"}.get(impl, "f16x3")]
    rows = run_audit(net_name, C, scales, hw, B, net, w, rec, mode, cid)
    assert max(r.ratio for r in rows) <= 1


TEETH_LAYER = "resnet_v1_50/block2/unit_2/bottleneck_v1/conv2"


def test_audit_names_a_corrupted_buffer(cuda, monkeypatch):
    """One element of one intermediate buffer moved by 1e-3 relative after the replay: the audit fails at that layer.  The
    element lies on the map's top border, which the audit samples whole (an element it does not sample fails the next layer)."""
    net, w, rec = build(monkeypatch, "res50", 21, (8, 16, 32), {}, None)

    def corrupt(walk, steps):
        i = [l.key for l in walk].index(TEETH_LAYER)
        row = steps[i][1]["out"][0, 0]                       # [w, c]: image 0's first row
        j = int(torch.argmax(row.abs()))
        row.view(-1)[j] *= 1 + 1e-3
    with pytest.raises(R.Finding) as e:
        run_audit("res50", 21, (8, 16, 32), (304, 400), 1, net, w, rec, M.F16X3, "corrupted", corrupt)
    assert str(e.value).startswith("conv:" + TEETH_LAYER + ":"), str(e.value)


def test_audit_names_a_shifted_variance(cuda, monkeypatch):
    """The engine's weights move one layer's moving_variance by 1e-3 - 1e-5 (what an eps mix-up does), the reference keeps
    the true tensors: the audit fails at that layer."""
    key = TEETH_LAYER + "/BatchNorm/moving_variance"

    def shifted(w):
        w2 = dict(w)
        w2[key] = (w[key] + F(1e-3 - 1e-5)).astype(F)
        return w2
    net, w, rec = build(monkeypatch, "res50", 21, (8, 16, 32), {}, None, weights=shifted)
    with pytest.raises(R.Finding) as e:
        run_audit("res50", 21, (8, 16, 32), (304, 400), 1, net, w, rec, M.F16X3, "variance")
    assert str(e.value).startswith("conv:" + TEETH_LAYER + ":"), str(e.value)
