"""The attribute head on the bottom-up regions, without a GPU: cfg.ATTRIBUTES and its refusals before any device work, the
checkpoint variables it adds, the float64 oracle's argmax rule and the mistakes its comparators catch, the C ABI's argument
refusals and the ptxas report of the two kernels."""
import os
import re
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import attr_oracle as AO  # noqa: E402
import stage_ref64 as S  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = np.float32
VG = (401, 256, 512)


@pytest.fixture(autouse=True)
def _unregister_networks():
    """Networks register themselves process-wide (the tensorflow shim's Saver.restore walks the registry), so the ones built here
    leave it when their test ends."""
    from nets import network
    before = list(network._REGISTRY)
    yield
    network._REGISTRY[:] = before


@pytest.fixture
def attr_cfg():
    from model.config import cfg
    saved = dict(cfg.ATTRIBUTES)
    yield cfg
    cfg.ATTRIBUTES.update(saved)


def make_net(name="res101"):
    from nets.mobilenet_v1 import mobilenetv1
    from nets.resnet_v1 import resnetv1
    from nets.vgg16 import vgg16
    return vgg16() if name == "vgg16" else mobilenetv1() if name == "mobile" else resnetv1(num_layers=int(name[3:]))


# ---- configuration ------------------------------------------------------------------------------------------------------------
def test_config_defaults_and_merges(attr_cfg, tmp_path):
    from model.config import cfg_from_file, cfg_from_list
    assert attr_cfg.ATTRIBUTES == {"NUM_CLASSES": 0, "EMBED_DIM": 256, "HIDDEN": 512}
    net = make_net()
    net.create_architecture("TEST", 81, tag="default")
    assert net.options["attributes"] is None
    y = tmp_path / "vg.yml"
    y.write_text("ATTRIBUTES:\n  NUM_CLASSES: 401\n")
    cfg_from_file(str(y))
    net.create_architecture("TEST", 1601, tag="default")
    assert net.options["attributes"] == VG
    cfg_from_list(["ATTRIBUTES.EMBED_DIM", "128", "ATTRIBUTES.HIDDEN", "1024"])
    net.create_architecture("TEST", 1601, tag="default")
    assert net.options["attributes"] == (401, 128, 1024)
    with pytest.raises(AssertionError):
        cfg_from_list(["ATTRIBUTES.NUM_CLASSES", "401.0"])        # the strict merge keeps the int type
    with pytest.raises(KeyError):
        y.write_text("ATTRIBUTES:\n  NUM_ATTRIBUTES: 401\n")
        cfg_from_file(str(y))


@pytest.mark.parametrize("update", [
    dict(NUM_CLASSES=1), dict(NUM_CLASSES=-1), dict(NUM_CLASSES=4097), dict(NUM_CLASSES=401.0), dict(NUM_CLASSES=True),
    dict(NUM_CLASSES="401"), dict(EMBED_DIM=0), dict(EMBED_DIM=100), dict(EMBED_DIM=-32), dict(EMBED_DIM=256.0),
    dict(HIDDEN=0), dict(HIDDEN=500), dict(HIDDEN=None), dict(NUM_CLASSES=0, HIDDEN=16),
])
def test_invalid_values_raise_before_device_work(attr_cfg, monkeypatch, update):
    from tf_faster_rcnn_b200 import _native
    monkeypatch.setattr(_native, "lib", lambda: pytest.fail("device work before the refusal"))
    attr_cfg.ATTRIBUTES.NUM_CLASSES = 401
    attr_cfg.ATTRIBUTES.update(update)
    for name in ("res101", "vgg16", "mobile"):
        with pytest.raises(ValueError):
            make_net(name).create_architecture("TEST", 1601, tag="default")


@pytest.mark.parametrize("a", [0, 2, 401, 4096])
def test_valid_values(attr_cfg, a):
    from tf_faster_rcnn_b200 import engine
    attr_cfg.ATTRIBUTES.NUM_CLASSES = a
    attr_cfg.ATTRIBUTES.EMBED_DIM, attr_cfg.ATTRIBUTES.HIDDEN = 32, np.int64(64)
    assert engine.attributes_option(attr_cfg.ATTRIBUTES) == (None if a == 0 else (a, 32, 64))


# ---- checkpoint variables -----------------------------------------------------------------------------------------------------
ATTR_KEYS = ("cls_embedding/weights", "fc_attr/weights", "fc_attr/biases", "attr_score/weights", "attr_score/biases")


@pytest.mark.parametrize("net,scope,mult,fdim", [("res101", "resnet_v1_101", 1.0, 2048), ("res50", "resnet_v1_50", 1.0, 2048),
                                                 ("vgg16", "vgg_16", 1.0, 4096), ("mobile", "MobilenetV1", 1.0, 1024),
                                                 ("mobile", "MobilenetV1", 0.5, 512)])
def test_spec_lists_attribute_variables_only_with_the_head(net, scope, mult, fdim):
    from tf_faster_rcnn_b200 import synth
    off = synth.spec(net, 1601, 12, depth_multiplier=mult)
    on = synth.spec(net, 1601, 12, depth_multiplier=mult, attributes=(401, 64, 96))
    assert not any("attr" in k or "embedding" in k for k in off)
    assert {k: v for k, v in on.items() if k in off} == off
    extra = {k[len(scope) + 1:]: v for k, v in on.items() if k not in off}
    assert extra == {"cls_embedding/weights": (1601, 64), "fc_attr/weights": (fdim + 64, 96), "fc_attr/biases": (96,),
                     "attr_score/weights": (96, 401), "attr_score/biases": (401,)}
    # the drawn weights: the same variables as spec, the others bit-identical to a draw without the head
    if net in ("res50", "mobile"):
        w_off = synth.make(net, 21, 9, depth_multiplier=mult)
        w_on = synth.make(net, 21, 9, depth_multiplier=mult, attributes=(401, 64, 96))
        assert {k: v.shape for k, v in w_on.items()} == synth.spec(net, 21, 9, depth_multiplier=mult, attributes=(401, 64, 96))
        assert all(w_on[k].tobytes() == v.tobytes() for k, v in w_off.items())


def test_check_variables_reports_attribute_variables_only_with_the_head(attr_cfg):
    from tf_faster_rcnn_b200 import synth
    w = synth.make("res50", 21, 9)
    net = make_net("res50")
    net.create_architecture("TEST", 21, tag="default")
    assert net.check_variables(w) == []
    attr_cfg.ATTRIBUTES.NUM_CLASSES = 401
    net.create_architecture("TEST", 21, tag="default")
    problems = net.check_variables(w)
    assert len(problems) == 5 and all("not found" in p for p in problems)
    assert sorted(p.split()[1] for p in problems) == sorted("resnet_v1_50/" + k for k in ATTR_KEYS)
    good = synth.make("res50", 21, 9, attributes=VG)
    assert net.check_variables(good) == []
    bad = dict(good)
    bad["resnet_v1_50/fc_attr/weights"] = np.zeros((2048 + 128, 512), F)      # an embedding of another width
    problems = net.check_variables(bad)
    assert len(problems) == 1 and "fc_attr/weights" in problems[0]
    with pytest.raises(ValueError):
        net.load_weights(bad, strict=True)


# ---- the oracle's argmax rule -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("row", [
    [1.0, 3.0, 3.0, 2.0], [5.0, 5.0, 5.0], [-np.inf, -np.inf], [0.0, np.nan, 7.0, np.nan], [np.nan, np.nan],
    [np.inf, 1.0, np.inf], [-0.0, 0.0], [0.0, -0.0, 1e-45], [np.float32(3.4e38), np.inf, 2.0],
])
def test_argmax_rule_is_numpys(row):
    r = np.array(row, F)
    assert AO.argmax_rule(r) == int(np.argmax(r))


def test_argmax_rule_random_rows_with_ties():
    rng = np.random.default_rng(0)
    for _ in range(300):
        r = rng.integers(0, 4, rng.integers(2, 40)).astype(F)
        if rng.random() < 0.2:
            r[rng.integers(0, r.size)] = np.nan
        assert AO.argmax_rule(r) == int(np.argmax(r)) and AO.pick(r[None])[0][0] == 1 + int(np.argmax(r[1:]))


# ---- mutants: each plausible mistake fails a comparator ----------------------------------------------------------------------
def small_head(rng, C=6, A=5, E=32, H=32, Fd=32):
    sc = "net"
    w = {sc + "/cls_embedding/weights": rng.normal(0, 1, (C, E)).astype(F),
         sc + "/fc_attr/weights": rng.normal(0, 0.3, (Fd + E, H)).astype(F), sc + "/fc_attr/biases": rng.normal(0, 1, H).astype(F),
         sc + "/attr_score/weights": rng.normal(0, 0.5, (H, A)).astype(F), sc + "/attr_score/biases": rng.normal(0, 1, A).astype(F)}
    return sc, w


def outputs_agree(got, want):
    """The comparators of the GPU tests, applied to the float64 chain of a mutant: class and embedding exact, attr_prob within
    the softmax bound, attributes exact where decided."""
    S.check_exact(got["classes"], want["classes"], "classes")
    S.check_exact(got["emb"], want["emb"], "emb")
    p = got["attr_prob"]
    bound = np.maximum(want["attr_prob"], 2.0 ** -126) * 64 * AO.U
    S.check_bounded(p, want["attr_prob"], bound, "attr_prob")
    S.check_exact(got["attributes"], want["attributes"], "attributes")


@pytest.mark.parametrize("mutant", ["fg_only", "emb_first", "no_relu", "attr_from_0", "ties_last"])
def test_oracle_mutants_fail(mutant):
    rng = np.random.default_rng(5)
    sc, w = small_head(rng)
    n = 64
    fc7 = np.abs(rng.normal(0, 1, (n, 32))).astype(F)
    z = rng.normal(0, 1, (n, 6)).astype(F)
    z[:16, 0] = 10.0                                     # background wins: a foreground-only argmax picks another row
    z[16:32, 2] = z[16:32, 4] = 9.0                      # tied classes: first vs last
    want = AO.head64(fc7, z, w, sc)
    assert (want["classes"][:16] == 0).all() and (want["classes"][16:32] == 2).all()
    assert np.array_equal(want["classes"], np.argmax(z, axis=1))
    outputs_agree(want, want)
    if mutant == "ties_last":
        # ties on the attribute side as well: equal logits give equal probabilities
        w[sc + "/attr_score/weights"][:, 3] = w[sc + "/attr_score/weights"][:, 1]
        w[sc + "/attr_score/biases"][3] = w[sc + "/attr_score/biases"][1]
        want = AO.head64(fc7, z, w, sc)
    knobs = dict(fg_only=dict(fg_only=True), emb_first=dict(emb_first=True), no_relu=dict(relu=False),
                 attr_from_0=dict(attr_first=0), ties_last=dict(argmax=AO.argmax_last))[mutant]
    got = AO.head64(fc7, z, w, sc, **knobs)
    with pytest.raises(AssertionError):
        outputs_agree(got, want)


def test_check_attributes_has_teeth():
    rng = np.random.default_rng(9)
    s = rng.normal(0, 3, (50, 401)).astype(F)
    p64, bound = AO.softmax64(s, 401)
    p = p64.astype(F)
    a, c = AO.pick(p)
    AO.check_attributes(p, a, c, p64, bound)
    with pytest.raises(AssertionError):
        AO.check_attributes(p, a - 1, p[np.arange(50), a - 1], p64, bound)        # counted from column 0
    p2 = p.copy()
    p2[7, 20] *= F(1.001)
    with pytest.raises(AssertionError):
        AO.check_attributes(p2, a, c, p64, bound)


def test_fc64_bound_catches_a_dropped_term():
    rng = np.random.default_rng(3)
    x = np.abs(rng.normal(0, 1, (20, 64))).astype(F)
    w = rng.normal(0, 0.2, (64, 16)).astype(F)
    b = rng.normal(0, 1, 16).astype(F)
    y64, bound = AO.fc64(x, w, b, relu=False)
    S.check_bounded(y64.astype(F), y64, bound)
    dropped = (x[:, 1:].astype(np.float64) @ w[1:].astype(np.float64) + b).astype(F)
    with pytest.raises(AssertionError):
        S.check_bounded(dropped, y64, bound)


# ---- C ABI and compile --------------------------------------------------------------------------------------------------------
P = 1 << 20                                               # an aligned non-null address: every call below is refused before use


def embed_args(**kw):
    a = dict(cls_score=P, r=300, batch=2, C=81, index=P, count=P, M=100, table=P, E=256, out=P, stream=None)
    a.update(kw)
    return list(a.values())


def finish_args(**kw):
    a = dict(score=P, ld=404, batch=2, M=100, A=401, count=P, prob=P, attr=P, conf=P, stream=None)
    a.update(kw)
    return list(a.values())


@pytest.mark.parametrize("kw", [dict(cls_score=None), dict(index=None), dict(count=None), dict(table=None), dict(out=None),
                                dict(C=1), dict(C=4097), dict(C=0), dict(M=0), dict(M=301), dict(batch=0), dict(E=0), dict(E=6),
                                dict(table=P + 4), dict(out=P + 8), dict(batch=1 << 20, M=100, r=300)])
def test_embed_abi_refusals(kw):
    from tf_faster_rcnn_b200 import _native
    assert _native.lib().frcnn_regions_attr_embed(*embed_args(**kw)) == -2
    assert "regions_attr_embed" in _native.last_error()


@pytest.mark.parametrize("kw", [dict(score=None), dict(count=None), dict(prob=None), dict(attr=None), dict(conf=None), dict(A=1),
                                dict(A=4097), dict(M=0), dict(batch=0), dict(ld=400), dict(prob=P + 2), dict(score=P + 1)])
def test_finish_abi_refusals(kw):
    from tf_faster_rcnn_b200 import _native
    assert _native.lib().frcnn_attr_finish(*finish_args(**kw)) == -2
    assert "attr_finish" in _native.last_error()


@pytest.mark.parametrize("kernel", ["regions_attr_embed_kernel", "attr_finish_kernel"])
def test_new_kernels_do_not_spill(kernel):
    """ptxas -v output written by the build."""
    log = open(os.path.join(ROOT, "tf_faster_rcnn_b200", "csrc", "_obj", "attributes.o.log")).read()
    found = re.findall(r"Function properties for \w*%s\w*\n\s*([^\n]*)" % kernel, log)
    assert len(found) == 1, "ptxas reports for %s: %d" % (kernel, len(found))
    assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in found[0], found[0]


def test_tool_options():
    from tf_faster_rcnn_b200 import synth
    import subprocess
    tmp = os.path.join(os.environ.get("TMPDIR", "/tmp"), "attr_ckpt_%d" % os.getpid())
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "make_synthetic_ckpt.py"), "--net", "mobile", "--classes", "5",
                        "--anchors", "9", "--attributes", "7", "--attr_embed", "32", "--attr_hidden", "64", "--out", tmp],
                       capture_output=True, text=True, cwd=ROOT)
    try:
        assert r.returncode == 0, r.stderr[-2000:]
        z = np.load(tmp + ".npz")
        assert {k: z[k].shape for k in z.files} == synth.spec("mobile", 5, 9, attributes=(7, 32, 64))
    finally:
        for ext in (".npz", ".meta"):
            if os.path.exists(tmp + ext):
                os.remove(tmp + ext)
