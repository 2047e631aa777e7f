"""Seeded synthetic weights + input blobs under the reference's TF variable names.

Product-side helper (bench.py, smoke, tests feed BOTH the CUDA path and the oracle from it;
the oracle itself never generates weights).

No checkpoints exist offline, so parity/bench use random-init weights of the exact
architectures, keyed by the slim variable scopes the reference builds
(SURVEY.md section 5 'Checkpoint / resume'): HWIO conv kernels, [in,out] FC matrices,
BatchNorm/{gamma,beta,moving_mean,moving_variance}.  He-scaled so that activations stay
O(1) through 100+ layers; the residual-branch closing BN gets a small gamma so the
running sum does not blow up.  Same generator feeds the oracle and the CUDA path.
"""
import zlib
import numpy as np

F = np.float32


def _rng(seed, name):
    return np.random.default_rng((zlib.crc32(name.encode()) + 7919 * seed) % (2 ** 31))


class _Gen:
    def __init__(self, seed, shapes_only=False):
        self.seed = seed
        self.shapes_only = shapes_only          # record {name: shape} instead of drawing values (spec())
        self.w = {}

    def conv(self, name, kh, kw, cin, cout, std=None, bias=False, bias_std=0.01):
        if self.shapes_only:
            self.w[name + "/weights"] = (kh, kw, cin, cout)
            if bias:
                self.w[name + "/biases"] = (cout,)
            return
        r = _rng(self.seed, name)
        s = np.sqrt(2.0 / (kh * kw * cin)) if std is None else std
        self.w[name + "/weights"] = (r.standard_normal((kh, kw, cin, cout)) * s).astype(F)
        if bias:
            self.w[name + "/biases"] = (r.standard_normal(cout) * bias_std).astype(F)

    def dw(self, name, k, c):
        if self.shapes_only:
            self.w[name + "/depthwise_weights"] = (k, k, c, 1)
            return
        r = _rng(self.seed, name)
        self.w[name + "/depthwise_weights"] = (r.standard_normal((k, k, c, 1)) * np.sqrt(2.0 / (k * k))).astype(F)

    def bn(self, name, c, gamma=(0.5, 1.5)):
        p = name + "/BatchNorm/"
        if self.shapes_only:
            for leaf in ("gamma", "beta", "moving_mean", "moving_variance"):
                self.w[p + leaf] = (c,)
            return
        r = _rng(self.seed, name + "/BatchNorm")
        self.w[p + "gamma"] = r.uniform(gamma[0], gamma[1], c).astype(F)
        self.w[p + "beta"] = (r.standard_normal(c) * 0.1).astype(F)
        self.w[p + "moving_mean"] = (r.standard_normal(c) * 0.1).astype(F)
        self.w[p + "moving_variance"] = r.uniform(0.5, 1.5, c).astype(F)

    def fc(self, name, cin, cout, std=None, bias_std=0.01):
        if self.shapes_only:
            self.w[name + "/weights"] = (cin, cout)
            self.w[name + "/biases"] = (cout,)
            return
        r = _rng(self.seed, name)
        s = np.sqrt(2.0 / cin) if std is None else std
        self.w[name + "/weights"] = (r.standard_normal((cin, cout)) * s).astype(F)
        self.w[name + "/biases"] = (r.standard_normal(cout) * bias_std).astype(F)

    def heads(self, scope, c_body, c_tail, num_classes, num_anchors, rpn_channels=512, attributes=None):
        """lib/nets/network.py:323-378: rpn_conv/3x3 (bias+ReLU, no BN), two 1x1 RPN heads, two FCs; with attributes = (A, E, H)
        also the attribute head: cls_embedding [C, E], fc_attr [c_tail + E, H], attr_score [H, A]."""
        self.conv(scope + "/rpn_conv/3x3", 3, 3, c_body, rpn_channels, bias=True)
        self.conv(scope + "/rpn_cls_score", 1, 1, rpn_channels, 2 * num_anchors, std=0.05, bias=True, bias_std=0.5)
        self.conv(scope + "/rpn_bbox_pred", 1, 1, rpn_channels, 4 * num_anchors, std=0.01, bias=True)
        self.fc(scope + "/cls_score", c_tail, num_classes, std=0.02, bias_std=0.5)
        self.fc(scope + "/bbox_pred", c_tail, 4 * num_classes, std=0.01)
        if attributes is not None:
            a, e, h = attributes
            self.embedding(scope + "/cls_embedding", num_classes, e)
            self.fc(scope + "/fc_attr", c_tail + e, h)
            self.fc(scope + "/attr_score", h, a, std=0.05, bias_std=0.5)

    def embedding(self, name, n, dim):
        if self.shapes_only:
            self.w[name + "/weights"] = (n, dim)
            return
        self.w[name + "/weights"] = (_rng(self.seed, name).standard_normal((n, dim)) * 0.5).astype(F)


RESNET_UNITS = {50: (3, 4, 6, 3), 101: (3, 4, 23, 3), 152: (3, 8, 36, 3)}


def resnet_block_plan(num_layers):
    """[(block_name, base_depth, [unit strides])] per lib/nets/resnet_v1.py:127-152 and slim's
    resnet_v1_block (stride sits on the LAST unit)."""
    n1, n2, n3, n4 = RESNET_UNITS[num_layers]
    return [("block1", 64, [1] * (n1 - 1) + [2]), ("block2", 128, [1] * (n2 - 1) + [2]),
            ("block3", 256, [1] * n3), ("block4", 512, [1] * n4)]


def make_vgg16(num_classes, num_anchors, seed=3, shapes_only=False, rpn_channels=512, pooling_size=7, attributes=None):
    g = _Gen(seed, shapes_only)
    cin = 3
    for b, (n, c) in enumerate([(2, 64), (2, 128), (3, 256), (3, 512), (3, 512)], start=1):
        for i in range(1, n + 1):
            # the first conv also maps the +-120 pixel range down to O(1) activations
            g.conv("vgg_16/conv%d/conv%d_%d" % (b, b, i), 3, 3, cin, c, bias=True,
                   std=(np.sqrt(2.0 / 27) / 60.0 if cin == 3 else None))
            cin = c
    g.fc("vgg_16/fc6", pooling_size * pooling_size * 512, 4096)      # fc6 reads the flattened P x P x 512 pool5
    g.fc("vgg_16/fc7", 4096, 4096)
    g.heads("vgg_16", 512, 4096, num_classes, num_anchors, rpn_channels, attributes)
    return g.w


def make_resnet(num_layers, num_classes, num_anchors, seed=3, shapes_only=False, rpn_channels=512, attributes=None):
    g = _Gen(seed, shapes_only)
    sc = "resnet_v1_%d" % num_layers
    g.conv(sc + "/conv1", 7, 7, 3, 64, std=np.sqrt(2.0 / 147) / 60.0); g.bn(sc + "/conv1", 64)
    cin = 64
    for bname, base, strides in resnet_block_plan(num_layers):
        for u, _ in enumerate(strides, start=1):
            p = "%s/%s/unit_%d/bottleneck_v1" % (sc, bname, u)
            if cin != base * 4:
                g.conv(p + "/shortcut", 1, 1, cin, base * 4); g.bn(p + "/shortcut", base * 4, gamma=(0.3, 0.7))
            g.conv(p + "/conv1", 1, 1, cin, base); g.bn(p + "/conv1", base)
            g.conv(p + "/conv2", 3, 3, base, base); g.bn(p + "/conv2", base)
            g.conv(p + "/conv3", 1, 1, base, base * 4); g.bn(p + "/conv3", base * 4, gamma=(0.1, 0.3))
            cin = base * 4
    g.heads(sc, 1024, 2048, num_classes, num_anchors, rpn_channels, attributes)
    return g.w


MOBILENET_DEFS = [("conv", 2, 32), ("sep", 1, 64), ("sep", 2, 128), ("sep", 1, 128), ("sep", 2, 256),
                  ("sep", 1, 256), ("sep", 2, 512), ("sep", 1, 512), ("sep", 1, 512), ("sep", 1, 512),
                  ("sep", 1, 512), ("sep", 1, 512), ("sep", 1, 1024), ("sep", 1, 1024)]


def mobilenet_depth(d, mult=1.0, min_depth=8):
    return max(int(d * mult), min_depth)


def make_mobilenet(num_classes, num_anchors, seed=3, mult=1.0, shapes_only=False, rpn_channels=512, attributes=None):
    g = _Gen(seed, shapes_only)
    sc = "MobilenetV1"
    cin = 3
    for i, (kind, _, d) in enumerate(MOBILENET_DEFS):
        c = mobilenet_depth(d, mult)
        if kind == "conv":
            g.conv("%s/Conv2d_%d" % (sc, i), 3, 3, cin, c, std=np.sqrt(2.0 / 27) / 60.0); g.bn("%s/Conv2d_%d" % (sc, i), c)
        else:
            g.dw("%s/Conv2d_%d_depthwise" % (sc, i), 3, cin); g.bn("%s/Conv2d_%d_depthwise" % (sc, i), cin)
            g.conv("%s/Conv2d_%d_pointwise" % (sc, i), 1, 1, cin, c); g.bn("%s/Conv2d_%d_pointwise" % (sc, i), c)
        cin = c
    g.heads(sc, mobilenet_depth(512, mult), mobilenet_depth(1024, mult), num_classes, num_anchors, rpn_channels, attributes)
    return g.w


def make(net, num_classes, num_anchors, seed=3, shapes_only=False, rpn_channels=512, depth_multiplier=1.0, pooling_size=7,
         attributes=None):
    """net in {'vgg16','res50','res101','res152','mobile'} (tools/test_net.py:92-103 names).  pooling_size (cfg.POOLING_SIZE)
    sets VGG16's fc6 rows, P * P * 512; the other networks do not depend on it.  attributes: None (no attribute head), or
    (A, E, H) of cfg.ATTRIBUTES for the attribute head's variables; the other variables are the same either way."""
    if net == "vgg16":
        return make_vgg16(num_classes, num_anchors, seed, shapes_only, rpn_channels, pooling_size, attributes)
    if net.startswith("res"):
        return make_resnet(int(net[3:]), num_classes, num_anchors, seed, shapes_only, rpn_channels, attributes)
    if net == "mobile":
        return make_mobilenet(num_classes, num_anchors, seed, depth_multiplier, shapes_only, rpn_channels, attributes)
    raise ValueError(net)


def spec(net, num_classes, num_anchors, **arch):
    """{TF variable name: shape} the TEST graph of `net` restores (the variables `make` draws), without drawing them.
    arch: rpn_channels (cfg.RPN_CHANNELS), depth_multiplier (cfg.MOBILENET.DEPTH_MULTIPLIER), pooling_size (cfg.POOLING_SIZE),
    attributes (None, or (A, E, H): engine.attributes_option of cfg.ATTRIBUTES)."""
    return make(net, num_classes, num_anchors, shapes_only=True, **arch)


def check(net, tensors, num_classes, num_anchors, limit=12, **arch):
    """Problems that would make `Saver.restore` fail in the reference: variables of the TEST graph that are missing from
    `tensors`, or present with another shape (wrong class count / anchor set / backbone).  Extra variables (optimizer
    slots, global_step) are ignored, as a restore ignores them.  Returns a list of messages, empty when compatible."""
    problems = []
    for name, shape in spec(net, num_classes, num_anchors, **arch).items():
        if name not in tensors:
            problems.append("Key %s not found in checkpoint" % name)
        elif tuple(np.shape(tensors[name])) != tuple(shape):
            problems.append("%s: checkpoint has shape %s, the %s graph for %d classes / %d anchors needs %s"
                            % (name, list(np.shape(tensors[name])), net, num_classes, num_anchors, list(shape)))
    if len(problems) > limit:
        problems = problems[:limit] + ["... and %d more" % (len(problems) - limit)]
    return problems


def synthetic_blob(h, w, seed=3):
    """COCO/VOC-shaped input blob: uint8 noise, 5x5 box-blurred, minus PIXEL_MEANS; fp32 [1,h,w,3]."""
    import cv2
    r = np.random.default_rng(seed)
    im = r.integers(0, 256, (h, w, 3), dtype=np.uint8).astype(F)
    im = cv2.blur(im, (5, 5))
    im = (im - im.mean()) * F(3.0) + F(115.0)
    im = np.clip(im, 0, 255).astype(F) - np.array([[[102.9801, 115.9465, 122.7717]]], dtype=F)
    return np.ascontiguousarray(im[None], dtype=F)
