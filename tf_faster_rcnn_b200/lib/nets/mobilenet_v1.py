"""MobileNet-v1 (lib/nets/mobilenet_v1.py:63-172, 214-250): Conv2d_0 + 11 depthwise-separable layers as the
body, layers 12-13 + spatial mean as the per-RoI head.  Depthwise 3x3 is a bandwidth kernel; every pointwise
1x1 runs on the wgmma GEMM path.  BN eps 1e-3, ReLU6."""
import numpy as np

from model.config import cfg
from nets.network import Network
from tf_faster_rcnn_b200 import _native as N, engine

# (kind, stride, depth)
_DEFS = [("conv", 2, 32), ("sep", 1, 64), ("sep", 2, 128), ("sep", 1, 128), ("sep", 2, 256), ("sep", 1, 256),
         ("sep", 2, 512), ("sep", 1, 512), ("sep", 1, 512), ("sep", 1, 512), ("sep", 1, 512), ("sep", 1, 512),
         ("sep", 1, 1024), ("sep", 1, 1024)]
_EPS = 1e-3
KBLOCK = 32          # the conv kernel takes input depths in multiples of its 32-channel k-block
FIRST_COUTS = (32, 64)   # the output depths frcnn_conv_first takes


def layer_depths(depth_multiplier, min_depth=8):
    """The output depth of each of the 14 layers (mobilenet_v1_base: max(int(d * depth_multiplier), min_depth))."""
    return [max(int(d * depth_multiplier), min_depth) for _, _, d in _DEFS]


def padded_depth(d):
    return -(-d // KBLOCK) * KBLOCK


def check_depth_multiplier(depth_multiplier):
    """cfg.MOBILENET.DEPTH_MULTIPLIER -> the layer depths; ValueError before any device work when the device cannot run them.
    Layers narrower than a multiple of 32 channels run zero-padded to one (pad_depths); the first layer's padded depth must
    be one that frcnn_conv_first takes, and the depths the RPN and the head FCs read (layers 11 and 13) are not padded."""
    m = depth_multiplier
    if isinstance(m, (bool, np.bool_)) or not isinstance(m, (int, float, np.integer, np.floating)) or not np.isfinite(m) or m <= 0:
        raise ValueError("MOBILENET.DEPTH_MULTIPLIER must be a finite number > 0, got %r" % (m,))
    d = layer_depths(float(m))
    if any(v % 4 for v in d):
        raise ValueError("MOBILENET.DEPTH_MULTIPLIER %r gives layer depths %s: every depth must be a multiple of 4" % (m, d))
    if padded_depth(d[0]) not in FIRST_COUTS:
        raise ValueError("MOBILENET.DEPTH_MULTIPLIER %r gives Conv2d_0 depth %d: at most %d is supported" % (m, d[0], FIRST_COUTS[-1]))
    if d[11] % KBLOCK or d[13] % KBLOCK:
        raise ValueError("MOBILENET.DEPTH_MULTIPLIER %r gives feature depths %d (RPN) and %d (head): both must be multiples of %d"
                         % (m, d[11], d[13], KBLOCK))
    return d


def pad_depths(tensors):
    """The checkpoint tensors with every layer's depth padded up to a multiple of KBLOCK by zero channels: zero filter taps,
    and BatchNorm gamma = beta = mean = 0, variance 1, so a pad channel's output is exactly 0 and it adds exact zeros to the
    next layer's sums.  Unchanged (the same dict) when every depth already is a multiple of KBLOCK."""
    sc = "MobilenetV1"
    depths = [int(tensors["%s/Conv2d_%d/weights" % (sc, 0)].shape[3])]
    for i in range(1, len(_DEFS)):
        depths.append(int(tensors["%s/Conv2d_%d_pointwise/weights" % (sc, i)].shape[3]))
    if all(d % KBLOCK == 0 for d in depths):
        return tensors
    t = dict(tensors)

    def pad(key, axis, n, value=0.0):
        a = np.asarray(t[key])
        if a.shape[axis] < n:
            width = [(0, 0)] * a.ndim
            width[axis] = (0, n - a.shape[axis])
            t[key] = np.pad(a, width, constant_values=value).astype(a.dtype)

    def pad_bn(name, n):
        for leaf in ("gamma", "beta", "moving_mean"):
            pad(name + "/BatchNorm/" + leaf, 0, n)
        pad(name + "/BatchNorm/moving_variance", 0, n, 1.0)

    cin = 3
    for i, d in enumerate(depths):
        p = padded_depth(d)
        if i == 0:
            pad("%s/Conv2d_0/weights" % sc, 3, p); pad_bn("%s/Conv2d_0" % sc, p)
        else:
            dw, pw = "%s/Conv2d_%d_depthwise" % (sc, i), "%s/Conv2d_%d_pointwise" % (sc, i)
            pad(dw + "/depthwise_weights", 2, cin); pad_bn(dw, cin)
            pad(pw + "/weights", 2, cin); pad(pw + "/weights", 3, p); pad_bn(pw, p)
        cin = p
    return t


class mobilenetv1(Network):
    def __init__(self):
        Network.__init__(self)
        self._depth_multiplier = cfg.MOBILENET.DEPTH_MULTIPLIER
        self._scope = 'MobilenetV1'

    def create_architecture(self, mode, num_classes, tag=None, anchor_scales=(8, 16, 32), anchor_ratios=(0.5, 1, 2)):
        check_depth_multiplier(self._depth_multiplier)
        return Network.create_architecture(self, mode, num_classes, tag, anchor_scales, anchor_ratios)

    def load_weights(self, tensors, strict=False):
        Network.load_weights(self, tensors, strict)
        self.weights = engine.Weights(pad_depths(self.weights.t))

    def _layers_range(self, t, x, first, last):
        for i in range(first, last):
            kind, stride, _ = _DEFS[i]
            if kind == "conv":
                x = t.conv_first(x, "MobilenetV1/Conv2d_%d" % i, 3, stride, "EXPLICIT", N.ACT_RELU6, _EPS)
            else:
                x = t.depthwise(x, "MobilenetV1/Conv2d_%d_depthwise" % i, stride, N.ACT_RELU6, _EPS)
                x = t.conv(x, "MobilenetV1/Conv2d_%d_pointwise" % i, 1, "SAME", N.ACT_RELU6, _EPS)
        return x

    def _image_to_head(self, t, image):
        x = self._layers_range(t, image, 0, 12)
        self._layers['head'] = x
        return x

    def _head_to_tail(self, t, pool5):
        return t.spatial_mean(self._layers_range(t, pool5, 12, 14))
