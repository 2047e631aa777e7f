"""ResNet-v1-50/101/152 (lib/nets/resnet_v1.py:80-152 + slim's bottleneck_v1) on the device tape.
BatchNorm (eps 1e-5, frozen) is the conv epilogue's scale/shift; the residual add + ReLU is fused into the
closing 1x1 conv's epilogue, a projection shortcut into that conv's K loop, and the head's spatial mean into the last
conv's epilogue."""
from nets.network import Network
from tf_faster_rcnn_b200 import _native as N

_UNITS = {50: (3, 4, 6, 3), 101: (3, 4, 23, 3), 152: (3, 8, 36, 3)}
_EPS = 1e-5


class resnetv1(Network):
    def __init__(self, num_layers=50):
        Network.__init__(self)
        if num_layers not in _UNITS:
            raise NotImplementedError
        self._num_layers = num_layers
        self._scope = 'resnet_v1_%d' % num_layers
        n1, n2, n3, n4 = _UNITS[num_layers]
        # (name, base depth, per-unit strides): stride sits on the LAST unit (resnet_v1_block); block3/4 stride 1
        self._blocks = [("block1", 64, [1] * (n1 - 1) + [2]), ("block2", 128, [1] * (n2 - 1) + [2]),
                        ("block3", 256, [1] * n3), ("block4", 512, [1] * n4)]

    def crop_pre_pool(self):
        return bool(self.options["resnet_max_pool"])     # default: crop 7x7 directly (resnet_v1.py:68-75)

    def _bottleneck(self, t, x, prefix, base, stride, mean=False):
        """mean: return each RoI's spatial mean of the unit's output instead of the map (the head's last unit)."""
        depth = 4 * base
        r = t.conv(x, prefix + "/conv1", 1, "SAME", N.ACT_RELU, _EPS)
        r = t.conv(r, prefix + "/conv2", stride, "SAME" if stride == 1 else "EXPLICIT", N.ACT_RELU, _EPS)
        if x.shape[3] == depth:
            shortcut = x if stride == 1 else t.max_pool(x, 1, stride, "VALID")
            return t.conv(r, prefix + "/conv3", 1, "SAME", N.ACT_RELU, _EPS, residual=shortcut, mean=mean)
        # projection shortcut: linear, so conv3 computes it in its own K loop, relu(r.W3' + x.Wsc' + (b3 + bsc)) with the two
        # BatchNorm scales folded into the weights -- the shortcut's output never goes through memory
        assert stride == 1
        pc = t.w.packed_concat([prefix + "/conv3", prefix + "/shortcut"], _EPS)
        return t.conv(r, prefix + "/conv3", 1, "SAME", N.ACT_RELU, packed=pc, x2=x, mean=mean)

    def _run_blocks(self, t, x, blocks, mean_last=False):
        for bi, (bname, base, strides) in enumerate(blocks):
            for u, s in enumerate(strides, start=1):
                last = bi == len(blocks) - 1 and u == len(strides)
                x = self._bottleneck(t, x, "%s/%s/unit_%d/bottleneck_v1" % (self._scope, bname, u), base, s, mean_last and last)
        return x

    def _image_to_head(self, t, image):
        x = t.conv_first(image, self._scope + "/conv1", 7, 2, "EXPLICIT", N.ACT_RELU, _EPS)
        x = t.max_pool(x, 3, 2, "ZEROPAD1")               # tf.pad 1 + 3x3/2 VALID (resnet_v1.py:83-84)
        x = self._run_blocks(t, x, self._blocks[:3])
        self._layers['head'] = x
        return x

    def _head_to_tail(self, t, pool5):
        # fc7 = the spatial mean of block4, reduced in the last conv3's epilogue: the 7x7 map itself has no reader
        return self._run_blocks(t, pool5, self._blocks[3:], mean_last=True)
