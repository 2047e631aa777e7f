"""Minimal stand-in for the handful of TensorFlow-1.x symbols the reference's tools touch
(tools/demo.py:24,129-144; tools/test_net.py:18,86-117) so that they can drive this engine unchanged.
Only used when a real `tensorflow` is not importable (tf_faster_rcnn_b200.paths.add_lib_path(with_shims=True)).
No graph, no ops: the Session is an opaque token; Saver.restore reads a TF V2 checkpoint (or an .npz) of TF-named variables."""

__version__ = "1.x-shim (tf_faster_rcnn_b200)"


class _GPUOptions(object):
    allow_growth = False


class ConfigProto(object):
    def __init__(self, allow_soft_placement=False, **kw):
        self.allow_soft_placement = allow_soft_placement
        self.gpu_options = _GPUOptions()


class _InitOp(object):
    pass


def global_variables_initializer():
    return _InitOp()


def _networks():
    from nets import network
    return list(network._REGISTRY)


class Session(object):
    def __init__(self, config=None, **kw):
        self.config = config

    def run(self, fetches, feed_dict=None):
        if isinstance(fetches, _InitOp):
            # test_net.py:116-117 path (no --model): seeded synthetic initialisation
            from tf_faster_rcnn_b200 import synth
            for net in _networks():
                if net.weights is None:
                    net.load_weights(synth.make(net.arch_name(), net.num_classes, net.num_anchors,
                                                rpn_channels=int(net.options["rpn_channels"]),
                                                pooling_size=int(net.options["pooling_size"]),
                                                depth_multiplier=float(getattr(net, "_depth_multiplier", 1.0)),
                                                attributes=net.options["attributes"]))
            return None
        raise NotImplementedError("tensorflow shim: Session.run only supports the variable initializer; "
                                  "inference goes through Network.test_image / im_detect")

    def close(self):
        pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False


class _Saver(object):
    def restore(self, sess, save_path):
        """Assigns every variable found under `save_path`: a TensorFlow V2 checkpoint (`.index` + `.data-*`, read by
        tf_faster_rcnn_b200.checkpoint without TensorFlow) or, failing that, `<save_path>.npz` keyed by TF names."""
        from tf_faster_rcnn_b200 import checkpoint
        tensors = checkpoint.load_variables(save_path)
        for net in _networks():
            net.load_weights(tensors, strict=True)         # missing keys / shape mismatches raise, as a TF restore does


class _Train(object):
    Saver = _Saver


train = _Train()
