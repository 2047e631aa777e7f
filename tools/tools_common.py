from model.config import cfg
from nets.vgg16 import vgg16
from nets.resnet_v1 import resnetv1
from nets.mobilenet_v1 import mobilenetv1
from tf_faster_rcnn_b200 import checkpoint, synth


def build_net(net_name, num_classes, model=None):
    cfg.TEST.HAS_RPN = True
    net = vgg16() if net_name == "vgg16" else mobilenetv1() if net_name == "mobile" else resnetv1(int(net_name[3:]))
    net.create_architecture("TEST", num_classes, tag="default", anchor_scales=cfg.ANCHOR_SCALES, anchor_ratios=cfg.ANCHOR_RATIOS)
    if model:
        net.load_weights(checkpoint.load_variables(model), strict=True)   # TF V2 bundle or .npz
    else:
        net.load_weights(synth.make(net_name, num_classes, net.num_anchors, attributes=net.options["attributes"]))
    return net
