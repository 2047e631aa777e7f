#!/usr/bin/env python
"""Cost of test-time augmentation (TEST.BBOX_AUG) on the bench.py workload: ResNet-101, one 600x800 synthetic image per slot
(base view 600x800), 300 proposals per view, 81 classes, seeded synthetic weights, device-resident inputs, greedy NMS.

    python tools/bench_aug.py [--batches 1,4] [--steps 30] [--warmup 3] [--rounds 3]

Configurations (view shapes of a 600x800 image):
  plain          Network.detect / detect_batch: one 600x800 graph replay (no augmentation)
  1view          BBOX_AUG enabled, no flip, no extra scale: the augmented path with one view
  flip           H_FLIP: base + mirrored base, one batch-2B replay of the 600x800 plan
  3scales_flip   H_FLIP, SCALES (480, 720): six views, three batch-2B plans (480x640, 720x960, 600x800)

Prints one JSON line.  Per batch and configuration: images/s of the whole call (sub-plan graph replays + the union/post graph),
and, for the augmented ones, the sub-plan graphs alone and the union + post graph alone (ms per call); best of --rounds rounds of
--steps calls, the configurations timed alternately (CUDA events).  gpu: card name, power limit and max SM clock read in the same
run."""
import argparse
import json
import subprocess
import sys

import _init_paths  # noqa: F401
import cv2
import numpy as np
import torch

from model.config import cfg
from model.test import _set_post_options, aug_view_blob, aug_views
from nets.resnet_v1 import resnetv1
from tf_faster_rcnn_b200 import _native, synth

C, ANCHORS, H0, W0 = 81, (4, 8, 16, 32), 600, 800
CONFIGS = (("1view", dict(H_FLIP=False, SCALES=())), ("flip", dict(H_FLIP=True, SCALES=())),
           ("3scales_flip", dict(H_FLIP=True, SCALES=(480, 720))))


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=10).stdout.strip()
        return out or torch.cuda.get_device_name()
    except Exception:
        return torch.cuda.get_device_name()


def timed_ms(fn, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def setup(net, ims):
    """-> {name: (call, sub-plan graphs only, union + post only)} with every input already on the device."""
    B = len(ims)
    hws = [im.shape[:2] for im in ims]
    out = {}
    base = [aug_view_blob(im, cfg.TEST.SCALES[0], cfg.TEST.MAX_SIZE, False) for im in ims]
    plan = net.plan_for(base[0][0].shape[1], base[0][0].shape[2], B)
    plan.image.copy_(torch.from_numpy(np.concatenate([b[0] for b in base])))
    meta = [(b[1], h, w) for b, (h, w) in zip(base, hws)]
    out["plain"] = (lambda: plan.launch(post=True, detect=True, meta=meta), None, None)
    for name, upd in CONFIGS:
        cfg.TEST.BBOX_AUG.update(ENABLED=True, **upd)
        views = aug_views(ims[0].shape)
        blobs = [[aug_view_blob(im, *v) for im in ims] for v in views]
        aug = net.aug_plan([(bl[0][0].shape[1], bl[0][0].shape[2], v[2]) for bl, v in zip(blobs, views)], B)
        for v, bl in enumerate(blobs):
            aug.view_image(v).copy_(torch.from_numpy(np.concatenate([x[0] for x in bl])))
        scales = [[x[1] for x in bl] for bl in blobs]
        aug.launch(scales, hws)                                     # captures the sub-plan and union/post graphs
        aug.launch(scales, hws)
        subs = [p.graphs["im_detect"] for p in aug.subs.values()]
        out[name] = (lambda aug=aug, scales=scales: aug.launch(scales, hws), lambda subs=subs: [g.replay() for g in subs],
                     lambda aug=aug: aug.graphs[("detect", aug.slot)].replay())
    cfg.TEST.BBOX_AUG.ENABLED = False
    return out


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,4")
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args(argv)
    _native.check(_native.lib().frcnn_check_device(torch.cuda.current_device()), "check_device")
    cfg.TEST.HAS_RPN = True
    cfg.TEST.RPN_POST_NMS_TOP_N = 300
    weights = synth.make("res101", C, 3 * len(ANCHORS), 3)
    result = {}
    for B in [int(b) for b in args.batches.split(",")]:
        net = resnetv1(101)
        net.create_architecture("TEST", C, tag="default", anchor_scales=ANCHORS, anchor_ratios=(0.5, 1, 2))
        net.load_weights(weights)
        net.MAX_PLANS = 8                                           # every plan of the four configurations stays resident
        _set_post_options(net, 0.0, 100)
        rng = np.random.default_rng(B)
        ims = [cv2.blur(rng.integers(0, 256, (H0, W0, 3), dtype=np.uint8), (5, 5)) for _ in range(B)]
        calls = setup(net, ims)
        for fn, _, _ in calls.values():
            for _ in range(args.warmup):
                fn()
        best = {name: [float("inf")] * 3 for name in calls}
        for _ in range(max(1, args.rounds)):
            for name, fns in calls.items():
                for k, fn in enumerate(fns):
                    if fn is not None:
                        best[name][k] = min(best[name][k], timed_ms(fn, args.steps))
        result["batch%d" % B] = {
            name: dict(images_per_s=B * 1000.0 / t[0], ms_per_call=t[0],
                       **({} if name == "plain" else dict(sub_plan_graphs_ms=t[1], union_post_ms=t[2])))
            for name, t in best.items()}
        del calls, net
        torch.cuda.empty_cache()
    if "batch1" in result:       # time of one image with its flip over one plain batch-1 detect
        result["flip_over_plain_batch1"] = result["batch1"]["flip"]["ms_per_call"] / result["batch1"]["plain"]["ms_per_call"]
    line = {"workload": "res101 600x800 synthetic uint8 images, 300 proposals per view, %d classes, device-resident, greedy NMS 0.3, "
                        "max_per_image 100; 3scales_flip = SCALES (480, 720) + H_FLIP" % C,
            "results": result, "steps": args.steps, "rounds": args.rounds, "gpu": gpu_info()}
    print(json.dumps(line))


if __name__ == "__main__":
    sys.exit(main())
