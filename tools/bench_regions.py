#!/usr/bin/env python
"""Cost of the bottom-up regions (Network.detect_regions) on the bench.py workload: ResNet-101, 600x800 synthetic blobs, 300
proposals, 81 classes, seeded synthetic weights, device-resident input.

    python tools/bench_regions.py [--net res101|vgg16|mobile] [--batch 4] [--steps 50] [--warmup 5] [--rounds 3]

Prints one JSON line:
  detect / regions    images/s of the detect graph (network + box decode + per-class NMS + cap + records) and of the regions
                      graph (network + the regions step: RoI-box broadcast, per-class NMS over every RoI, fold, selection, fc7
                      gather), on the same plan and images, timed alternately for --rounds rounds of --steps graph replays (CUDA
                      events); best round of each
  step                the regions step alone (frcnn_detect_regions: its five launches): 20 back-to-back steps per graph replay,
                      CUDA events, per batch
  gpu                 card name, power limit and max SM clock read in the same run"""
import argparse
import json
import sys

import _init_paths  # noqa: F401
import numpy as np
import torch

from bench_features import NETS, gpu_info, timed_ms
from model.config import cfg
from nets.mobilenet_v1 import mobilenetv1
from nets.resnet_v1 import resnetv1
from nets.vgg16 import vgg16
from tf_faster_rcnn_b200 import _native, engine, synth


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--net", default="res101", choices=sorted(NETS))
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args(argv)
    _native.check(_native.lib().frcnn_check_device(torch.cuda.current_device()), "check_device")
    C, scales = NETS[args.net]
    H, W, B = 600, 800, max(1, args.batch)
    cfg.TEST.HAS_RPN = True
    cfg.TEST.RPN_POST_NMS_TOP_N = 300
    cfg.USE_GPU_NMS = False
    net = vgg16() if args.net == "vgg16" else mobilenetv1() if args.net == "mobile" else resnetv1(int(args.net[3:]))
    net.create_architecture("TEST", C, tag="default", anchor_scales=scales, anchor_ratios=(0.5, 1, 2))
    net.load_weights(synth.make(args.net, C, 3 * len(scales), 3))
    blobs = np.concatenate([synth.synthetic_blob(H, W, 3 + b) for b in range(B)], axis=0)
    plan = net.plan_for(H, W, B)
    plan.image.copy_(torch.from_numpy(blobs))
    reg = engine.region_args(0.2, 10, 100)

    def detect():
        plan.launch(post=True, detect=True)

    def regions():
        plan.launch(regions=reg)

    for _ in range(max(args.warmup, 1)):
        detect()
        regions()
    best = {"detect": float("inf"), "regions": float("inf")}
    for _ in range(max(args.rounds, 1)):
        for name, fn in (("detect", detect), ("regions", regions)):
            best[name] = min(best[name], timed_ms(fn, args.steps) / args.steps)
    REP, NREP = 20, 10
    g = engine.LaunchGraph([plan.regions_step] * REP)
    g.replay()
    step_us = timed_ms(g.replay, NREP) * 1000.0 / (REP * NREP)
    counts = plan.reg_out["count"].cpu().tolist()
    line = {"workload": "%s %dx%d synthetic, 300 proposals, %d classes, batch %d, device-resident" % (args.net, H, W, C, B),
            "detect": {"value": B * 1000.0 / best["detect"], "unit": "images/s", "ms_per_step": best["detect"]},
            "regions": {"value": B * 1000.0 / best["regions"], "unit": "images/s", "ms_per_step": best["regions"],
                        "api": "Network.detect_regions(conf_thresh=0.2, min_boxes=10, max_boxes=100): one graph replay"},
            "steps": args.steps, "rounds": args.rounds,
            "step": {"name": "frcnn_detect_regions", "us": step_us, "batch": B, "regions_per_image": counts},
            "gpu": gpu_info()}
    print(json.dumps(line))


if __name__ == "__main__":
    sys.exit(main())
