#!/usr/bin/env python
"""Cost of the per-detection features (Network.detect_features) on the bench.py workload: ResNet-101, 600x800 synthetic
blobs, 300 proposals, 81 classes, seeded synthetic weights, device-resident input.

    python tools/bench_features.py [--net res101|vgg16|mobile] [--batch 4] [--steps 50] [--warmup 5] [--rounds 3]

Prints one JSON line:
  detect / features   images/s of the detect graph and of the detect + feature-gather graph, on the same plan and images,
                      timed alternately for --rounds rounds of --steps graph replays (CUDA events); best round of each
  kernel              frcnn_detect_features alone: 20 back-to-back launches per graph replay, CUDA events; bytes counted from
                      the detections of the timed images (one fc7 row read per detection, at most max_det per image, every
                      feat_out row written, zeros past the count, + the int32 RoI indices) over kernel time, against the
                      HBM peak (MEASURED_PEAKS.json `hbm_gbs` when present, else the H100 SXM data sheet's 3.35 TB/s)
  gpu                 card name, power limit and max SM clock read in the same run"""
import argparse
import json
import os
import subprocess
import sys

import _init_paths  # noqa: F401
import numpy as np
import torch

from model.config import cfg
from nets.mobilenet_v1 import mobilenetv1
from nets.resnet_v1 import resnetv1
from nets.vgg16 import vgg16
from tf_faster_rcnn_b200 import _native, engine, synth

NETS = {"res101": (81, (4, 8, 16, 32)), "vgg16": (21, (8, 16, 32)), "mobile": (81, (4, 8, 16, 32))}
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def hbm_peak():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        with open(p) as f:
            return float(json.load(f)["hbm_gbs"]), "measured"
    return 3350.0, "H100 SXM data sheet"


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
    return e0.elapsed_time(e1)


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

    def detect():
        plan.launch(post=True, detect=True)

    def features():
        plan.launch(post=True, features=True)

    for _ in range(max(args.warmup, 1)):
        detect()
        features()
    best = {"detect": float("inf"), "features": float("inf")}
    for _ in range(max(args.rounds, 1)):
        for name, fn in (("detect", detect), ("features", features)):
            best[name] = min(best[name], timed_ms(fn, args.steps) / args.steps)
    REP, NREP = 20, 10
    g = engine.LaunchGraph([plan.features_step] * REP)
    g.replay()
    kernel_us = timed_ms(g.replay, NREP) * 1000.0 / (REP * NREP)
    max_det, fdim = plan.max_det, int(plan.feat_out.shape[2])
    rows_read = int(plan.ndet.cpu().clamp(max=max_det).sum())
    nbytes = (rows_read + B * max_det) * fdim * 4 + B * max_det * 4
    gbs = nbytes / (kernel_us * 1e-6) / 1e9
    peak, peak_src = hbm_peak()
    line = {"workload": "%s %dx%d synthetic, 300 proposals, %d classes, batch %d, device-resident" % (args.net, H, W, C, B),
            "detect": {"value": B * 1000.0 / best["detect"], "unit": "images/s", "ms_per_step": best["detect"]},
            "features": {"value": B * 1000.0 / best["features"], "unit": "images/s", "ms_per_step": best["features"],
                         "api": "Network.detect_features: detect + head feature / RoI index of every detection, one graph replay"},
            "steps": args.steps, "rounds": args.rounds,
            "kernel": {"name": "detect_features_kernel", "us": kernel_us, "feature_dim": fdim, "max_det": max_det,
                       "detections": rows_read, "bytes": nbytes, "achieved_gbs": gbs, "peak_gbs": peak, "peak_source": peak_src,
                       "frac": gbs / peak},
            "gpu": gpu_info()}
    print(json.dumps(line))


if __name__ == "__main__":
    sys.exit(main())
