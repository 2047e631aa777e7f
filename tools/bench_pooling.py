#!/usr/bin/env python
"""Cost of the RoI pooling modes (POOLING_MODE crop / align / pool) at 600x800, batch 4, 300 proposals per image, 81 classes,
seeded synthetic weights and blobs.

    python tools/bench_pooling.py [--batch 4] [--steps 30] [--warmup 5] [--rounds 3] [--iters 200]

Prints one JSON line:
  kernel   the pooling launch alone, per mode (crop, align with SAMPLING_RATIO 0 and 2, pool), on the ResNet-101 (C = 1024) and
           VGG16 (C = 512) networks' own feature maps and RPN RoIs: --iters back-to-back launches between CUDA events, after
           warm-up; with the samples (bilinear taps of 4 cells) or max-pool cells per launch and the bytes they gather, counted
           from the shapes and RoIs on the host
  detect   images/s of the ResNet-101 detect graph per mode, one network per mode, the modes timed alternately for --rounds
           rounds of --steps graph replays; best round of each
  gpu      card name, power limit and max SM clock read in the same run"""
import argparse
import json
import math
import sys

import _init_paths  # noqa: F401
import numpy as np
import torch

from bench_soft_nms import gpu_info, timed_ms
from model.config import cfg
from nets.resnet_v1 import resnetv1
from nets.vgg16 import vgg16
from tf_faster_rcnn_b200 import _native, engine, ops, synth

C, SCALES, H, W, P = 81, (4, 8, 16, 32), 600, 800, 7
MODES = (("crop", 0), ("align_sr0", 0), ("align_sr2", 2), ("pool", 0))
F = np.float32


def make_net(arch, weights, mode, sr):
    cfg.POOLING_MODE = mode.split("_")[0]
    cfg.ROI_ALIGN.update(SAMPLING_RATIO=sr, ALIGNED=False)
    net = vgg16() if arch == "vgg16" else resnetv1(101)
    net.create_architecture("TEST", C, tag="default", anchor_scales=SCALES, anchor_ratios=(0.5, 1, 2))
    net.load_weights(weights)
    return net


def work(mode, sr, rois, fh, fw, c, pre_pool):
    """(samples or cells per launch, bytes gathered from the map, bytes written) from the shapes and the RoIs."""
    r = rois.shape[0]
    written = r * P * P * c * 4
    if mode == "crop":
        s = int(r * P * P * (4 if pre_pool else 1))
        return s, s * 4 * c * 4, written
    s16 = F(1.0 / 16)
    if mode.startswith("align"):
        rw = np.maximum((rois[:, 3] * s16 - rois[:, 1] * s16).astype(F), F(1))
        rh = np.maximum((rois[:, 4] * s16 - rois[:, 2] * s16).astype(F), F(1))
        g = (np.full(r, sr * sr) if sr else np.ceil(rh / F(P)) * np.ceil(rw / F(P))).astype(np.int64)
        s = int(g.sum()) * P * P
        return s, s * 4 * c * 4, written
    rnd = lambda v: (np.sign(v) * np.floor(np.abs(v.astype(np.float64)) + 0.5)).astype(np.int64)   # noqa: E731
    x1, y1, x2, y2 = (rnd((rois[:, k] * s16).astype(F)) for k in (1, 2, 3, 4))
    cells = 0
    for k in range(r):
        bh, bw = F(max(y2[k] - y1[k] + 1, 1)) / F(P), F(max(x2[k] - x1[k] + 1, 1)) / F(P)
        rows = [min(max(math.ceil(F(p + 1) * bh) + y1[k], 0), fh) - min(max(math.floor(F(p) * bh) + y1[k], 0), fh) for p in range(P)]
        cols = [min(max(math.ceil(F(p + 1) * bw) + x1[k], 0), fw) - min(max(math.floor(F(p) * bw) + x1[k], 0), fw) for p in range(P)]
        cells += sum(max(a, 0) for a in rows) * sum(max(b, 0) for b in cols)
    cells = int(cells)
    return cells, cells * c * 4, written


def kernel_times(arch, weights, blobs, iters):
    net = make_net(arch, weights, "crop", 0)
    plan = net.plan_for(H, W, blobs.shape[0])
    plan.image.copy_(blobs)
    plan.launch(post=True, detect=True)
    torch.cuda.synchronize()
    feat, rois = plan.feat, plan.rois
    _, fh, fw, c = feat.shape
    out = torch.empty((rois.shape[0], P, P, c), device="cuda")
    pre_pool = net.crop_pre_pool()
    host_rois = rois.cpu().numpy()
    calls = {"crop": lambda: ops.crop_pool(feat, rois, P, pre_pool, out),
             "align_sr0": lambda: ops.roi_align(feat, rois, P, engine.SPATIAL_SCALE, 0, False, out),
             "align_sr2": lambda: ops.roi_align(feat, rois, P, engine.SPATIAL_SCALE, 2, False, out),
             "pool": lambda: ops.roi_pool(feat, rois, P, engine.SPATIAL_SCALE, out)}
    res = {}
    for name, sr in MODES:
        for _ in range(20):
            calls[name]()
        us = timed_ms(calls[name], iters) * 1000.0 / iters
        s, gathered, written = work(name, sr, host_rois, fh, fw, c, pre_pool)
        res[name] = {"us": us, "samples_or_cells": s, "gather_bytes": gathered, "write_bytes": written,
                     "gather_GB_per_s": gathered / us / 1e3}
    res["shape"] = {"feature_map": [int(x) for x in feat.shape], "rois": int(rois.shape[0]), "pooled": P,
                    "crop_pre_pool": bool(pre_pool)}
    del plan, net
    torch.cuda.empty_cache()
    return res


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=200)
    args = ap.parse_args(argv)
    _native.check(_native.lib().frcnn_check_device(torch.cuda.current_device()), "check_device")
    B = max(1, args.batch)
    cfg.TEST.HAS_RPN = True
    cfg.TEST.RPN_POST_NMS_TOP_N = 300
    saved = (cfg.POOLING_MODE, dict(cfg.ROI_ALIGN))
    blobs = torch.from_numpy(np.concatenate([synth.synthetic_blob(H, W, 3 + b) for b in range(B)], axis=0))
    try:
        kernel = {}
        for arch in ("res101", "vgg16"):
            kernel[arch] = kernel_times(arch, synth.make(arch, C, 3 * len(SCALES), 3), blobs, args.iters)
        weights = synth.make("res101", C, 3 * len(SCALES), 3)
        plans = {}
        for name, sr in MODES:
            plan = make_net("res101", weights, name, sr).plan_for(H, W, B)
            plan.image.copy_(blobs)
            plans[name] = plan
            for _ in range(max(args.warmup, 1)):
                plan.launch(post=True, detect=True)
        best = {name: float("inf") for name, _ in MODES}
        for _ in range(max(args.rounds, 1)):
            for name, _ in MODES:
                fn = lambda p=plans[name]: p.launch(post=True, detect=True)   # noqa: E731
                best[name] = min(best[name], timed_ms(fn, args.steps) / args.steps)
    finally:
        cfg.POOLING_MODE = saved[0]
        cfg.ROI_ALIGN.update(saved[1])
    line = {"workload": "%dx%d synthetic, %d classes, batch %d, %d proposals per image, POOLING_SIZE %d, device-resident"
                        % (H, W, C, B, 300, P),
            "kernel": kernel,
            "detect_res101": {name: {"value": B * 1000.0 / best[name], "unit": "images/s", "ms_per_step": best[name]} for name, _ in MODES},
            "steps": args.steps, "rounds": args.rounds, "gpu": gpu_info()}
    print(json.dumps(line))


if __name__ == "__main__":
    sys.exit(main())
