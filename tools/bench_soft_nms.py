#!/usr/bin/env python
"""Cost of Soft-NMS (TEST.SOFT_NMS) on the bench.py workload: ResNet-101, 600x800 synthetic blobs, 300 proposals, 81 classes,
batch 4, seeded synthetic weights, device-resident input.

    python tools/bench_soft_nms.py [--batch 4] [--steps 50] [--warmup 5] [--rounds 3] [--post-iters 50]

Prints one JSON line:
  detect   images/s of the detect graph with Soft-NMS off, linear and gaussian, on the same plan and images, timed alternately
           for --rounds rounds of --steps graph replays (CUDA events; the untimed first launch after a switch rebuilds the
           post step and recaptures the graph); best round of each
  post     the post stage alone on the network's own cls_prob / pred_boxes of the timed images: frcnn_detect_post (greedy,
           TEST.NMS 0.3) against frcnn_detect_post_soft (linear, gaussian), each --post-iters back-to-back calls between CUDA
           events, at 300 RoIs per image and at 5000 (TEST.MODE top, RPN_TOP_N 5000); also the candidates per (class, image)
           and the detections kept after the cap
  gpu      card name, power limit and max SM clock read in the same run"""
import argparse
import json
import subprocess
import sys

import _init_paths  # noqa: F401
import numpy as np
import torch

from model.config import cfg
from nets.resnet_v1 import resnetv1
from tf_faster_rcnn_b200 import _native, engine, ops, synth

C, SCALES, H, W = 81, (4, 8, 16, 32), 600, 800
MODES = (("off", None), ("linear", ("linear", 0.5, 0.001)), ("gaussian", ("gaussian", 0.5, 0.001)))


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


def make_net(mode, weights):
    cfg.TEST.MODE = mode
    net = resnetv1(101)
    net.create_architecture("TEST", C, tag="default", anchor_scales=SCALES, anchor_ratios=(0.5, 1, 2))
    net.load_weights(weights)
    return net


def post_times(plan, iters):
    """Post stage alone on the plan's cls_prob / pred_boxes (left by its last detect launch): microseconds per call."""
    B, R = plan.batch, plan.R
    max_det = 256
    det, ndet = ops.zeros((B, max_det, 6)), ops.zeros((B,), dtype=torch.int32)
    keep, cnt, ks = ops.zeros((B, C, R), dtype=torch.int32), ops.zeros((B, C), dtype=torch.int32), ops.zeros((B, C, R))
    ws = ops.detect_post_workspace(R, C, B)
    t32, flags = engine.nms_threshold(0.3, True)
    nt = float(np.float32(0.3))
    calls = {"greedy": lambda: ops.detect_post(plan.cls_prob, plan.pred_boxes, plan.num_rois, C, 0.0, t32, flags, 100, det, ndet, keep, cnt,
                                               ks, ws, B)}
    for name, soft in MODES[1:]:
        code, s32, p32 = engine.soft_nms_args(*soft)
        calls[name] = (lambda code=code, s32=s32, p32=p32: ops.detect_post_soft(plan.cls_prob, plan.pred_boxes, plan.num_rois, C, 0.0, code,
                                                                                 s32, nt, p32, 100, det, ndet, keep, cnt, ks, B))
    out = {}
    for name, fn in calls.items():
        fn()
        torch.cuda.synchronize()
        kept = int(cnt.sum())                  # after the cap; the pre-cap count is not kept by the stage
        out[name] = {"us": timed_ms(fn, iters) * 1000.0 / iters, "kept_after_cap": kept}
    nr = plan.num_rois.cpu().numpy()
    prob = plan.cls_prob.view(B, R, C).cpu().numpy()
    out["candidates_per_class_image"] = float(np.mean([(prob[b, :nr[b], 1:] > 0).sum(0).mean() for b in range(B)]))
    out["rois_per_image"] = int(R)
    return out


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--post-iters", type=int, default=50)
    args = ap.parse_args(argv)
    _native.check(_native.lib().frcnn_check_device(torch.cuda.current_device()), "check_device")
    B = max(1, args.batch)
    cfg.TEST.HAS_RPN = True
    cfg.TEST.RPN_POST_NMS_TOP_N = 300
    weights = synth.make("res101", C, 3 * len(SCALES), 3)
    blobs = torch.from_numpy(np.concatenate([synth.synthetic_blob(H, W, 3 + b) for b in range(B)], axis=0))
    net = make_net("nms", weights)
    plan = net.plan_for(H, W, B)
    plan.image.copy_(blobs)

    def detect():
        plan.launch(post=True, detect=True)

    for _, soft in MODES:
        net.options["soft_nms"] = soft
        for _ in range(max(args.warmup, 1)):
            detect()
    best = {name: float("inf") for name, _ in MODES}
    for _ in range(max(args.rounds, 1)):
        for name, soft in MODES:
            net.options["soft_nms"] = soft
            detect()                                   # rebuilds the post step and recaptures the graph (untimed)
            best[name] = min(best[name], timed_ms(detect, args.steps) / args.steps)
    net.options["soft_nms"] = None
    detect()
    torch.cuda.synchronize()
    post = {"r300": post_times(plan, args.post_iters)}
    del plan, net
    torch.cuda.empty_cache()
    net5 = make_net("top", weights)
    plan5 = net5.plan_for(H, W, B)
    plan5.image.copy_(blobs)
    plan5.launch(post=True, detect=True)
    torch.cuda.synchronize()
    post["r5000"] = post_times(plan5, max(1, args.post_iters // 5))
    cfg.TEST.MODE = "nms"
    line = {"workload": "res101 %dx%d synthetic, 300 proposals, %d classes, batch %d, device-resident; Soft-NMS sigma 0.5, "
                        "prune 0.001, Nt 0.3, max_per_image 100, score thresh 0" % (H, W, C, B),
            "detect": {name: {"value": B * 1000.0 / best[name], "unit": "images/s", "ms_per_step": best[name]} for name, _ in MODES},
            "steps": args.steps, "rounds": args.rounds, "post": post, "gpu": gpu_info()}
    print(json.dumps(line))


if __name__ == "__main__":
    sys.exit(main())
