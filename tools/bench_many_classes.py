#!/usr/bin/env python
"""Cost of large class counts on the bottom-up-attention layout: ResNet-101, 600x800 synthetic blobs, batch 4, 300 proposals,
12 anchors (ANCHOR_SCALES 4, 8, 16, 32), seeded synthetic weights, device-resident input, at C = 81, 1024, 1025, 1204 and 1601.

    python tools/bench_many_classes.py [--batch 4] [--steps 20] [--warmup 3] [--rounds 3] [--classes 81,1024,1025,1204,1601]

C = 81 is the COCO model, 1204 LVIS, 1601 Visual Genome.  1024 and 1025 sit on either side of frcnn_detect_regions' switch from the
per-class NMS path to the overlap-mask path, so the two implementations of its step 2 are compared at almost the same C.

Prints one JSON line; per C:
  detect / regions    images/s of the detect graph (network + box decode + per-class NMS + cap + records) and of the regions graph
                      (network + the regions step), timed in alternation over every C for --rounds rounds of --steps graph replays
                      (CUDA events); best round of each
  post_us / step_us   the post step (frcnn_detect_post) and the regions step (frcnn_detect_regions) alone: 20 back-to-back steps per
                      graph replay, CUDA events, per batch
  gpu                 card name, power limit and max SM clock read in the same run"""
import argparse
import json
import sys

import _init_paths  # noqa: F401
import numpy as np
import torch

from bench_features import gpu_info, timed_ms
from model.config import cfg
from nets.resnet_v1 import resnetv1
from tf_faster_rcnn_b200 import _native, engine, ops, synth

SCALES = (4, 8, 16, 32)


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--classes", default="81,1024,1025,1204,1601")
    args = ap.parse_args(argv)
    _native.check(_native.lib().frcnn_check_device(torch.cuda.current_device()), "check_device")
    classes = [int(c) for c in args.classes.split(",")]
    H, W, B = 600, 800, max(1, args.batch)
    cfg.TEST.HAS_RPN = True
    cfg.TEST.RPN_POST_NMS_TOP_N = 300
    cfg.USE_GPU_NMS = False
    blobs = torch.from_numpy(np.concatenate([synth.synthetic_blob(H, W, 3 + b) for b in range(B)], axis=0))
    reg = engine.region_args(0.2, 10, 100)
    plans = {}
    for C in classes:
        net = resnetv1(101)
        net.create_architecture("TEST", C, tag="default", anchor_scales=SCALES, anchor_ratios=(0.5, 1, 2))
        net.load_weights(synth.make("res101", C, 3 * len(SCALES), 3))
        plan = net.plan_for(H, W, B)
        plan.image.copy_(blobs)
        plans[C] = (net, plan)

    def fns(plan):
        return {"detect": lambda: plan.launch(post=True, detect=True), "regions": lambda: plan.launch(regions=reg)}

    for _ in range(max(args.warmup, 1)):
        for C in classes:
            for fn in fns(plans[C][1]).values():
                fn()
    best = {C: {"detect": float("inf"), "regions": float("inf")} for C in classes}
    for _ in range(max(args.rounds, 1)):
        for C in classes:
            for name, fn in fns(plans[C][1]).items():
                best[C][name] = min(best[C][name], timed_ms(fn, args.steps) / args.steps)
    REP, NREP = 20, 10
    out = {}
    for C in classes:
        plan = plans[C][1]
        steps = {}
        for name, step in (("post_us", plan.post_steps[plan.slot]), ("step_us", plan.regions_step)):
            g = engine.LaunchGraph([step] * REP)
            g.replay()
            steps[name] = timed_ms(g.replay, NREP) * 1000.0 / (REP * NREP)
        out[str(C)] = {"detect": {"value": B * 1000.0 / best[C]["detect"], "unit": "images/s", "ms_per_step": best[C]["detect"]},
                       "regions": {"value": B * 1000.0 / best[C]["regions"], "unit": "images/s", "ms_per_step": best[C]["regions"]},
                       "post_us": steps["post_us"], "step_us": steps["step_us"],
                       "regions_path": "per-class NMS" if C <= ops.REGIONS_CLASS_NMS_MAX else "overlap mask",
                       "detections": [int(n) for n in plan.ndet.cpu().tolist()],
                       "regions_per_image": plan.reg_out["count"].cpu().tolist()}
    line = {"workload": "res101 %dx%d synthetic, 300 proposals, 12 anchors, batch %d, device-resident" % (H, W, B),
            "steps": args.steps, "rounds": args.rounds, "classes": out, "gpu": gpu_info()}
    print(json.dumps(line))


if __name__ == "__main__":
    sys.exit(main())
