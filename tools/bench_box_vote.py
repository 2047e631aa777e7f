#!/usr/bin/env python
"""Cost of box voting (TEST.BBOX_VOTE) on the bench.py workload: ResNet-101, 600x800 synthetic blobs, 81 classes, batch 4,
seeded synthetic weights, device-resident input.

    python tools/bench_box_vote.py [--batch 4] [--steps 50] [--warmup 5] [--rounds 3] [--post-iters 50]

Prints one JSON line:
  post     the post stage alone on the network's own cls_prob / pred_boxes: greedy (TEST.NMS 0.3) and Soft-NMS (linear), each
           without voting, with ID and with AVG (VOTE_TH 0.8), --post-iters back-to-back calls between CUDA events, at 300 RoIs
           per image and at 5000 (TEST.MODE top, RPN_TOP_N 5000); also the detections kept after the cap
  detect   images/s of the detect graph (300 proposals) with voting off and on (ID, AVG), on the same plan and images, timed
           alternately for --rounds rounds of --steps graph replays; best round of each
  gpu      card name, power limit and max SM clock read in the same run"""
import argparse
import json
import sys

import _init_paths  # noqa: F401
import numpy as np
import torch

from bench_soft_nms import gpu_info, make_net, timed_ms
from model.config import cfg
from tf_faster_rcnn_b200 import _native, engine, ops, synth

C, SCALES, H, W = 81, (4, 8, 16, 32), 600, 800
VOTES = (("off", None), ("ID", (0.8, "ID", 1.0)), ("AVG", (0.8, "AVG", 1.0)))


def post_times(plan, iters):
    """Post stage alone on the plan's cls_prob / pred_boxes (left by its last detect launch): microseconds per call."""
    B, R = plan.batch, plan.R
    max_det = 256
    det, ndet = ops.zeros((B, max_det, 6)), ops.zeros((B,), dtype=torch.int32)
    keep, cnt, ks = ops.zeros((B, C, R), dtype=torch.int32), ops.zeros((B, C), dtype=torch.int32), ops.zeros((B, C, R))
    vb = ops.zeros((B, C, R, 4))
    ws = ops.detect_post_workspace(R, C, B)
    t32, flags = engine.nms_threshold(0.3, True)
    nt = float(np.float32(0.3))
    code, s32, p32 = engine.soft_nms_args("linear", 0.5, 0.001)
    out = {}
    for vname, vote in VOTES:
        v = None if vote is None else (*engine.box_vote_args(*vote), vb)
        calls = {"greedy": lambda v=v: ops.detect_post(plan.cls_prob, plan.pred_boxes, plan.num_rois, C, 0.0, t32, flags, 100, det, ndet,
                                                       keep, cnt, ks, ws, B, vote=v),
                 "soft_linear": lambda v=v: ops.detect_post_soft(plan.cls_prob, plan.pred_boxes, plan.num_rois, C, 0.0, code, s32, nt, p32,
                                                                 100, det, ndet, keep, cnt, ks, B, vote=v)}
        for name, fn in calls.items():
            fn()
            torch.cuda.synchronize()
            out["%s/%s" % (name, vname)] = {"us": timed_ms(fn, iters) * 1000.0 / iters, "kept_after_cap": int(cnt.sum())}
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

    for _, vote in VOTES:
        net.options["box_vote"] = vote
        for _ in range(max(args.warmup, 1)):
            detect()
    best = {name: float("inf") for name, _ in VOTES}
    for _ in range(max(args.rounds, 1)):
        for name, vote in VOTES:
            net.options["box_vote"] = vote
            detect()                                   # rebuilds the post step and recaptures the graph (untimed)
            best[name] = min(best[name], timed_ms(detect, args.steps) / args.steps)
    net.options["box_vote"] = None
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
    post["r5000"] = post_times(plan5, max(1, args.post_iters // 10))
    cfg.TEST.MODE = "nms"
    line = {"workload": "res101 %dx%d synthetic, %d classes, batch %d, device-resident; NMS 0.3, Soft-NMS linear sigma 0.5 prune "
                        "0.001, VOTE_TH 0.8, max_per_image 100, score thresh 0" % (H, W, C, B),
            "detect": {name: {"value": B * 1000.0 / best[name], "unit": "images/s", "ms_per_step": best[name]} for name, _ in VOTES},
            "steps": args.steps, "rounds": args.rounds, "post": post, "gpu": gpu_info()}
    print(json.dumps(line))


if __name__ == "__main__":
    sys.exit(main())
