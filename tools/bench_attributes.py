#!/usr/bin/env python
"""Cost of the attribute head (cfg.ATTRIBUTES) on the bottom-up regions graph: ResNet-101, 600x800 synthetic blobs, batch 4,
300 proposals, 12 anchors, seeded synthetic weights, device-resident input, at (81 classes, 401 attributes) and (1601, 401).

    python tools/bench_attributes.py [--batch 4] [--steps 50] [--warmup 5] [--rounds 5] [--classes 81 1601]

Per class count, two networks load the same seeded weights, one with the head off and one with it on (EMBED_DIM 256, HIDDEN
512), and their regions graphs (Network.detect_regions, 10-100 regions per image) are timed in alternating rounds of --steps
graph replays (CUDA events); the best round of each is reported.  The head's four launches (frcnn_regions_attr_embed, the
fc_attr and attr_score FCs, frcnn_attr_finish) are also timed alone: 20 back-to-back copies per graph replay.  Prints one JSON
line per class count, with the card name, power limit and max SM clock read in the same run."""
import argparse
import json
import sys

import _init_paths  # noqa: F401
import numpy as np
import torch

from bench_features import gpu_info, timed_ms
from model.config import cfg
from nets.resnet_v1 import resnetv1
from tf_faster_rcnn_b200 import _native, engine, synth

SCALES = (4, 8, 16, 32)
ATTRS = (401, 256, 512)


def build(C, attributes, weights):
    old = dict(cfg.ATTRIBUTES)
    cfg.ATTRIBUTES.NUM_CLASSES = attributes[0] if attributes else 0
    try:
        net = resnetv1(num_layers=101)
        net.create_architecture("TEST", C, tag="default", anchor_scales=SCALES, anchor_ratios=(0.5, 1, 2))
    finally:
        cfg.ATTRIBUTES.update(old)
    net.load_weights(weights)
    return net


def head_flops(rows, F, attributes):
    A, E, H = attributes
    return 2.0 * rows * ((F + E) * H + H * A)


def run(C, args):
    H, W, B = 600, 800, max(1, args.batch)
    weights = synth.make("res101", C, 3 * len(SCALES), 3, attributes=ATTRS)
    nets = {"off": build(C, None, weights), "on": build(C, ATTRS, weights)}
    blobs = torch.from_numpy(np.concatenate([synth.synthetic_blob(H, W, 3 + b) for b in range(B)], axis=0))
    reg = engine.region_args(0.2, 10, 100)
    plans = {}
    for k, net in nets.items():
        plans[k] = net.plan_for(H, W, B)
        plans[k].image.copy_(blobs)
    fns = {k: (lambda p=p: p.launch(regions=reg)) for k, p in plans.items()}
    for _ in range(max(args.warmup, 1)):
        for fn in fns.values():
            fn()
    torch.cuda.synchronize()
    same = all(plans["off"].reg_out[k].cpu().numpy().tobytes() == plans["on"].reg_out[k].cpu().numpy().tobytes()
               for k in engine.REGION_FIELDS + ("count",))
    best = {k: float("inf") for k in fns}
    for _ in range(max(args.rounds, 1)):
        for k, fn in fns.items():
            best[k] = min(best[k], timed_ms(fn, args.steps) / args.steps)
    REP, NREP = 20, 10
    on = plans["on"]
    g = engine.LaunchGraph(on.attr_steps * REP)
    g.replay()
    head_us = timed_ms(g.replay, NREP) * 1000.0 / (REP * NREP)
    M = on.reg_out["conf"].shape[1]
    F = int(on.fc7.shape[1])
    line = {"workload": "res101 %dx%d synthetic, 300 proposals, %d classes, %d attributes, batch %d, device-resident"
                        % (H, W, C, ATTRS[0], B),
            "regions_off": {"ms_per_step": best["off"], "images_per_s": B * 1000.0 / best["off"]},
            "regions_on": {"ms_per_step": best["on"], "images_per_s": B * 1000.0 / best["on"]},
            "head_share": (best["on"] - best["off"]) / best["off"],
            "head_launches": {"us": head_us, "rows": B * M, "gflop": head_flops(B * M, F, ATTRS) / 1e9,
                              "tflops": head_flops(B * M, F, ATTRS) / (head_us * 1e-6) / 1e12},
            "region_fields_identical": same, "counts": on.reg_out["count"].cpu().tolist(),
            "steps": args.steps, "rounds": args.rounds, "gpu": gpu_info()}
    print(json.dumps(line), flush=True)
    for net in nets.values():
        for p in net._plans.values():
            p.release()
        net._plans.clear()
    torch.cuda.empty_cache()


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--classes", type=int, nargs="+", default=[81, 1601])
    args = ap.parse_args(argv)
    _native.check(_native.lib().frcnn_check_device(torch.cuda.current_device()), "check_device")
    cfg.TEST.HAS_RPN = True
    cfg.TEST.RPN_POST_NMS_TOP_N = 300
    cfg.USE_GPU_NMS = False
    for C in args.classes:
        run(C, args)


if __name__ == "__main__":
    sys.exit(main())
