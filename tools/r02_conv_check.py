"""Development check of the dense kernels on a GPU: correctness vs float64 and speed of FP16x3 vs TF32x3.

    FRCNN_LIB_VARIANT=wd python tools/r02_conv_check.py [quick|full]

With the watchdog library a barrier-protocol deadlock aborts the kernel and prints who waited on what instead of hanging.
It prints numbers and asserts nothing.  Its range cases (tiny and large weights, the tf32 mode) are asserted element by
element in tests/test_conv_gpu.py (weight channel spread, layer scale, activation scale sweep).
"""
import ctypes as C
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from tf_faster_rcnn_b200 import ops, _native as N  # noqa: E402

F = np.float32
TAGS = {1: "consumer:full", 4: "producer:empty"}


def watchdog(reset=True):
    out = (C.c_uint * 16)()
    N.check(N.lib().frcnn_debug_watchdog(out, int(reset)), "debug_watchdog")
    v = list(out)
    if v[15] == 0xffffffff:
        return None
    if v[0]:
        return "ABORTED: %d waits timed out; first: block %d thread %d (warp %d) wait %s parity %d aux %d" % (
            v[1], v[2], v[3], v[3] // 32, TAGS.get(v[4], v[4]), v[5], v[6])
    return ""


def ref64(x, w, stride, pt, pl, ho, wo):
    xt = torch.from_numpy(x.astype(np.float64)).permute(0, 3, 1, 2)
    wt = torch.from_numpy(w.astype(np.float64)).permute(3, 2, 0, 1)
    kh, kw = w.shape[:2]
    h, wd = x.shape[1:3]
    pb = max((ho - 1) * stride + kh - h - pt, 0)
    pr = max((wo - 1) * stride + kw - wd - pl, 0)
    xt = torch.nn.functional.pad(xt, (pl, pr, pt, pb))
    return torch.nn.functional.conv2d(xt, wt, None, stride=stride).permute(0, 2, 3, 1).numpy()[:, :ho, :wo]


def one(name, n, h, w, cin, cout, k, impl, kpc=0, bn=0, check=True, reps=20, stride=1, relu_in=True, wscale=None, split_k=0):
    rng = np.random.default_rng(abs(hash(name)) % (2 ** 31))
    x = rng.standard_normal((n, h, w, cin)).astype(F)
    if relu_in:
        x = np.maximum(x, 0)
    ws = np.sqrt(2.0 / (k * k * cin)) if wscale is None else wscale
    wt = (rng.standard_normal((k, k, cin, cout)) * ws).astype(F)
    ho, wo, pt, pl = ops.conv_out_hw(h, w, k, stride, "SAME")
    pc = ops.PackedConv(wt, impl=impl)
    xd = torch.from_numpy(x).cuda()
    out = torch.full((n, ho, wo, cout), float("nan"), dtype=torch.float32, device="cuda")
    plan = ops.ConvPlan(xd, pc, out, stride, pt, pl, 0, None, bn, kpc, split_k)
    plan.run()
    torch.cuda.synchronize()
    wd = watchdog()
    info = plan.info()
    msg = "[%s] impl=%s kpc=%d bn=%d grid=%dx%d splits=%d" % (name, "f16" if impl == 0 else "tf32", kpc, info["block_n"], info["grid_m"],
                                                          info["grid_n"], info["splits"])
    if wd:
        print(msg, wd, flush=True)
        return False
    if check:
        got = out.cpu().numpy()
        want = ref64(x, wt, stride, pt, pl, ho, wo)
        sc = np.abs(want).max()
        nan = int(np.isnan(got).sum())
        err = np.nanmax(np.abs(got - want)) / sc
        msg += " err_vs_f64=%.2e nan=%d" % (err, nan)
    for _ in range(3):
        plan.run()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        plan.run()
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1000 / reps
    fl = 2.0 * n * ho * wo * cout * k * k * cin
    msg += "  %.1f us  %.1f TFLOP/s" % (us, fl / us / 1e6)
    wd = watchdog()
    if wd:
        msg += " " + wd
    print(msg, flush=True)
    return True


def main():
    mode = sys.argv[1] if len(sys.argv) > 1 else "quick"
    if mode == "ncu":
        one("res_head_c3", 300, 7, 7, 512, 512, 3, impl=0, kpc=4, check=False, reps=2)
        one("res_head_pw512_2048", 300, 7, 7, 512, 2048, 1, impl=0, kpc=4, check=False, reps=2)
        one("res_head_pw1024_2048", 300, 7, 7, 1024, 2048, 1, impl=0, kpc=4, check=False, reps=2)
        one("res_b3_pw1024_256", 1, 38, 50, 1024, 256, 1, impl=0, kpc=4, check=False, reps=2)
        return one("res_b3_c3_256", 1, 38, 50, 256, 256, 3, impl=0, kpc=4, check=False, reps=2)
    print("lib:", N.LIB_PATH, "watchdog:", watchdog() is not None, flush=True)
    t0 = time.time()
    # ---- correctness first, smallest first ----------------------------------------------------------------------------
    small = [("fc_small", 1, 1, 300, 64, 64, 1), ("pw_1900", 1, 38, 50, 256, 256, 1), ("c3_64", 1, 38, 50, 64, 64, 3),
             ("c3_odd_cout", 1, 20, 30, 128, 96, 3), ("rois_c3", 20, 7, 7, 64, 64, 3), ("rpn_cout72", 1, 38, 50, 512, 72, 1),
             ("fc_k3136", 1, 1, 300, 3136, 128, 1), ("pw_cin32", 1, 38, 50, 32, 64, 1), ("c3_cin96", 1, 20, 30, 96, 64, 3)]
    ok = True
    for s in small:
        ok = one(*s, impl=0) and ok
        if not ok:
            print("stopping: watchdog abort", flush=True)
            return
    one("c3_64", 1, 38, 50, 64, 64, 3, impl=1)
    # range robustness: tiny weights / large weights / large activations
    one("pw_tinyw", 1, 38, 50, 256, 256, 1, impl=0, wscale=1e-6)
    one("pw_bigw", 1, 38, 50, 256, 256, 1, impl=0, wscale=300.0)
    # ---- speed + accuracy on the shapes that matter ----------------------------------------------------------------------
    big = [("res_head_c3", 300, 7, 7, 512, 512, 3), ("res_head_pw2048_512", 300, 7, 7, 2048, 512, 1), ("res_head_pw512_2048", 300, 7, 7, 512, 2048, 1),
           ("res_head_pw1024_2048", 300, 7, 7, 1024, 2048, 1), ("res_b3_pw1024_256", 1, 38, 50, 1024, 256, 1), ("res_b3_c3_256", 1, 38, 50, 256, 256, 3),
           ("res_b3_pw256_1024", 1, 38, 50, 256, 1024, 1), ("vgg_conv3", 1, 150, 200, 256, 256, 3), ("vgg_conv5", 1, 38, 50, 512, 512, 3),
           ("res_b1_pw64_256", 1, 150, 200, 64, 256, 1), ("res_b2_c3_128", 1, 75, 100, 128, 128, 3)]
    for s in big:
        chk = mode == "full" or s[0] in ("res_head_c3", "res_b3_pw1024_256")
        for kpc in ((2, 4, 8) if s[0] in ("res_head_c3", "res_head_pw2048_512") else (4,)):
            one(*s, impl=0, kpc=kpc, check=chk)
        one(*s, impl=1, kpc=8, check=False)
        if time.time() - t0 > 420:
            print("time budget reached", flush=True)
            break


if __name__ == "__main__":
    main()
