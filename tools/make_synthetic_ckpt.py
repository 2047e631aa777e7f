#!/usr/bin/env python
"""Writes a seeded synthetic checkpoint of TF-named variables -- `--format bundle`: a TensorFlow V2 checkpoint
(<out>.index + <out>.data-00000-of-00001); `--format npz`: <out>.npz -- plus an empty <out>.meta so that the reference's
demo.py existence check passes.  python tools/make_synthetic_ckpt.py --net res101 --classes 21 --anchors 9 --out /tmp/x.ckpt
--attributes A (with --attr_embed E, --attr_hidden H) also writes the attribute head's variables (cfg.ATTRIBUTES)."""
import argparse
import _init_paths  # noqa: F401
import numpy as np
from tf_faster_rcnn_b200 import checkpoint, engine, synth

ap = argparse.ArgumentParser()
ap.add_argument("--net", default="res101")
ap.add_argument("--classes", type=int, default=21)
ap.add_argument("--anchors", type=int, default=9)
ap.add_argument("--out", required=True)
ap.add_argument("--format", choices=("npz", "bundle"), default="npz")
ap.add_argument("--attributes", type=int, default=0, help="attribute classes of the attribute head (0: none; Visual Genome: 401)")
ap.add_argument("--attr_embed", type=int, default=256, help="ATTRIBUTES.EMBED_DIM")
ap.add_argument("--attr_hidden", type=int, default=512, help="ATTRIBUTES.HIDDEN")
a = ap.parse_args()
attributes = engine.attributes_option(dict(NUM_CLASSES=a.attributes, EMBED_DIM=a.attr_embed, HIDDEN=a.attr_hidden))
tensors = synth.make(a.net, a.classes, a.anchors, attributes=attributes)
if a.format == "bundle":
    checkpoint.write_bundle(a.out, tensors)
else:
    np.savez(a.out + ".npz", **tensors)
open(a.out + ".meta", "w").close()
print("wrote", a.out + (".index / .data-00000-of-00001" if a.format == "bundle" else ".npz"))
