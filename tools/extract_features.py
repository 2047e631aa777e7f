#!/usr/bin/env python
"""Region features ("bottom-up" features for captioning / VQA / grounding): one .npz per image of an imdb.

    python tools/extract_features.py --imdb voc_2007_test --net res101 --model ckpt --out DIR [--batch B] [--boxes FILE.pkl]
    python tools/extract_features.py ... --regions [--conf_thresh 0.2 --min_boxes 10 --max_boxes 100] [--tsv FILE.tsv]

Without --boxes, each file holds the detector's final detections (per-class NMS + max_per_image cap, as test_net) and the
head feature of the RoI each came from (2048-d ResNet, 4096-d VGG16, 1024-d MobileNet):
    boxes [n,4] fp32 (x1,y1,x2,y2, image pixels), scores [n] fp32, classes [n] int32, features [n,F] fp32,
    roi_index [n] int32 (RoI row within the image), image_h, image_w.
With --boxes FILE.pkl (a dict image index -> [n,4] boxes in image pixels, or a list in imdb order), the given boxes are
scored instead of RPN proposals (the Fast R-CNN mode):
    boxes [n,4], scores [n,C] fp32 (class probabilities), features [n,F], image_h, image_w.
With --regions, the bottom-up-attention protocol (Anderson et al. 2018, Network.detect_regions): distinct RoIs ranked by
their best class confidence after per-class NMS, 10-100 per image by default, with unregressed boxes:
    boxes [n,4] fp32, features [n,F] fp32, conf [n] fp32, classes [n] int32, roi_index [n] int32, image_h, image_w, num_boxes;
--tsv FILE also writes the protocol's TSV (image_id, image_w, image_h, num_boxes, boxes, features; the arrays as base64 of
their float32 bytes), one row per image.  --regions and --boxes exclude each other.
With the attribute head on (--set ATTRIBUTES.NUM_CLASSES 401), each --regions file also holds attr_prob [n,A] fp32, attributes
[n] int32 and attr_conf [n] fp32, and the TSV gains the columns attrs_id (base64 of the int32 attributes) and attrs_conf
(base64 of the float32 attr_conf) after the existing ones.
Consecutive images whose blobs have the same shape are run together, up to --batch per device launch.  Without --model
the network gets seeded synthetic weights."""
import argparse
import base64
import csv
import os
import pickle
import sys

import _init_paths  # noqa: F401
import cv2
import numpy as np

from datasets.factory import get_imdb
from model.config import cfg_from_file, cfg_from_list
from model.test import _get_blobs, _set_post_options
from tools_common import build_net


def parse_args(argv=None):
    p = argparse.ArgumentParser(description="Per-region head features of a Faster R-CNN network on the H100 path")
    p.add_argument("--imdb", dest="imdb_name", required=True)
    p.add_argument("--net", default="res101", help="vgg16, res50, res101, res152, mobile")
    p.add_argument("--model", default=None, help="TF checkpoint or .npz (default: seeded synthetic weights)")
    p.add_argument("--batch", type=int, default=1, help="images per device launch (consecutive images of one blob shape)")
    mode = p.add_mutually_exclusive_group()
    mode.add_argument("--boxes", default=None, help="pickle of caller boxes per image: score these instead of detecting")
    mode.add_argument("--regions", action="store_true", help="bottom-up regions (the bottom-up-attention protocol)")
    p.add_argument("--conf_thresh", type=float, default=0.2, help="--regions: confidence threshold")
    p.add_argument("--min_boxes", type=int, default=10, help="--regions: fewest regions per image")
    p.add_argument("--max_boxes", type=int, default=100, help="--regions: most regions per image")
    p.add_argument("--tsv", default=None, help="--regions: also write the protocol's TSV file")
    p.add_argument("--num_dets", dest="max_per_image", type=int, default=100)
    p.add_argument("--out", required=True)
    p.add_argument("--cfg", dest="cfg_file", default=None)
    p.add_argument("--set", dest="set_cfgs", default=None, nargs=argparse.REMAINDER)
    return p.parse_args(argv)


def image_boxes(boxes, imdb, i):
    if isinstance(boxes, dict):
        key = imdb.image_index[i]
        b = boxes[key] if key in boxes else boxes[i]
    else:
        b = boxes[i]
    return np.asarray(b, dtype=np.float32).reshape(-1, 4)


TSV_FIELDS = ["image_id", "image_w", "image_h", "num_boxes", "boxes", "features"]
TSV_ATTR_FIELDS = ["attrs_id", "attrs_conf"]       # appended with the attribute head on
csv.field_size_limit(2 ** 31 - 1)


def _b64(a, dtype=np.float32):
    return base64.b64encode(np.ascontiguousarray(a, dtype=dtype).tobytes()).decode("ascii")


def tsv_row(image_id, image_h, image_w, boxes, features, attributes=None, attr_conf=None):
    """One row of the bottom-up-attention TSV: the arrays as base64 of their float32 bytes (row-major); with the attribute head
    also attrs_id (int32 bytes) and attrs_conf (float32 bytes)."""
    row = {"image_id": image_id, "image_w": int(image_w), "image_h": int(image_h), "num_boxes": int(boxes.shape[0]),
           "boxes": _b64(boxes), "features": _b64(features)}
    if attributes is not None:
        row.update(attrs_id=_b64(attributes, np.int32), attrs_conf=_b64(attr_conf))
    return row


def tsv_writer(f, attributes=False):
    return csv.DictWriter(f, delimiter="\t", fieldnames=TSV_FIELDS + (TSV_ATTR_FIELDS if attributes else []))


def extract(net, imdb, out_dir, batch=1, boxes=None, max_per_image=100, regions=None, tsv=None):
    """Writes <out_dir>/<image index>.npz for every image of `imdb`; returns the number of files written.  regions: None, or
    (conf_thresh, min_boxes, max_boxes) for the bottom-up regions; tsv: None, or a csv.DictWriter (tsv_writer) for their rows."""
    _set_post_options(net, 0.0, max_per_image)
    os.makedirs(out_dir, exist_ok=True)
    group = []                                   # (image number, blob, scale, (h, w))

    def flush():
        blobs = np.concatenate([g[1] for g in group], axis=0)
        scales, hws = [g[2] for g in group], [g[3] for g in group]
        if regions is not None:
            res, _ = net.detect_regions(blobs, scales, hws, *regions)
            for (i, _, _, hw), reg in zip(group, res):
                np.savez(os.path.join(out_dir, "%s.npz" % imdb.image_index[i]), image_h=hw[0], image_w=hw[1],
                         num_boxes=reg["boxes"].shape[0], **reg)
                if tsv is not None:
                    tsv.writerow(tsv_row(imdb.image_index[i], hw[0], hw[1], reg["boxes"], reg["features"], reg.get("attributes"),
                                         reg.get("attr_conf")))
        elif boxes is None:
            res, _ = net.detect_features(blobs, scales, hws)
            for (i, _, _, hw), (det, feats, roi) in zip(group, res):
                np.savez(os.path.join(out_dir, "%s.npz" % imdb.image_index[i]), boxes=det[:, :4], scores=det[:, 4],
                         classes=det[:, 5].astype(np.int32), features=feats, roi_index=roi, image_h=hw[0], image_w=hw[1])
        else:
            given = [image_boxes(boxes, imdb, g[0]) for g in group]
            res, _ = net.score_boxes(blobs, scales, hws, given)
            for (i, _, _, hw), bx, (scores, _, feats) in zip(group, given, res):
                np.savez(os.path.join(out_dir, "%s.npz" % imdb.image_index[i]), boxes=bx, scores=scores, features=feats,
                         image_h=hw[0], image_w=hw[1])
        del group[:]

    for i in range(len(imdb.image_index)):
        im = cv2.imread(imdb.image_path_at(i))
        blobs, im_scales = _get_blobs(im)
        blob = blobs["data"]
        if group and (len(group) >= batch or group[0][1].shape != blob.shape):
            flush()
        group.append((i, blob, float(im_scales[0]), tuple(im.shape[:2])))
    if group:
        flush()
    return len(imdb.image_index)


def main(argv=None):
    args = parse_args(argv)
    if args.cfg_file is not None:
        cfg_from_file(args.cfg_file)
    if args.set_cfgs is not None:
        cfg_from_list(args.set_cfgs)
    imdb = get_imdb(args.imdb_name)
    net = build_net(args.net, imdb.num_classes, args.model)
    boxes = None
    if args.boxes:
        with open(args.boxes, "rb") as f:
            boxes = pickle.load(f)
    regions = (args.conf_thresh, args.min_boxes, args.max_boxes) if args.regions else None
    if args.tsv and not args.regions:
        raise SystemExit("--tsv needs --regions")
    if args.tsv:
        with open(args.tsv, "w", newline="") as f:
            n = extract(net, imdb, args.out, max(1, args.batch), None, args.max_per_image, regions,
                        tsv_writer(f, net.options["attributes"] is not None))
    else:
        n = extract(net, imdb, args.out, max(1, args.batch), boxes, args.max_per_image, regions)
    print("wrote %d feature files to %s" % (n, args.out))


if __name__ == "__main__":
    sys.exit(main())
