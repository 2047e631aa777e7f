"""Global option tree `cfg` with the reference's keys, defaults and merge rules
(lib/model/config.py: defaults :19-290, get_output_dir :293-306, _merge_a_into_b :325-355,
cfg_from_file :358-364, cfg_from_list :367-387).

easydict is not a dependency here: `AttrDict` below gives the same attribute access.  TRAIN.* keys
are carried as data only (the experiment YAMLs set them and the strict merge rejects unknown keys);
nothing on the inference path reads them except BBOX_NORMALIZE_MEANS/STDS (network.py:429-430).
"""
import os
import os.path as osp
from ast import literal_eval

import numpy as np


class AttrDict(dict):
    """dict whose items are also attributes; nested dicts are converted on construction."""

    def __init__(self, *args, **kw):
        super().__init__()
        for k, v in dict(*args, **kw).items():
            self[k] = v

    def __setitem__(self, k, v):
        super().__setitem__(k, AttrDict(v) if isinstance(v, dict) and not isinstance(v, AttrDict) else v)

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError:
            raise AttributeError(k)

    __setattr__ = __setitem__


# the REPOSITORY root (three levels above lib/model/): data/, output/ live next to tools/ as in the reference layout
_ROOT = osp.abspath(osp.join(osp.dirname(__file__), "..", "..", ".."))

cfg = AttrDict(
    TRAIN=dict(
        LEARNING_RATE=0.001, MOMENTUM=0.9, WEIGHT_DECAY=0.0001, GAMMA=0.1, STEPSIZE=[30000], DISPLAY=10,
        DOUBLE_BIAS=True, TRUNCATED=False, BIAS_DECAY=False, USE_GT=False, ASPECT_GROUPING=False,
        SNAPSHOT_KEPT=3, SUMMARY_INTERVAL=180, SCALES=(600,), MAX_SIZE=1000, IMS_PER_BATCH=1, BATCH_SIZE=128,
        FG_FRACTION=0.25, FG_THRESH=0.5, BG_THRESH_HI=0.5, BG_THRESH_LO=0.1, USE_FLIPPED=True, BBOX_REG=True,
        BBOX_THRESH=0.5, SNAPSHOT_ITERS=5000, SNAPSHOT_PREFIX="res101_faster_rcnn",
        BBOX_NORMALIZE_TARGETS=True, BBOX_INSIDE_WEIGHTS=(1.0, 1.0, 1.0, 1.0),
        BBOX_NORMALIZE_TARGETS_PRECOMPUTED=True, BBOX_NORMALIZE_MEANS=(0.0, 0.0, 0.0, 0.0),
        BBOX_NORMALIZE_STDS=(0.1, 0.1, 0.2, 0.2), PROPOSAL_METHOD="gt", HAS_RPN=True,
        RPN_POSITIVE_OVERLAP=0.7, RPN_NEGATIVE_OVERLAP=0.3, RPN_CLOBBER_POSITIVES=False, RPN_FG_FRACTION=0.5,
        RPN_BATCHSIZE=256, RPN_NMS_THRESH=0.7, RPN_PRE_NMS_TOP_N=12000, RPN_POST_NMS_TOP_N=2000,
        RPN_BBOX_INSIDE_WEIGHTS=(1.0, 1.0, 1.0, 1.0), RPN_POSITIVE_WEIGHT=-1.0, USE_ALL_GT=True,
    ),
    TEST=dict(
        SCALES=(600,), MAX_SIZE=1000, NMS=0.3, SVM=False, BBOX_REG=True, HAS_RPN=False, PROPOSAL_METHOD="gt",
        RPN_NMS_THRESH=0.7, RPN_PRE_NMS_TOP_N=6000, RPN_POST_NMS_TOP_N=300, MODE="nms", RPN_TOP_N=5000,
        # extension (Detectron's TEST.SOFT_NMS): Soft-NMS in place of the final per-class NMS; overlap threshold TEST.NMS.
        # METHOD linear | gaussian | hard, SIGMA > 0 (gaussian), SCORE_THRESH > 0 (prune threshold); USE_GPU_NMS does not apply
        SOFT_NMS=dict(ENABLED=False, METHOD="linear", SIGMA=0.5, SCORE_THRESH=0.001),
        # extension (Detectron's TEST.BBOX_AUG, union mode): test-time augmentation.  Views: the base (SCALES[0], MAX_SIZE), one per
        # BBOX_AUG.SCALES entry (short side, long side capped by BBOX_AUG.MAX_SIZE), and with H_FLIP the mirrored twin of each; the
        # boxes of every view are merged ahead of the per-class NMS (model/test.py::aug_views gives the order)
        BBOX_AUG=dict(ENABLED=False, H_FLIP=False, SCALES=(), MAX_SIZE=2000),
        # extension (Detectron's TEST.BBOX_VOTE): after the per-class NMS / Soft-NMS each kept box becomes the score-weighted mean
        # of its class's candidates overlapping it by >= VOTE_TH (0 < VOTE_TH <= 1); SCORING_METHOD ID (score unchanged) | AVG |
        # IOU_AVG | GENERALIZED_AVG | QUASI_SUM | TEMP_AVG, SCORING_METHOD_BETA finite and > 0.  The max_per_image cap follows.
        BBOX_VOTE=dict(ENABLED=False, VOTE_TH=0.8, SCORING_METHOD="ID", SCORING_METHOD_BETA=1.0),
    ),
    RESNET=dict(MAX_POOL=False, FIXED_BLOCKS=1),
    MOBILENET=dict(REGU_DEPTH=False, FIXED_LAYERS=5, WEIGHT_DECAY=0.00004, DEPTH_MULTIPLIER=1.0),
    PIXEL_MEANS=np.array([[[102.9801, 115.9465, 122.7717]]]),
    RNG_SEED=3,
    ROOT_DIR=_ROOT,
    DATA_DIR=osp.join(_ROOT, "data"),
    MATLAB="matlab",
    EXP_DIR="default",
    USE_GPU_NMS=True,
    USE_E2E_TF=True,
    # 'crop' (crop_and_resize, the reference's), or the extensions 'align' (RoIAlign, torchvision.ops.roi_align) and 'pool'
    # (Fast R-CNN's RoIPool, torchvision.ops.roi_pool), which pool straight to POOLING_SIZE x POOLING_SIZE (1..16)
    POOLING_MODE="crop",
    POOLING_SIZE=7,
    # 'align' mode only: SAMPLING_RATIO int in [0, 16] samples per bin and axis (0 = adaptive, ceil(RoI size / POOLING_SIZE));
    # ALIGNED: shift the RoI by -0.5 feature cells and drop the minimum size of 1 (Detectron2's RoIAlignV2)
    ROI_ALIGN=dict(SAMPLING_RATIO=0, ALIGNED=False),
    ANCHOR_SCALES=[8, 16, 32],
    ANCHOR_RATIOS=[0.5, 1, 2],
    RPN_CHANNELS=512,
    # extension (the Visual Genome model of bottom-up-attention): the attribute head on detect_regions' regions.  NUM_CLASSES 0 =
    # no head, else 2..4096 attribute classes (Visual Genome: 401, 0 = "no attribute"); EMBED_DIM (the class embedding) and HIDDEN
    # (fc_attr's width) are positive multiples of 32
    ATTRIBUTES=dict(NUM_CLASSES=0, EMBED_DIM=256, HIDDEN=512),
)


def _artifact_dir(kind, imdb, weights_filename):
    d = osp.join(osp.abspath(osp.join(cfg.ROOT_DIR, kind, cfg.EXP_DIR, imdb.name)), weights_filename or "default")
    os.makedirs(d, exist_ok=True)
    return d


def get_output_dir(imdb, weights_filename):
    """<ROOT>/output/<EXP_DIR>/<imdb.name>/<weights_filename|default>, created on demand."""
    return _artifact_dir("output", imdb, weights_filename)


def get_output_tb_dir(imdb, weights_filename):
    return _artifact_dir("tensorboard", imdb, weights_filename)


def _merge(src, dst, path=""):
    """Strict merge: every key of `src` must exist in `dst` with the same type
    (ndarray targets accept anything convertible)."""
    for key, val in src.items():
        where = path + key
        if key not in dst:
            raise KeyError("{} is not a valid config key".format(where))
        cur = dst[key]
        if isinstance(cur, AttrDict):
            if not isinstance(val, dict):
                raise ValueError("Type mismatch ({} vs. {}) for config key: {}".format(type(cur), type(val), where))
            _merge(val, cur, where + ".")
            continue
        if type(cur) is not type(val):
            if isinstance(cur, np.ndarray):
                val = np.array(val, dtype=cur.dtype)
            elif isinstance(cur, (list, tuple)) and isinstance(val, (list, tuple)):
                # deviation (superset): the reference rejects `SCALES: [800]` against the tuple default, which makes
                # its own experiments/cfgs/res101-lg.yml unloadable; sequences are coerced to the default's type.
                val = type(cur)(val)
            else:
                raise ValueError("Type mismatch ({} vs. {}) for config key: {}".format(type(cur), type(val), where))
        dst[key] = val


def cfg_from_file(filename):
    """Merge a YAML experiment file (experiments/cfgs/*.yml) into `cfg`."""
    import yaml
    with open(filename, "r") as f:
        loaded = yaml.safe_load(f) or {}
    _merge(loaded, cfg)


def cfg_from_list(cfg_list):
    """`--set KEY VALUE ...` overrides; VALUE goes through literal_eval, strings stay strings."""
    assert len(cfg_list) % 2 == 0
    for dotted, raw in zip(cfg_list[0::2], cfg_list[1::2]):
        node = cfg
        *parents, leaf = dotted.split(".")
        for name in parents:
            assert name in node
            node = node[name]
        assert leaf in node
        try:
            value = literal_eval(raw)
        except Exception:
            value = raw
        assert type(value) == type(node[leaf]), \
            "type {} does not match original type {}".format(type(value), type(node[leaf]))
        node[leaf] = value
