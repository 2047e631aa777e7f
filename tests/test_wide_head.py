"""The fused cls_score | bbox_pred FC of detectors past 1024 classes, host side (frcnn_conv_plan_geometry: no GPU needed): the
work decompositions a 132-SM part (H100 SXM) gives the wide heads, pinned.  `HEAD_CASES` is the case list of
test_wide_head_gpu.py's per-element test: each case's `covers` predicate names the path it exists for, so a change of
decide_geometry's heuristics that moves a case off its path fails here, without a GPU.

The head is one GEMM of rows = RoIs x K = fc7 width with ld_head = ceil(5C/4)*4 output columns (engine.py, fused_cls)."""
import pytest

from tf_faster_rcnn_b200 import _native as N
from test_plan_geometry import geom

IMPLS = {"f16x3": N.CONV_F16X3, "tf32x3": N.CONV_TF32X3, "f16x1": N.CONV_F16X1}


def ld_head(C):
    """Output columns of the fused head: 5C zero-padded to a multiple of 4 (vector stores and split-K apply)."""
    return (5 * C + 3) // 4 * 4


def last_cols(g, cout):
    """Columns of the last N tile."""
    return cout - (g["n_tiles"] - 1) * g["block_n"]


def _ragged(g, n_split, splits):
    """The ragged last round split: n_split tiles, `splits` ways, the K loop cut evenly (no short last split)."""
    return (g["split_tiles"] == n_split and 0 < n_split < g["tiles"] and g["splits"] == splits
            and g["kb_per_split"] * splits == g["k_blocks"])


# name, classes, K (fc7 width), rows (RoIs of the batch), forced plan options, what the case covers (asserted on the geometry)
HEAD_CASES = [
    ("res101_1601", 1601, 2048, 300, {},                                   # bottom-up-attention Visual Genome ResNet-101
     lambda g: g["n_tiles"] == 63 and _ragged(g, 57, 2) and last_cols(g, 8008) == 72),
    ("res101_1601_bn64", 1601, 2048, 300, {"block_n": 64},                 # the same layer at block_n 64: 126 N tiles, no split
     lambda g: g["block_n"] == 64 and g["n_tiles"] == 126 and g["split_tiles"] == 0 and last_cols(g, 8008) == 8),
    ("lvis_1204", 1204, 2048, 300, {},                                     # LVIS: ragged round split 8 ways, last tile 4 wide
     lambda g: g["n_tiles"] == 48 and _ragged(g, 12, 8) and last_cols(g, 6020) == 4),
    ("mobile_1639", 1639, 1024, 300, {},                                   # MobileNet's fc7 width: 65 N tiles, nothing split
     lambda g: g["n_tiles"] == 65 and g["split_tiles"] == 0 and g["splits"] == 1 and last_cols(g, 8196) == 4),
    ("vgg_1601", 1601, 4096, 300, {},                                      # VGG16's fc7 width: the long K loop, split 2 ways
     lambda g: g["n_tiles"] == 63 and _ragged(g, 57, 2) and last_cols(g, 8008) == 72),
    ("b4_4096", 4096, 2048, 1200, {},                                      # the class limit at batch 4: 160 N tiles, 1600 tiles
     lambda g: g["n_tiles"] == 160 and g["tiles"] == 1600 and _ragged(g, 16, 8) and last_cols(g, 20480) == 128),
    ("b4_4096_split3", 4096, 2048, 1200, {"split_k": 3},                   # forced 3-way split of every tile, short last split
     lambda g: g["n_tiles"] == 160 and g["splits"] == 3 and g["split_tiles"] == g["tiles"] == 1600
     and g["k_blocks"] % g["kb_per_split"] != 0),
    ("top_1601", 1601, 2048, 5000, {},                                     # TEST.MODE 'top': 5000 RoIs, 40 M tiles
     lambda g: g["m_tiles"] == 40 and g["n_tiles"] == 63 and _ragged(g, 12, 8) and last_cols(g, 8008) == 72),
]


def head_geom(C, K, M, opt, impl, sms=132):
    return geom(1, 1, M, K, ld_head(C), 1, sms=sms, impl=impl, **opt)


@pytest.mark.parametrize("mode", list(IMPLS))
@pytest.mark.parametrize("case", HEAD_CASES, ids=[c[0] for c in HEAD_CASES])
def test_head_cases_cover_their_paths(case, mode):
    name, C, K, M, opt, covers = case
    g = head_geom(C, K, M, opt, IMPLS[mode])
    assert covers(g), "%s no longer covers its path: %s" % (name, g)


# classes, K, rows -> (cout, N tiles, split tiles, splits, kb_per_split in F16X3, columns of the last N tile)
TABLE = [
    ((1601, 2048, 300), (8008, 63, 57, 2, 16, 72)),
    ((1204, 2048, 300), (6020, 48, 12, 8, 4, 4)),
    ((1639, 1024, 300), (8196, 65, 0, 1, 16, 4)),
    ((1601, 4096, 300), (8008, 63, 57, 2, 32, 72)),
    ((4096, 2048, 1200), (20480, 160, 16, 8, 4, 128)),
    ((1601, 2048, 5000), (8008, 63, 12, 8, 4, 72)),
]


@pytest.mark.parametrize("shape,want", TABLE, ids=["%d_%d_%d" % t[0] for t in TABLE])
def test_wide_head_geometry_table(shape, want):
    """The decompositions of the wide heads in F16X3 (64-wide k-blocks); TF32X3's 32-wide k-blocks double kb_per_split."""
    C, K, M = shape
    cout, n_tiles, n_split, splits, kbs, last = want
    assert ld_head(C) == cout
    g = head_geom(C, K, M, {}, N.CONV_F16X3)
    assert (g["block_n"], g["n_tiles"], g["split_tiles"], g["splits"], g["kb_per_split"], last_cols(g, cout)) == \
        (128, n_tiles, n_split, splits, kbs, last), g
    assert g["grid"] == 132 and g["units"] == g["tiles"] - n_split + n_split * splits
    t = head_geom(C, K, M, {}, N.CONV_TF32X3)
    assert (t["n_tiles"], t["split_tiles"], t["splits"], t["kb_per_split"]) == (n_tiles, n_split, splits, 2 * kbs), t
