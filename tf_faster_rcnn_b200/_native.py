"""ctypes binding of libfrcnn_b200.so (the C ABI declared in include/frcnn_b200.h).

There is NO Python/CPU fallback: if the library is missing or a call fails, a
RuntimeError carrying frcnn_last_error() is raised.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# FRCNN_LIB_VARIANT=wd selects the development build with barrier-wait watchdogs (tools only; never the default)
LIB_PATH = os.path.join(_HERE, "libfrcnn_b200_wd.so" if os.environ.get("FRCNN_LIB_VARIANT") == "wd" else "libfrcnn_b200.so")

NMS_PLUS_ONE, NMS_INCLUSIVE, NMS_SKIP_DEGENERATE = 1, 2, 4
NMS_MODE_CPU_NMS = NMS_PLUS_ONE | NMS_INCLUSIVE
NMS_MODE_GPU_NMS = NMS_PLUS_ONE
NMS_MODE_TF = NMS_SKIP_DEGENERATE
ACT_NONE, ACT_RELU, ACT_RELU6 = 0, 1, 2
CONV_F16X3, CONV_TF32X3, CONV_F16X1 = 0, 1, 2
SOFT_NMS_METHODS = {"linear": 0, "gaussian": 1, "hard": 2}   # FRCNN_SOFT_NMS_*
AUG_MAX_VIEWS = 16                                            # FRCNN_AUG_MAX_VIEWS
BOX_VOTE_METHODS = {"ID": 0, "AVG": 1, "IOU_AVG": 2, "GENERALIZED_AVG": 3, "QUASI_SUM": 4, "TEMP_AVG": 5}   # FRCNN_BOX_VOTE_*
ROI_ALIGN_MAX_SAMPLING = 16                                   # FRCNN_ROI_ALIGN_MAX_SAMPLING
ROI_MAX_POOLED = 16                                           # pooled sizes 1..16 of frcnn_roi_align / frcnn_roi_pool

vp, ci, cf, cu, sz = C.c_void_p, C.c_int, C.c_float, C.c_uint, C.c_size_t
ip, fp = C.POINTER(C.c_int), C.POINTER(C.c_float)


class ConvDesc(C.Structure):
    """frcnn_conv_desc"""
    _fields_ = [("in_dev", vp), ("w_hi_dev", vp), ("w_lo_dev", vp), ("scale_dev", vp), ("shift_dev", vp),
                ("residual_dev", vp), ("out_dev", vp),
                ("n", ci), ("h", ci), ("w", ci), ("cin", ci), ("cout", ci), ("kh", ci), ("kw", ci), ("stride", ci),
                ("pad_t", ci), ("pad_l", ci), ("ho", ci), ("wo", ci), ("act", ci), ("block_n", ci), ("kb_per_chunk", ci), ("split_k", ci),
                ("impl", ci), ("out_mult", cf), ("in2_dev", vp), ("cin2", ci), ("mean_dev", vp), ("mean_hw", ci)]


# name -> (restype, argtypes); must list every symbol of include/frcnn_b200.h (checked by tests/test_abi.py)
SIGNATURES = {
    "frcnn_version": (ci, []),
    "frcnn_last_error": (ci, [C.c_char_p, sz]),
    "frcnn_check_device": (ci, [ci]),
    "frcnn_zero_async": (ci, [vp, sz, vp]),
    "frcnn_graph_begin": (ci, [vp]),
    "frcnn_graph_end": (ci, [vp, C.POINTER(vp)]),
    "frcnn_graph_launch": (ci, [vp, vp]),
    "frcnn_graph_destroy": (None, [vp]),
    "frcnn_nms_host": (ci, [ip, ip, fp, ci, ci, cf, ci, cu]),
    "frcnn_nms_sorted_dev": (ci, [vp, ci, cf, cu, ci, vp, vp, vp]),
    "frcnn_conv_plan_create": (ci, [C.POINTER(vp), C.POINTER(ConvDesc)]),
    "frcnn_conv_plan_run": (ci, [vp, vp]),
    "frcnn_conv_plan_geometry": (ci, [C.POINTER(ConvDesc), ci, ip]),
    "frcnn_conv_plan_info": (ci, [vp, ip, ip, ip, ip, ip, ip, ip, ip]),
    "frcnn_conv_plan_set_trace": (ci, [vp, vp]),
    "frcnn_conv_plan_destroy": (None, [vp]),
    "frcnn_debug_watchdog": (ci, [C.POINTER(C.c_uint), ci]),
    "frcnn_pack_conv_weights": (ci, [vp, vp, vp, ci, ci, ci, ci, ci, vp]),
    "frcnn_pack_conv_weights_tf32": (ci, [vp, vp, vp, ci, ci, ci, ci, vp]),
    "frcnn_conv_first": (ci, [vp, vp, vp, vp, vp, ci, ci, ci, ci, ci, ci, ci, ci, ci, ci, ci, vp]),
    "frcnn_depthwise3x3": (ci, [vp, vp, vp, vp, vp, ci, ci, ci, ci, ci, ci, ci, ci, ci, ci, vp]),
    "frcnn_max_pool": (ci, [vp, vp, ci, ci, ci, ci, ci, ci, ci, ci, ci, ci, ci, vp]),
    "frcnn_spatial_mean": (ci, [vp, vp, ci, ci, ci, vp]),
    "frcnn_preprocess": (ci, [vp, ci, ci, C.POINTER(C.c_double), C.c_double, C.c_double, vp, ci, ci, vp]),
    "frcnn_rpn_decode": (ci, [vp, ci, ci, vp, ci, ci, ci, ci, ci, cf, cf, vp, vp, vp]),
    "frcnn_sort_workspace_bytes": (sz, [ci]),
    "frcnn_sort_desc": (ci, [vp, ci, ci, vp, vp, vp, sz, vp]),
    "frcnn_proposals": (ci, [vp, vp, vp, ci, ci, ci, ci, cf, cu, vp, vp, vp, vp, vp]),
    "frcnn_crop_pool": (ci, [vp, ci, ci, ci, ci, vp, ci, ci, ci, vp, vp]),
    "frcnn_roi_align": (ci, [vp, ci, ci, ci, ci, vp, ci, ci, cf, ci, ci, vp, vp]),
    "frcnn_roi_pool": (ci, [vp, ci, ci, ci, ci, vp, ci, ci, cf, vp, vp]),
    "frcnn_cls_finish": (ci, [vp, ci, ci, ci, fp, fp, vp, vp, vp, vp]),
    "frcnn_bbox_decode": (ci, [vp, vp, ci, ci, ci, vp, vp, vp]),
    "frcnn_detect_post_workspace_bytes": (sz, [ci, ci, ci]),
    "frcnn_detect_regions_workspace_bytes": (ci, [ci, ci, ci, C.POINTER(sz)]),
    "frcnn_detect_post": (ci, [vp, vp, vp, ci, ci, ci, cf, cf, cu, ci, ci, vp, vp, ci, vp, vp, vp, vp, sz, vp]),
    "frcnn_soft_nms_host": (ci, [fp, ip, ip, fp, ci, ci, ci, cf, cf, cf, ci]),
    "frcnn_detect_post_soft": (ci, [vp, vp, vp, ci, ci, ci, cf, ci, cf, cf, cf, ci, ci, vp, vp, ci, vp, vp, vp, vp, sz, vp]),
    "frcnn_detect_features": (ci, [vp, vp, vp, ci, ci, ci, ci, ci, vp, vp, vp]),
    "frcnn_detect_regions": (ci, [vp, vp, vp, vp, vp, ci, ci, ci, ci, cf, cu, cf, ci, ci, vp, vp, vp, vp, sz, vp, vp, vp, vp, vp, vp, vp,
                                  vp, vp]),
    "frcnn_regions_attr_embed": (ci, [vp, ci, ci, ci, vp, vp, ci, vp, ci, vp, vp]),
    "frcnn_attr_finish": (ci, [vp, ci, ci, ci, ci, vp, vp, vp, vp, vp]),
    "frcnn_boxes_to_rois": (ci, [vp, vp, vp, ci, ci, vp, vp, vp]),
    "frcnn_preprocess_hflip": (ci, [vp, ci, ci, C.POINTER(C.c_double), C.c_double, C.c_double, vp, ci, ci, vp]),
    "frcnn_aug_union": (ci, [C.POINTER(vp), C.POINTER(vp), C.POINTER(vp), ip, ip, ci, ci, ci, vp, vp, vp, vp, vp]),
    "frcnn_box_vote_host": (ci, [fp, fp, ci, ci, fp, ci, ci, cf, ci, cf, ci]),
    "frcnn_detect_post_vote": (ci, [vp, vp, vp, ci, ci, ci, cf, cf, cu, ci, ci, vp, vp, ci, vp, vp, vp, vp, sz, cf, ci, cf, vp, vp]),
    "frcnn_detect_post_soft_vote": (ci, [vp, vp, vp, ci, ci, ci, cf, ci, cf, cf, cf, ci, ci, vp, vp, ci, vp, vp, vp, vp, sz, cf, ci, cf, vp,
                                         vp]),
}

_lib = None


def lib():
    """Load the shared library (once).  Raises if it has not been built -- build with
    `python -m tf_faster_rcnn_b200.csrc.build` or `__graft_entry__.build()`."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError("libfrcnn_b200.so not built (%s): the CUDA extension is mandatory, "
                               "there is no CPU fallback" % LIB_PATH)
        L = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def last_error():
    buf = C.create_string_buffer(512)
    lib().frcnn_last_error(buf, 512)
    return buf.value.decode("utf-8", "replace")


def check(rc, what=""):
    if rc != 0:
        raise RuntimeError("frcnn_b200 %s failed (status %d): %s" % (what, rc, last_error()))
