"""ctypes binding of libdd3d_b200.so (C ABI declared in include/dd3d_b200.h).

There is NO fallback: if the shared library has not been built (``python -c "import __graft_entry__ as g; g.build()"``
or ``make -C dd3d_b200/csrc``) loading raises, and every compute entry point fails without a CUDA device.
"""
import ctypes as C
import hashlib
import os
import struct
import sys
from typing import Callable, NamedTuple, Optional

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_lib", "libdd3d_b200.so")

MAX_CLASSES = 16        # DD3D_MAX_CLASSES: canonical-size rows of ModelDesc
MAX_NUM_CLASSES = 128   # DD3D_MAX_NUM_CLASSES: largest DD3D.NUM_CLASSES (rows past 16 go through dd3d_set_canonical_sizes)
NUM_LEVELS = 5
FPN_IN_STEM = 1  # DD3D_FPN_IN_STEM: dd3d_set_fpn_inputs number of the VoVNet stem
ARCH_DLA34, ARCH_V2_99 = 0, 1
# dd3d_arch of every arch key (dd3d_b200.arch.ARCH_KEYS)
ARCH_IDS = {"dla34": ARCH_DLA34, "v2_99": ARCH_V2_99, "v2_19_slim_dw": 2, "v2_19_dw": 3, "v2_19_slim": 4, "v2_19": 5,
            "v2_39": 6, "v2_57": 7, "dla_x_46_c": 8, "dla_x_60_c": 9, "dla_x_60": 10, "dla_x_102": 11, "dla_x_102_64": 12}
IMG_U8, IMG_F32 = 0, 1
ACT_BF16, ACT_FP16 = 0, 1
POSE_GLOBAL, POSE_CAMERA = 0, 1
AGG_PATH_ONE_CTA, AGG_PATH_BLOCKED = 1, 2  # dd3d_sample_aggregate_path
GLOBAL_WORDS = 10  # pred_boxes3d_global row: quat (w, x, y, z), tvec, size
NORM_BN_PER_LEVEL, NORM_BN_SHARED, NORM_GN, NORM_NONE = 0, 1, 2, 3  # dd3d_norm
# NORM value -> dd3d_norm (get_norm's table: any other string raises KeyError like its dict lookup).  In a head tower BN /
# FrozenBN are per level (ModuleListDial, fcos2d.py:73-80); the FPN's norms are one per conv, so every BN is "shared" there.
HEAD_NORMS = {"BN": NORM_BN_PER_LEVEL, "FrozenBN": NORM_BN_PER_LEVEL, "SyncBN": NORM_BN_SHARED, "GN": NORM_GN, "": NORM_NONE}
FPN_NORMS = {"BN": NORM_BN_SHARED, "FrozenBN": NORM_BN_SHARED, "SyncBN": NORM_BN_SHARED, "GN": NORM_GN, "": NORM_NONE}
# FE.BACKBONE.NORM -> dd3d_norm of dd3d_set_backbone_norm (eval BatchNorm2d and FrozenBatchNorm2d fold alike)
BACKBONE_NORMS = {"BN": NORM_BN_SHARED, "FrozenBN": NORM_BN_SHARED, "SyncBN": NORM_BN_SHARED, "GN": NORM_GN, "": NORM_NONE}
DET_WORDS = 24  # sizeof(dd3d_det) / 4


class ModelDesc(C.Structure):
    _fields_ = [
        ("arch", C.c_int32),
        ("num_classes", C.c_int32),
        ("pixel_mean", C.c_float * 3),
        ("pixel_std", C.c_float * 3),
        ("feature_locations_offset_half", C.c_int32),
        ("pre_nms_thresh", C.c_float),
        ("pre_nms_topk", C.c_int32),
        ("post_nms_topk", C.c_int32),
        ("nms_thresh", C.c_float),
        ("do_nms", C.c_int32),
        ("min_depth", C.c_float),
        ("max_depth", C.c_float),
        ("scale_depth_by_focal_lengths", C.c_int32),
        ("scale_depth_by_focal_lengths_factor", C.c_float),
        ("predict_allocentric_rot", C.c_int32),
        ("predict_distance", C.c_int32),
        ("canonical_box3d_sizes", C.c_float * (MAX_CLASSES * 3)),
        ("out_cap", C.c_int32),
        ("nuscenes_heads", C.c_int32),
        ("act_dtype", C.c_int32),
        ("thresh_with_ctr", C.c_int32),
        ("fcos2d_use_scale", C.c_int32),
        ("fcos3d_use_scale", C.c_int32),
        ("class_agnostic_box3d", C.c_int32),
        ("per_level_predictors", C.c_int32),
        ("box3d_on", C.c_int32),
    ]


class LayoutDesc(C.Structure):
    """dd3d_layout_desc: the FPN / head structure switches (dd3d_set_layout)."""
    _fields_ = [
        ("fcos2d_norm", C.c_int32),
        ("fcos3d_norm", C.c_int32),
        ("fpn_norm", C.c_int32),
        ("num_cls_convs", C.c_int32),
        ("num_box2d_convs", C.c_int32),
        ("num_box3d_convs", C.c_int32),
        ("fpn_fuse_avg", C.c_int32),
    ]


class TtaView(C.Structure):
    """dd3d_tta_view."""
    _fields_ = [("flip", C.c_int32), ("view_w", C.c_float), ("inv_sx", C.c_float * 2), ("inv_sy", C.c_float * 2),
                ("K_view", C.c_float * 9), ("K_orig", C.c_float * 9)]


# name -> (restype, argtypes); every symbol include/dd3d_b200.h declares
_P, _I, _I64 = C.c_void_p, C.c_int, C.c_int64
SIGNATURES = {
    "dd3d_create": (_I, [C.POINTER(ModelDesc), C.POINTER(_P)]),
    "dd3d_destroy": (None, [_P]),
    "dd3d_last_error": (C.c_char_p, [_P]),
    "dd3d_create_from_file": (_I, [C.c_char_p, C.POINTER(_P)]),
    "dd3d_out_cap": (_I, [_P]),
    "dd3d_size_divisibility": (_I, [_P]),
    "dd3d_set_layout": (_I, [_P, C.POINTER(LayoutDesc)]),
    "dd3d_set_backbone_norm": (_I, [_P, C.c_int32]),
    "dd3d_set_fpn_channels": (_I, [_P, C.c_int32]),
    "dd3d_set_canonical_sizes": (_I, [_P, C.c_int32, C.POINTER(C.c_float)]),
    "dd3d_set_fpn_inputs": (_I, [_P, C.POINTER(C.c_int32), _I]),
    "dd3d_set_in_features": (_I, [_P, C.POINTER(C.c_int32), _I]),
    "dd3d_load_weight": (_I, [_P, C.c_char_p, _P, C.POINTER(_I64), _I]),
    "dd3d_finalize": (_I, [_P]),
    "dd3d_workspace_bytes": (_I64, [_P, _I, _I, _I]),
    "dd3d_plan": (_I, [_P, _I, _I, _I, _P, _I64]),
    "dd3d_forward": (_I, [_P, _P, _I, _P, _P, _P, _P, _P]),
    "dd3d_graph_create": (_I, [_P, _P, _I, _P, _P, _P, _P, _P, C.POINTER(_P)]),
    "dd3d_graph_launch": (_I, [_P, _P]),
    "dd3d_graph_destroy": (None, [_P]),
    "dd3d_graph_kernel_nodes": (_I, [_P]),
    "dd3d_graph_programmatic_edges": (_I, [_P]),
    "dd3d_forward_host": (_I, [_P, _P, _I, _P, _P, _P, _P, _P]),
    "dd3d_set_conv_policy": (_I, [C.c_char_p, _I]),
    "dd3d_submit_host": (_I, [_P, _I, _P, _I, _P, _P, _P, _P, _P]),
    "dd3d_wait_host": (_I, [_P, _I]),
    "dd3d_overflow_flags": (_I, [_P, _P, C.POINTER(C.c_int32)]),
    "dd3d_set_option": (_I, [_P, C.c_char_p, _I]),
    "dd3d_copy_flags": (_I, [_P, _P, _P]),
    "dd3d_set_bev_nms": (_I, [_P, _I, C.c_float]),
    "dd3d_set_poses": (_I, [_P, _P]),
    "dd3d_set_host_poses": (_I, [_P, _I, _P]),
    "dd3d_bev_nms_path": (_I, [C.POINTER(ModelDesc)]),
    "dd3d_set_sample_aggregate": (_I, [_P, _I, C.c_float, _I]),
    "dd3d_set_groups": (_I, [_P, _P, _I]),
    "dd3d_set_host_groups": (_I, [_P, _I, _P, _I]),
    "dd3d_set_global_out": (_I, [_P, _P]),
    "dd3d_set_host_global_out": (_I, [_P, _I, _P]),
    "dd3d_sample_aggregate_path": (_I, [C.POINTER(ModelDesc)]),
    "dd3d_packed_bytes": (_I64, [_I, _I]),
    "dd3d_packed_bytes_global": (_I64, [_I, _I]),
    "dd3d_comm_unique_id": (_I, [_P]),
    "dd3d_comm_create": (_I, [_P, _I, _I, C.POINTER(_P)]),
    "dd3d_comm_from_nccl": (_I, [_P, _I, _I, C.POINTER(_P)]),
    "dd3d_comm_world": (_I, [_P]),
    "dd3d_comm_destroy": (None, [_P]),
    "dd3d_comm_last_error": (C.c_char_p, []),
    "dd3d_allgather": (_I, [_P, _P, _P, _I64, _P]),
    "dd3d_launches_per_forward": (_I, [_P]),
    "dd3d_num_ops": (_I, [_P]),
    "dd3d_get_profile": (_I, [_P, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_double),
                               C.POINTER(C.c_int32)]),
    "dd3d_get_op_times": (_I, [_P, C.POINTER(C.c_float), C.POINTER(C.c_int32), C.POINTER(C.c_double),
                                  C.POINTER(C.c_int32), _I]),
    "dd3d_get_conv_info": (_I, [_P, C.POINTER(C.c_int32), _I]),
    "dd3d_get_tensor": (_I, [_P, C.c_char_p, C.POINTER(_P), C.POINTER(C.c_int32 * 6)]),
    "dd3d_op_conv2d": (_I, [_P, _I, _I, _I, _I, _I, _P, _I, _I, _I, _P, _P, _I, _P, _I, _I, _P, _I, _I, _P]),
    "dd3d_op_conv2d_grouped": (_I, [_P, _I, _I, _I, _I, _I, _P, _I, _I, _P, _P, _I, _P, _I, _P]),
    "dd3d_op_conv2d_tiles": (_I, [_P, _I, _I, _I, _I, _I, _P, _I, _P, _P, _I, _P, _I, _P, _P, _P]),
    "dd3d_op_conv2d_tiles8x8": (_I, [_P, _I, _I, _I, _I, _I, _P, _I, _P, _P, _I, _P, _I, _P, _P, _P]),
    "dd3d_op_conv2d_taps_tiles": (_I, [_P, _I, _I, _I, _I, _I, _P, _I, _P, _P, _I, _P, _I, _I, _P, _P, _P]),
    "dd3d_op_b3d_sparse": (_I, [C.POINTER(_P), C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(_P), C.POINTER(_P),
                                C.POINTER(_P), _P, _P, _I, _I, _I, _I, _P, _I, _P]),
    "dd3d_op_b3d_sparse_c": (_I, [C.POINTER(_P), C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(_P), C.POINTER(_P),
                                  C.POINTER(_P), _P, _P, _I, _I, _I, _I, _P, _I, _I, _P]),
    "dd3d_op_b3d_gather_scratch_bytes": (_I64, [_I, _I, _I]),
    "dd3d_op_b3d_gather": (_I, [C.POINTER(_P), C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(_P), C.POINTER(_P),
                                C.POINTER(_P), _P, _P, _I, _I, _I, _I, _P, _P, _P]),
    "dd3d_op_dla_front": (_I, [_P, _P, _P, _P, _P, _P, _P, _P, _I, _P, _I, _I, _I, _I, _P]),
    "dd3d_op_stem_s2_mma": (_I, [_P, _P, _P, _P, _I, _I, _I, _I, _P]),
    "dd3d_op_dwconv3x3": (_I, [_P, _I, _I, _I, _I, _I, _P, _I, _P, _I, _P]),
    "dd3d_op_group_norm_scratch_bytes": (_I64, [_I, _I, _I]),
    "dd3d_op_group_norm": (_I, [_P, _I, _I, _I, _I, _P, _P, _I, _P, _I, _I, _P, _I, _P, _P]),
    "dd3d_op_group_norm_c": (_I, [_P, _I, _I, _I, _I, _I, _I, _P, _P, _I, _P, _I, _I, _P, _P]),
    "dd3d_op_preprocess": (_I, [_P, _I, _P, _P, _I, _I, _I, _I, _I, C.POINTER(C.c_float), C.POINTER(C.c_float), _P]),
    "dd3d_op_maxpool": (_I, [_P, _P, _I, _I, _I, _I, _I, _I, _I, _P]),
    "dd3d_op_ese": (_I, [_P, _I, _P, _P, _P, _I, _P, _I, _P, _I, _I, _I, _P]),
    "dd3d_op_ese_scratch_bytes": (_I64, [_I, _I, _I]),
    "dd3d_op_bev_nms": (_I, [_P, _P, _P, _P, _P, _P, _I, _I, C.c_float, _I, _P]),
    "dd3d_op_bev_nms_large_scratch_bytes": (_I64, [_I, _I]),
    "dd3d_op_bev_nms_large": (_I, [_P, _P, _P, _P, _P, _P, _P, _I, _I, C.c_float, _I, _P]),
    "dd3d_op_rotated_iou": (_I, [_P, _P, _I, _P, _P]),
    "dd3d_resize_shape": (_I, [_I, _I, _I, _I, _P, _P]),
    "dd3d_forward_raw": (_I, [_P, _P, _I, _I, _P, _P, _I, _I, _P, _P, _P, _P, _P]),
    "dd3d_forward_resized": (_I, [_P, _P, _I, _I, _P, _P, _P, _P, _P, _P, _P, _P]),
    "dd3d_op_tta_merged_cap": (_I, [_I, _I]),
    "dd3d_op_tta_merge_scratch_bytes": (_I64, [_I, _I]),
    "dd3d_op_tta_merge": (_I, [_P, _P, _P, _I, _I, C.c_float, _I, _P, _P, _P, _P, _P]),
    "dd3d_op_tta_merged_cap_large": (_I, [_I, _I]),
    "dd3d_op_tta_merge_large_scratch_bytes": (_I64, [_I, _I]),
    "dd3d_op_tta_merge_large": (_I, [_P, _P, _P, _I, _I, C.c_float, _I, _P, _P, _P, _P, _P]),
    "dd3d_op_resize_preprocess": (_I, [_P, _I, _I, _P, _P, _P, _P, _I, _I, _I, _P, _P, _P]),
    "dd3d_op_sample_aggregate_scratch_bytes": (_I64, [_I, _I]),
    "dd3d_op_sample_aggregate": (_I, [_P, _P, _P, _P, _P, _I, _P, _P, _P, _I, _I, C.c_float, _I, _P]),
    "dd3d_op_group_bev_nms_scratch_bytes": (_I64, [_I, _I, _I]),
    "dd3d_op_group_bev_nms": (_I, [_P, _P, _P, _I, _P, _I, _P, _I, _I, _P, _P, _P, _I, _I, C.c_float, _I, _P]),
    "dd3d_op_group_bev_nms_large_scratch_bytes": (_I64, [_I, _I, _I]),
    "dd3d_op_group_bev_nms_large": (_I, [_P, _P, _P, _I, _P, _I, _P, _I, _I, _P, _P, _P, _I, _I, C.c_float, _I, _P]),
    "dd3d_op_detect_scratch_bytes": (_I64, [_I, _I]),
    "dd3d_op_detect": (_I, [C.POINTER(ModelDesc), _I, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(_P),
                            C.POINTER(_P), C.POINTER(_P), _I, _I, _P, _P, _P, _P, _P, _P, _P, _P]),
    "dd3d_op_detect_flags": (_I, [C.POINTER(ModelDesc), _I, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(_P),
                                  C.POINTER(_P), C.POINTER(_P), _I, _I, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "dd3d_op_detect_c_scratch_bytes": (_I64, [_I, _I, _I]),
    "dd3d_op_detect_c": (_I, [C.POINTER(ModelDesc), C.POINTER(C.c_float), _I, C.POINTER(C.c_int32), C.POINTER(C.c_int32),
                              C.POINTER(_P), C.POINTER(_P), C.POINTER(_P), _I, _I, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
}

_lib = None


def load():
    """Load (once) and return the ctypes library; raises if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} not found: the CUDA extension is not built (run __graft_entry__.build()). "
                "dd3d_b200 has no CPU / PyTorch fallback.")
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)  # AttributeError if the .so lacks a declared symbol
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


def desc_from_cfg(cfg, out_cap=None):
    """dd3d_model_desc from the reference-style cfg tree (the fields DD3D.__init__ reads, core.py:20-55)."""
    from .arch import arch_of
    d = ModelDesc()
    d.arch = ARCH_IDS[arch_of(cfg)]
    d.num_classes = cfg.DD3D.NUM_CLASSES
    for i in range(3):
        d.pixel_mean[i] = cfg.MODEL.PIXEL_MEAN[i]
        d.pixel_std[i] = cfg.MODEL.PIXEL_STD[i]
    d.feature_locations_offset_half = int(cfg.DD3D.FEATURE_LOCATIONS_OFFSET == "half")
    inf = cfg.DD3D.FCOS2D.INFERENCE
    d.thresh_with_ctr = int(bool(inf.THRESH_WITH_CTR))  # fcos2d.py:280-290
    d.pre_nms_thresh = inf.PRE_NMS_THRESH
    d.pre_nms_topk = inf.PRE_NMS_TOPK
    d.post_nms_topk = inf.POST_NMS_TOPK
    d.nms_thresh = inf.NMS_THRESH
    d.do_nms = int(cfg.DD3D.INFERENCE.DO_NMS)
    f3 = cfg.DD3D.FCOS3D
    d.fcos2d_use_scale = int(bool(cfg.DD3D.FCOS2D.USE_SCALE))       # fcos2d.py:100-108,145-152
    d.fcos3d_use_scale = int(bool(f3.USE_SCALE))                    # fcos3d.py:62,116,128-139,175-180
    d.class_agnostic_box3d = int(bool(f3.CLASS_AGNOSTIC_BOX3D))     # fcos3d.py:103,333,352
    d.per_level_predictors = int(bool(f3.PER_LEVEL_PREDICTORS))     # fcos3d.py:65,104,166
    d.box3d_on = int(bool(cfg.MODEL.BOX3D_ON))                      # core.py:34-40,117
    d.min_depth, d.max_depth = f3.MIN_DEPTH, f3.MAX_DEPTH
    d.scale_depth_by_focal_lengths = int(f3.SCALE_DEPTH_BY_FOCAL_LENGTHS)
    d.scale_depth_by_focal_lengths_factor = f3.SCALE_DEPTH_BY_FOCAL_LENGTHS_FACTOR
    d.predict_allocentric_rot = int(f3.PREDICT_ALLOCENTRIC_ROT)
    d.predict_distance = int(f3.PREDICT_DISTANCE)
    sizes = f3.CANONICAL_BOX3D_SIZES
    for c in range(min(len(sizes), MAX_CLASSES)):
        for k in range(3):
            d.canonical_box3d_sizes[c * 3 + k] = sizes[c][k]
    if out_cap is None:
        out_cap = ((inf.POST_NMS_TOPK + 28 + 31) // 32 * 32) if cfg.DD3D.INFERENCE.DO_NMS else max_candidates(cfg)
    d.out_cap = out_cap
    from .arch import is_nuscenes_arch
    d.nuscenes_heads = int(is_nuscenes_arch(cfg))
    d.act_dtype = act_dtype_of(cfg)
    return d


def max_candidates(cfg):
    """Detections one image can have before the 2-D NMS: PRE_NMS_TOPK per head level (DD3D.IN_FEATURES)."""
    from .arch import in_feature_levels
    return len(in_feature_levels(cfg)) * int(cfg.DD3D.FCOS2D.INFERENCE.PRE_NMS_TOPK)


def fpn_inputs_from_cfg(cfg):
    """FE.FPN.IN_FEATURES as the int32 array of dd3d_set_fpn_inputs (level<k> / stage<k> -> k, the VoVNet stem ->
    FPN_IN_STEM), or None for the builder's default list (the default graph, which needs no call)."""
    from .arch import DEFAULT_FPN_INPUTS, DLA_SPECS, arch_of, fpn_inputs
    names = [name for name, _ in fpn_inputs(cfg)]
    if names == DEFAULT_FPN_INPUTS[arch_of(cfg) in DLA_SPECS]:
        return None
    nums = [FPN_IN_STEM if name == "stem" else int(name[-1]) for name in names]
    return (C.c_int32 * len(nums))(*nums), len(nums)


def in_features_from_cfg(cfg):
    """DD3D.IN_FEATURES as the int32 array of dd3d_set_in_features, or None for every FPN output in order (the default
    graph, which needs no call)."""
    from .arch import fpn_output_names, in_feature_levels
    levels = in_feature_levels(cfg)
    if levels == list(range(len(fpn_output_names(cfg)))):
        return None
    return (C.c_int32 * len(levels))(*levels), len(levels)


def canonical_sizes_from_cfg(cfg):
    """FCOS3D.CANONICAL_BOX3D_SIZES rows 0..NUM_CLASSES-1 as the flat fp32 array of dd3d_set_canonical_sizes.  Fewer rows than
    classes raise IndexError (the reference indexes the table by predicted class, fcos3d.py:378)."""
    n, sizes = int(cfg.DD3D.NUM_CLASSES), cfg.DD3D.FCOS3D.CANONICAL_BOX3D_SIZES
    if len(sizes) < n:
        raise IndexError(f"FCOS3D.CANONICAL_BOX3D_SIZES has {len(sizes)} rows for DD3D.NUM_CLASSES = {n}")
    return (C.c_float * (3 * n))(*[float(sizes[c][k]) for c in range(n) for k in range(3)])


def layout_from_cfg(cfg):
    """dd3d_layout_desc from the cfg keys the reference builds the FPN and the heads from (fcos2d.py:46-91,
    fcos3d.py:75-112, detectron2 FPN norm / fuse_type).  Unknown NORM strings raise KeyError, like get_norm."""
    f2, f3, fpn = cfg.DD3D.FCOS2D, cfg.DD3D.FCOS3D, cfg.FE.FPN
    d = LayoutDesc()
    d.fcos2d_norm = HEAD_NORMS[f2.NORM]
    d.fcos3d_norm = HEAD_NORMS[f3.NORM]
    d.fpn_norm = FPN_NORMS[fpn.NORM]
    d.num_cls_convs = int(f2.NUM_CLS_CONVS)
    d.num_box2d_convs = int(f2.NUM_BOX_CONVS)
    d.num_box3d_convs = int(f3.NUM_CONVS)
    if fpn.FUSE_TYPE not in ("sum", "avg"):  # FPN.__init__: assert fuse_type in {"avg", "sum"}
        raise ValueError(f"FE.FPN.FUSE_TYPE must be 'sum' or 'avg', got {fpn.FUSE_TYPE!r}")
    d.fpn_fuse_avg = int(fpn.FUSE_TYPE == "avg")
    return d


def act_dtype_of(cfg):
    """cfg.B200.ACT_DTYPE ("bf16" default | "fp16"): the engine's 16-bit storage type; an engine-side key that reference
    configs do not carry (absent -> bf16)."""
    node = cfg.get("B200") if hasattr(cfg, "get") else getattr(cfg, "B200", None)
    name = str((node or {}).get("ACT_DTYPE", "bf16")).lower()
    if name not in ("bf16", "fp16"):
        raise ValueError(f"B200.ACT_DTYPE must be 'bf16' or 'fp16', got {name!r}")
    return ACT_FP16 if name == "fp16" else ACT_BF16


class EngineSpec(NamedTuple):
    """What dd3d_create .. dd3d_finalize receive, in call order (DD3DB200._engine_spec): DD3DB200._engine makes the calls
    from it, write_model_file stores it for dd3d_create_from_file, which makes the same calls."""
    desc: ModelDesc
    layout: LayoutDesc
    backbone_norm: int                  # dd3d_set_backbone_norm
    fpn_channels: int                   # dd3d_set_fpn_channels
    fpn_inputs: Optional[tuple]         # (int32 array, n) of dd3d_set_fpn_inputs, or None: not called
    in_features: Optional[tuple]        # (int32 array, n) of dd3d_set_in_features, or None: not called
    canonical_sizes: Optional[tuple]    # (num_classes, float array) of dd3d_set_canonical_sizes, or None: not called
    tensors: Callable                   # () -> iterable of (name, contiguous fp32 CPU tensor), one dd3d_load_weight each


MODEL_FILE_MAGIC = b"DD3DB200"
MODEL_FILE_VERSION = 1
MODEL_FILE_HEADER = struct.Struct("<8sIIIIQ")  # magic, version, desc bytes, layout bytes, tensor records, file bytes


def write_model_file(path, spec):
    """Writes `spec` as the self-contained model file dd3d_create_from_file reads (layout: include/dd3d_b200.h): header,
    dd3d_model_desc, dd3d_layout_desc, the dd3d_set_* values, one record per tensor, then the 8-byte BLAKE2b checksum of
    everything before it.  Host only: no GPU is needed."""
    if sys.byteorder != "little":
        raise NotImplementedError("the model file is little-endian and written from the host's own struct layout")
    tensors = list(spec.tensors())

    def int_list(arg):
        return struct.pack("<I", 0) if arg is None else struct.pack("<I", arg[1]) + bytes(arg[0])

    canon = spec.canonical_sizes
    body = (bytes(spec.desc) + bytes(spec.layout) + struct.pack("<ii", spec.backbone_norm, spec.fpn_channels) +
            int_list(spec.fpn_inputs) + int_list(spec.in_features) +
            (struct.pack("<I", 0) if canon is None else struct.pack("<I", canon[0]) + bytes(canon[1])))
    heads = [struct.pack(f"<I{len(name.encode())}sI{t.dim()}q", len(name.encode()), name.encode(), t.dim(), *t.shape)
             for name, t in tensors]
    size = MODEL_FILE_HEADER.size + len(body) + sum(len(h) + 4 * t.numel() for h, (_, t) in zip(heads, tensors)) + 8
    digest = hashlib.blake2b(digest_size=8)
    with open(path, "wb") as f:
        def put(data):
            digest.update(data)
            f.write(data)

        put(MODEL_FILE_HEADER.pack(MODEL_FILE_MAGIC, MODEL_FILE_VERSION, C.sizeof(ModelDesc), C.sizeof(LayoutDesc),
                                   len(tensors), size))
        put(body)
        for head, (name, t) in zip(heads, tensors):
            data = t.reshape(-1).numpy()
            if data.dtype.str != "<f4":
                raise TypeError(f"tensor {name}: the model file holds fp32, got {data.dtype}")
            put(head)
            put(memoryview(data).cast("B"))
        f.write(digest.digest())


def check(status, handle=None):
    if status < 0:
        msg = load().dd3d_last_error(handle)
        raise RuntimeError(f"dd3d_b200 error {status}: {msg.decode() if msg else ''}")
    return status
