"""ctypes binding of libb200det.so (include/b200det.h).  Loading never needs a GPU; every compute
entry point fails loudly (RuntimeError with b2_last_error()) instead of falling back to the CPU."""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, c_char_p, c_float, c_int, c_int32, c_int64, c_void_p

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libb200det.so")


class B2Config(ctypes.Structure):
    _fields_ = [
        ("batch", c_int32), ("height", c_int32), ("width", c_int32), ("input_dtype", c_int32),
        ("num_class", c_int32), ("resnet_blocks", c_int32 * 4), ("use_dilations", c_int32),
        ("class_agnostic", c_int32), ("rpn_topk", c_int32), ("result_per_im", c_int32),
        ("fpn_num_channel", c_int32), ("fc_head_dim", c_int32), ("precision", c_int32),
        ("conv_impl", c_int32), ("use_cuda_graph", c_int32),
        ("max_size", c_float), ("rpn_min_size", c_float), ("rpn_nms_thres", c_float),
        ("fastrcnn_nms_iou_thres", c_float), ("result_score_thres", c_float),
        ("anchor_strides", c_float * 5), ("anchor_sizes", c_float * 5), ("anchor_ratios", c_float * 3),
        ("bbox_reg_weights", c_float * 4), ("accum_chunk", c_int32), ("multi_semantics", c_int32),
        ("add_mask", c_int32), ("use_gn", c_int32), ("conv_head_dim", c_int32), ("use_se", c_int32),
        ("use_resnext", c_int32), ("add_relation_nn", c_int32), ("use_deformable", c_int32),
    ]


class B2ConfigExt(ctypes.Structure):
    _fields_ = [("use_basic_block", c_int32)]


class B2ConfigExt2(ctypes.Structure):
    _fields_ = [("num_partial_classes", c_int32), ("partial_class_ids", c_int32 * 80)]


class B2ConfigExt3(ctypes.Structure):
    _fields_ = [("use_att_frcnn_head", c_int32)]


class B2ConfigExt4(ctypes.Structure):
    _fields_ = [("use_small_object_head", c_int32), ("num_small_objects", c_int32),
                ("small_object_class_ids", c_int32 * 80), ("use_so_association", c_int32), ("so_person_class_id", c_int32),
                ("so_person_topk", c_int32), ("use_so_score_thres", c_int32)]


class B2ConfigExt5(ctypes.Structure):
    _fields_ = [("use_bg_score", c_int32)]


class B2EffdetConfig(ctypes.Structure):
    _fields_ = [
        ("image_h", c_int32), ("image_w", c_int32), ("min_level", c_int32), ("max_level", c_int32),
        ("fpn_num_filters", c_int32), ("fpn_cell_repeats", c_int32), ("box_class_repeats", c_int32),
        ("num_classes", c_int32), ("num_scales", c_int32), ("num_aspects", c_int32),
        ("aspect_ratios", (c_float * 2) * 3), ("anchor_scale", c_float), ("fpn_weight_method", c_int32),
        ("backbone_channels", c_int32 * 3), ("max_detection_topk", c_int32), ("result_per_im", c_int32),
        ("nms_iou_threshold", c_float), ("result_score_thres", c_float), ("precision", c_int32), ("backbone", c_int32),
        ("batch", c_int32),
    ]


class B2ConvView(ctypes.Structure):
    _fields_ = [(name, c_int32) for name in (
        "B", "pitch_H", "pitch_W", "in_ld", "in_H", "in_W", "Cin", "R", "S", "stride", "dil", "pad_t", "pad_b", "pad_l",
        "pad_r", "Cout", "out_H", "out_W", "off_h", "off_w", "ldc", "out_f32", "res_H", "res_W", "ldr", "res_shift", "relu",
        "acc_kb", "a_mode", "force_epi", "impl", "split", "b0", "nb")]


# every symbol include/b200det.h declares: (name, restype, argtypes)
SYMBOLS = [
    ("b2_last_error", c_char_p, []),
    ("b2_version", c_int, []),
    ("b2_create", c_int, [POINTER(c_void_p), c_int, POINTER(B2Config)]),
    ("b2_create_ex", c_int, [POINTER(c_void_p), c_int, POINTER(B2Config), POINTER(B2ConfigExt)]),
    ("b2_create_ex2", c_int, [POINTER(c_void_p), c_int, POINTER(B2Config), POINTER(B2ConfigExt), POINTER(B2ConfigExt2)]),
    ("b2_create_ex3", c_int, [POINTER(c_void_p), c_int, POINTER(B2Config), POINTER(B2ConfigExt), POINTER(B2ConfigExt2),
                              POINTER(B2ConfigExt3)]),
    ("b2_create_ex4", c_int, [POINTER(c_void_p), c_int, POINTER(B2Config), POINTER(B2ConfigExt), POINTER(B2ConfigExt2),
                              POINTER(B2ConfigExt3), POINTER(B2ConfigExt4)]),
    ("b2_create_ex5", c_int, [POINTER(c_void_p), c_int, POINTER(B2Config), POINTER(B2ConfigExt), POINTER(B2ConfigExt2),
                              POINTER(B2ConfigExt3), POINTER(B2ConfigExt4), POINTER(B2ConfigExt5)]),
    ("b2_get_small_objects", c_int, [c_void_p] + [c_void_p] * 6),
    ("b2_fpn_feature", c_int, [c_void_p, c_void_p, c_void_p]),
    ("b2_fpn_feature_launches", c_int, [c_void_p]),
    ("b2_get_proposals", c_int, [c_void_p] * 4),
    ("b2_get_all_boxes", c_int, [c_void_p, c_int] + [c_void_p] * 4),
    ("b2_masks_create", c_int, [POINTER(c_void_p), c_int]),
    ("b2_masks_destroy", None, [c_void_p]),
    ("b2_masks_paste", c_int, [c_void_p, c_void_p, c_void_p] + [c_int] * 6 + [c_void_p, c_int64]),
    ("b2_masks_encode", c_int, [c_void_p, c_void_p, c_void_p] + [c_int] * 6 + [c_void_p, c_void_p, c_int64]),
    ("b2_masks_fetch", c_int, [c_void_p, c_void_p, c_int64]),
    ("b2_encode_masks", c_int, [c_void_p, c_void_p, c_int, c_void_p] + [c_int] * 3 + [c_void_p, c_void_p, c_int64]),
    ("b2_destroy", None, [c_void_p]),
    ("b2_load_weights", c_int, [c_void_p, POINTER(c_char_p), POINTER(c_void_p), POINTER(c_int64), c_int]),
    ("b2_detect", c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int]),
    ("b2_detect_host", c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int]),
    ("b2_detect_host_resize", c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int]),
    ("b2_resize_frames", c_int, [c_int, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    ("b2_submit_host", c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int]),
    ("b2_wait", c_int, [c_void_p, c_int]),
    ("b2_submit_host_resize", c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int]),
    ("b2_box_features", c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p]),
    ("b2_get_masks", c_int, [c_void_p, c_void_p, c_int64]),
    ("b2_stage_shape", c_int, [c_void_p, c_char_p, POINTER(c_int64), POINTER(c_int32)]),
    ("b2_get_stage", c_int, [c_void_p, c_char_p, c_void_p, c_int64]),
    ("b2_set_stage", c_int, [c_void_p, c_char_p, c_void_p, c_int64]),
    ("b2_run_phases", c_int, [c_void_p, c_int]),
    ("b2_phase_times", c_int, [c_void_p, POINTER(c_float)]),
    ("b2_kernel_launches", c_int, [c_void_p]),
    ("b2_num_steps", c_int, [c_void_p]),
    ("b2_profile_steps", c_int, [c_void_p, c_int, POINTER(c_float), c_int, POINTER(c_int)]),
    ("b2_step_info", c_int, [c_void_p, c_int, ctypes.c_char_p, c_int, POINTER(ctypes.c_double), POINTER(ctypes.c_double), POINTER(c_int)]),
    ("b2_cosine_cost", c_int, [c_int, c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_void_p]),
    ("b2_tracker_create", c_int, [POINTER(c_void_p), c_int, ctypes.c_double, c_int, c_int, ctypes.c_double, c_int, c_int, c_int]),
    ("b2_tracker_destroy", None, [c_void_p]),
    ("b2_tracker_set_cost_fn", c_int, [c_void_p, c_void_p, c_void_p]),
    ("b2_tracker_predict", c_int, [c_void_p]),
    ("b2_tracker_update", c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int]),
    ("b2_tracker_num_tracks", c_int, [c_void_p]),
    ("b2_tracker_get_tracks", c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    ("b2_linear_sum_assignment", c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p]),
    ("b2_track_nms", c_int, [c_void_p, c_void_p, c_int, ctypes.c_double, c_void_p]),
    ("b2_lapjv", c_int, [c_void_p, c_int, c_int, ctypes.c_double, c_void_p, c_void_p, POINTER(ctypes.c_double)]),
    ("b2_tmot_iou_distance", c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p]),
    ("b2_tmot_fuse_motion", c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, ctypes.c_double]),
    ("b2_tmot_embedding_distance", c_int, [c_int, c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_void_p]),
    ("b2_jde_create", c_int, [POINTER(c_void_p), c_int] + [ctypes.c_double] * 8 + [c_int, c_int, c_void_p]),
    ("b2_jde_destroy", None, [c_void_p]),
    ("b2_jde_set_cost_fn", c_int, [c_void_p, c_void_p, c_void_p]),
    ("b2_jde_reset", c_int, [c_void_p]),
    ("b2_jde_reset_ids", c_int, [c_void_p]),
    ("b2_jde_update", c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int]),
    ("b2_jde_get_tracks", c_int, [c_void_p, c_int, c_int] + [c_void_p] * 12),
    ("b2_reid_create", c_int, [POINTER(c_void_p), c_int, c_int, c_int]),
    ("b2_reid_create_model", c_int, [POINTER(c_void_p), c_int, c_int, c_int, c_int]),
    ("b2_reid_destroy", None, [c_void_p]),
    ("b2_reid_load_weights", c_int, [c_void_p, POINTER(c_char_p), POINTER(c_void_p), POINTER(c_int64), c_int]),
    ("b2_reid_embed", c_int, [c_void_p, c_void_p, c_int, c_void_p]),
    ("b2_reid_embed_dev", c_int, [c_void_p, c_void_p, c_int, c_void_p]),
    ("b2_reid_embed_boxes", c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_int, c_void_p]),
    ("b2_reid_embed_boxes_dev", c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_int, c_void_p]),
    ("b2_reid_feat_dim", c_int, [c_void_p]),
    ("b2_reid_num_launches", c_int, [c_void_p]),
    ("b2_reid_get_activation", c_int, [c_void_p, c_char_p, c_void_p, c_int64, POINTER(c_int64)]),
    ("b2_effdet_create", c_int, [POINTER(c_void_p), POINTER(B2EffdetConfig), c_int]),
    ("b2_effdet_destroy", None, [c_void_p]),
    ("b2_effdet_load_weights", c_int, [c_void_p, POINTER(c_char_p), POINTER(c_void_p), POINTER(c_int64), c_int]),
    ("b2_effdet_run_features", c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_float] + [c_void_p] * 6),
    ("b2_effdet_detect", c_int, [c_void_p, c_void_p, c_int, c_int] + [c_void_p] * 7),
    ("b2_effdet_detect_batch", c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int] + [c_void_p] * 7),
    ("b2_effdet_replay", c_int, [c_void_p, c_int, POINTER(c_float)]),
    ("b2_effdet_get_stage", c_int, [c_void_p, c_char_p, c_void_p, c_int64, POINTER(c_int64)]),
    ("b2_effdet_set_stage", c_int, [c_void_p, c_char_p, c_void_p, c_int64]),
    ("b2_effdet_run_phases", c_int, [c_void_p, c_int]),
    ("b2_effdet_num_launches", c_int, [c_void_p]),
    ("b2_effdet_profile_steps", c_int, [c_void_p, c_int, POINTER(c_float), c_int, POINTER(c_int)]),
    ("b2_effdet_step_info", c_int, [c_void_p, c_int, ctypes.c_char_p, c_int, POINTER(ctypes.c_double), POINTER(ctypes.c_double), POINTER(c_int)]),
    ("b2_distance_matrix", c_int, [c_int, c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    ("b2_track_pair_cost", c_int, [c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_void_p, c_float, c_int, c_void_p]),
    ("b2_track_pair_cost_dev", c_int, [c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_void_p, c_float, c_int, c_void_p]),
    ("b2_gallery_create", c_int, [c_int, c_void_p, c_int, c_int, POINTER(c_void_p), c_void_p]),
    ("b2_gallery_open", c_int, [c_int, c_void_p, POINTER(c_void_p)]),
    ("b2_gallery_close", c_int, [c_int, c_void_p]),
    ("b2_gallery_free", c_int, [c_int, c_void_p]),
    ("b2_track_spatial_dist", c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, ctypes.c_double, c_void_p]),
    ("b2_tracklet_dist_dev", c_int, [c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_void_p, c_int, c_int, c_int, c_void_p]),
    ("b2_op_conv2d", c_int, [c_int, c_void_p, c_void_p, c_void_p, c_void_p] + [c_int] * 18 + [c_void_p]),
    ("b2_op_conv2d_view", c_int, [c_int, POINTER(B2ConvView)] + [c_void_p] * 9),
    ("b2_op_group_norm", c_int, [c_int, c_void_p, c_void_p, c_void_p, c_void_p] + [c_int] * 15 + [c_void_p]),
    ("b2_op_squeeze_excite", c_int, [c_int] + [c_void_p] * 6 + [c_int] * 6 + [c_void_p, c_void_p]),
    ("b2_op_group_conv2d", c_int, [c_int, c_void_p, c_void_p, c_void_p, c_void_p] + [c_int] * 16 + [c_void_p]),
    ("b2_op_relation", c_int, [c_int] + [c_void_p] * 10 + [c_int] * 4 + [c_void_p]),
    ("b2_op_so_attend", c_int, [c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int] + [c_void_p] * 7
     + [c_int, c_int, c_void_p]),
    ("b2_op_mask_head", c_int, [c_int, c_void_p, c_void_p, c_void_p] + [c_int] * 3 + [c_void_p] * 3
     + [c_int, POINTER(c_char_p), POINTER(c_void_p), POINTER(c_int64), c_int, c_void_p, c_int] + [c_void_p] * 11),
    ("b2_op_att_pool", c_int, [c_int, c_void_p, c_int, c_int, c_int, c_void_p]),
    ("b2_op_deform_sample", c_int, [c_int, c_void_p, c_void_p] + [c_int] * 5 + [c_void_p]),
    ("b2_op_deform_conv2d", c_int, [c_int] + [c_void_p] * 4 + [c_int] * 7 + [c_void_p, c_void_p]),
    ("b2_op_depthwise", c_int, [c_int] + [c_void_p] * 3 + [c_int] * 13 + [c_void_p] * 3),
    ("b2_op_pool", c_int, [c_int, c_void_p] + [c_int] * 9 + [c_void_p] * 3),
    ("b2_op_bifpn_combine", c_int, [c_int] + [c_void_p] * 3 + [c_int] * 7 + [c_void_p] * 4),
    ("b2_op_mbconv_se", c_int, [c_int] + [c_void_p] * 6 + [c_int] * 7 + [c_void_p] * 4),
    ("b2_op_channel_gate", c_int, [c_int] + [c_void_p] * 6 + [c_int] * 6 + [c_void_p] * 4),
    ("b2_op_stem_im2col", c_int, [c_int, c_void_p] + [c_int] * 7 + [c_void_p] * 3),
    ("b2_op_stem_pack", c_int, [c_int, c_void_p] + [c_int] * 8 + [c_void_p] * 3),
    ("b2_op_reid_crop_resize", c_int, [c_int, c_void_p, c_int, c_int, c_int, c_void_p, c_int, c_int, c_int, c_void_p]),
    ("b2_op_distance_operand", c_int, [c_int, c_void_p] + [c_int] * 4 + [c_float] + [c_void_p] * 4),
    ("b2_op_distance_epilogue", c_int, [c_int, c_int, c_void_p] + [c_int] * 3 + [c_void_p] * 3 + [c_int, c_void_p, c_int,
                                                                                                c_void_p, c_float, c_void_p]),
]

PHASES = dict(BACKBONE=1, FPN=2, RPN_HEAD=4, PROPOSALS=8, ROI=16, HEAD_FC=32, POST=64, BOX_FEAT=128, ALL=255)
PHASE_NAMES = ["backbone", "fpn", "rpn_head", "proposals", "roi", "head_fc", "post", "box_feat"]
EFFDET_PHASES = dict(BACKBONE=1, FEATURES=2, POST=4, BOX_FEAT=8)

_lib = None


def load(build_if_missing: bool = True) -> ctypes.CDLL:
    """Load (building in-tree if needed) libb200det.so and declare all prototypes."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        if not build_if_missing:
            raise RuntimeError("libb200det.so is not built: run `python -m object_detection_tracking_b200.build`")
        from . import build as _build
        _build.build()
    lib = ctypes.CDLL(LIB_PATH)
    for name, res, args in SYMBOLS:
        fn = getattr(lib, name)          # AttributeError if the export is missing
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc: int, what: str = "libb200det"):
    if rc != 0:
        msg = load().b2_last_error()
        raise RuntimeError("%s failed: %s" % (what, msg.decode() if msg else "unknown error"))


def ptr(a) -> c_void_p:
    """Raw pointer of a numpy array / torch tensor / None."""
    if a is None:
        return c_void_p(0)
    if isinstance(a, np.ndarray):
        return c_void_p(a.ctypes.data)
    return c_void_p(a.data_ptr())          # torch.Tensor


def make_config(cfg, batch: int, height: int, width: int, input_dtype: str = "float32", precision: str = "split",
                conv_impl: str = "tcgen05", use_cuda_graph: bool = True, multi_semantics: bool = False,
                accum_chunk: int = 0) -> B2Config:
    """Translate the reference-style namespace (config.py / obj_detect_tracking.py:236-389)."""
    c = B2Config()
    c.batch, c.height, c.width = int(batch), int(height), int(width)
    c.input_dtype = {"float32": 0, "uint8": 1}[input_dtype]
    c.num_class = int(cfg.num_class)
    for i, v in enumerate(cfg.resnet_num_block):
        c.resnet_blocks[i] = int(v)
    c.use_dilations = int(bool(cfg.use_dilations))
    c.class_agnostic = int(bool(getattr(cfg, "use_frcnn_class_agnostic", False)))
    c.rpn_topk = int(cfg.rpn_test_post_nms_topk)
    c.result_per_im = int(cfg.result_per_im)
    c.fpn_num_channel = int(cfg.fpn_num_channel)
    c.fc_head_dim = int(cfg.fpn_frcnn_fc_head_dim)
    c.precision = {"fp16": 0, "split": 1}[precision]
    c.conv_impl = {"tcgen05": 0, "simt": 1}[conv_impl]
    c.use_cuda_graph = int(bool(use_cuda_graph))
    c.max_size = float(cfg.max_size)
    c.rpn_min_size = float(cfg.rpn_min_size)
    c.rpn_nms_thres = float(cfg.rpn_proposal_nms_thres)
    c.fastrcnn_nms_iou_thres = float(cfg.fastrcnn_nms_iou_thres)
    c.result_score_thres = float(cfg.result_score_thres)
    for i in range(5):
        c.anchor_strides[i] = float(cfg.anchor_strides[i])
        c.anchor_sizes[i] = float(cfg.anchor_sizes[i])
    for i in range(3):
        c.anchor_ratios[i] = float(cfg.anchor_ratios[i])
    for i in range(4):
        c.bbox_reg_weights[i] = float(cfg.fastrcnn_bbox_reg_weights[i])
    c.multi_semantics = int(bool(multi_semantics))
    c.accum_chunk = int(accum_chunk)
    c.add_mask = int(bool(getattr(cfg, "add_mask", False)))
    c.use_gn = int(bool(getattr(cfg, "use_gn", False)))
    c.conv_head_dim = int(getattr(cfg, "conv_frcnn_head_dim", 256)) if getattr(cfg, "use_conv_frcnn_head", False) else 0
    c.use_se = int(bool(getattr(cfg, "use_se", False)))
    c.use_resnext = int(bool(getattr(cfg, "use_resnext", False)))
    c.add_relation_nn = int(bool(getattr(cfg, "add_relation_nn", False)))
    c.use_deformable = int(bool(getattr(cfg, "use_deformable", False)))
    return c


def make_config_ext(cfg) -> B2ConfigExt:
    """The options of the namespace that b2_config_ext carries."""
    e = B2ConfigExt()
    e.use_basic_block = int(bool(getattr(cfg, "use_basic_block", False)))
    return e


def make_config_ext2(cfg) -> B2ConfigExt2:
    """The options of the namespace that b2_config_ext2 carries: the partial class ids (config.normalize_config resolves
    and checks them; () = off)."""
    e = B2ConfigExt2()
    ids = tuple(getattr(cfg, "partial_class_ids", ()))
    if len(ids) > 80:
        raise ValueError("at most 80 partial classes, got %d" % len(ids))
    e.num_partial_classes = len(ids)
    for i, v in enumerate(ids):
        e.partial_class_ids[i] = int(v)
    return e


def make_config_ext3(cfg) -> B2ConfigExt3:
    """The options of the namespace that b2_config_ext3 carries."""
    e = B2ConfigExt3()
    e.use_att_frcnn_head = int(bool(getattr(cfg, "use_att_frcnn_head", False)))
    return e


def make_config_ext4(cfg) -> B2ConfigExt4:
    """The options of the namespace that b2_config_ext4 carries (the small-object branch; all 0 when it is off)."""
    e = B2ConfigExt4()
    if not getattr(cfg, "use_small_object_head", False):
        return e
    ids = tuple(cfg.small_object_class_ids)
    if len(ids) > 80:
        raise ValueError("use_small_object_head: at most 80 small objects, got %d" % len(ids))
    e.use_small_object_head = 1
    e.num_small_objects = len(ids)
    for i, v in enumerate(ids):
        e.small_object_class_ids[i] = int(v)
    e.use_so_association = int(bool(cfg.use_so_association))
    e.so_person_class_id = int(cfg.so_person_class_id)
    e.so_person_topk = int(cfg.so_person_topk)
    e.use_so_score_thres = int(bool(cfg.use_so_score_thres))
    return e


def make_config_ext5(cfg) -> B2ConfigExt5:
    """The options of the namespace that b2_config_ext5 carries."""
    e = B2ConfigExt5()
    e.use_bg_score = int(bool(getattr(cfg, "use_bg_score", False)))
    return e
