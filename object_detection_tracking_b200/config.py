"""Model configuration namespace for the detect hot path.

Mirrors the derived-constant block of the reference CLI
(`obj_detect_tracking.py:236-389`): the reference passes its argparse namespace
straight into `models.get_model(config, ...)`, so the drop-in backend accepts an
object with the same attribute names.  `make_config()` builds such a namespace
without argparse; `normalize_config()` fills anything a caller left out.
"""
from __future__ import annotations

import math
from types import SimpleNamespace

import numpy as np

# obj_detect_tracking.py:327-387 -- fixed hyper-parameters of the inference graph
_DEFAULTS = dict(
    num_class=15,                      # obj_detect_tracking.py:122 (ActEV 15-class incl. BG)
    version=3,                         # --version 3  => use_dilations (:270-271)
    use_dilations=True,
    use_frcnn_class_agnostic=False,
    resnet_num_block=(3, 4, 23, 3),    # :348 ResNet-101
    short_edge_size=720,
    max_size=1280,
    rpn_test_post_nms_topk=300,
    rpn_min_size=0,
    rpn_proposal_nms_thres=0.7,
    anchor_strides=(4, 8, 16, 32, 64),
    anchor_sizes=(32, 64, 128, 256, 512),
    anchor_ratios=(0.5, 1.0, 2.0),
    fpn_num_channel=256,
    fpn_frcnn_fc_head_dim=1024,
    fastrcnn_bbox_reg_weights=(10.0, 10.0, 5.0, 5.0),
    fastrcnn_nms_iou_thres=0.5,
    threshold_conf=1e-4,               # -> result_score_thres (:385)
    result_per_im=100,
    im_batch_size=1,
    is_train=False,
    add_mask=False,
    mrcnn_head_dim=256,                # obj_detect_tracking.py:324
    use_gn=False,                      # --use_gn (obj_detect_tracking.py:101-102): GroupNorm backbone + FPN
    use_conv_frcnn_head=False,         # --use_conv_frcnn_head (:103-104): 4-conv box head
    conv_frcnn_head_dim=256,           # only main.py:250 sets it (default 256); the inference drivers never do
    use_se=False,                      # --use_se (obj_detect_tracking.py:192-193; set by --version 6, :278-280):
                                       # squeeze-excite in every bottleneck (nn.py:506-519)
    use_resnext=False,                 # --use_resnext (obj_detect_tracking.py:196): ResNeXt 32x4d blocks with grouped
                                       # 3x3 convs (nn.py:524-549, 864-868); the block has no SE branch
    add_relation_nn=False,             # --add_relation_nn (obj_detect_tracking.py:226): relation modules RM_r1 / RM_r2 in
                                       # the 2fc box head (models.py:1044-1054, nn.py:115-190); not with the conv head
    use_deformable=False,              # --use_deformable (obj_detect_tracking.py:215): deformable conv2 in the stride-2
                                       # blocks among the last 3 of a group (nn.py:459-521, 568-588): res5 block 0 of
                                       # R50 / R101; ignored with use_resnext, refused with use_dilations
    use_basic_block=False,             # set by --resnet34 / --resnet18 (obj_detect_tracking.py:349-359): resnet_basicblock
                                       # (nn.py:439-456) instead of the bottleneck; use_resnext wins (nn.py:864-868);
                                       # the block ignores use_dilations, use_deformable and use_se
    use_partial_classes=False,         # --use_partial_classes (obj_detect_tracking.py:233-239): a COCO-81 checkpoint whose
                                       # box head keeps only partial_classes (models.py:807-828); labels become 1..C
    partial_classes=None,              # class names, in output-label order; None = the keys of coco_obj_to_actev_obj
    use_att_frcnn_head=False,          # --use_att_frcnn_head (obj_detect_tracking.py:197-199): hidden + relu(att_trans(sum
                                       # of the ROI's 49 cells)) in the class-specific box head (models.py:1064-1089); the
                                       # class-agnostic heads have no attention branch (models.py:1126-1170)
    use_small_object_head=False,       # main.py --use_small_object_head (:263): the per-class small-object branch of the
                                       # single-image graph (models.py:590-692, 845-897), outputs so_final_*
    use_so_association=False,          # --use_so_association (:273): person_object_relation on the branch's rows
    use_so_score_thres=False,          # --use_so_score_thres (:264): the branch's final NMS filters logit > thres
    so_person_topk=10,                 # --so_person_topk (:274): reference person boxes of the association
    small_objects=None,                # class names, in so label order; None = class_ids.SMALL_OBJECTS (main.py:506-507)
    use_bg_score=False,                # main.py --use_bg_score (:171): the single-image graph's fastrcnn_predictions drops the
                                       # ROIs whose argmax is background before its NMS (models.py:1263-1270); the batch
                                       # graph ignores it
    use_cpu_nms=False,                 # main.py --use_cpu_nms, set by --no_nms / --save_all_box (:493-497): the single-image
                                       # graph returns every proposal's boxes and probabilities of every class instead of
                                       # the NMS outputs (models.py:899-916)
    is_efficientdet=False,
)

# (flag, resnet_num_block, use_basic_block) of the backbone flags, in the order obj_detect_tracking.py:350-359 applies them
_BACKBONE_FLAGS = (("resnet152", (3, 8, 36, 3), False), ("resnet50", (3, 4, 6, 3), False),
                   ("resnet34", (3, 4, 6, 3), True), ("resnet18", (2, 2, 2, 2), True))


def make_config(**overrides) -> SimpleNamespace:
    cfg = dict(_DEFAULTS)
    cfg.update(overrides)
    return normalize_config(SimpleNamespace(**cfg))


def normalize_config(cfg):
    """Fill derived fields exactly as obj_detect_tracking.py:320-387 does."""
    for k, v in _DEFAULTS.items():
        if not hasattr(cfg, k):
            setattr(cfg, k, v)
    # :348-359: the flags apply in this order, so with several set the last one's blocks win, and the basic block is used
    # iff --resnet34 or --resnet18 is set; without any flag the blocks and use_basic_block are what the caller gave
    flags = [f for f in _BACKBONE_FLAGS if getattr(cfg, f[0], False)]
    if flags:
        cfg.resnet_num_block = flags[-1][1]
        cfg.use_basic_block = any(basic for _, _, basic in flags)
    cfg.resnet_num_block = tuple(int(x) for x in cfg.resnet_num_block)
    cfg.fpn_resolution_requirement = float(cfg.anchor_strides[3])   # :323
    # :330-331  max_size rounded up to a multiple of 32
    cfg.max_size = float(np.ceil(cfg.max_size / cfg.fpn_resolution_requirement)
                         * cfg.fpn_resolution_requirement)
    cfg.bbox_decode_clip = float(np.log(cfg.max_size / 16.0))        # :370
    cfg.result_score_thres = float(cfg.threshold_conf)               # :385
    cfg.num_anchors_per_loc = len(cfg.anchor_ratios)
    cfg.partial_class_ids = _partial_class_ids(cfg)
    _small_object_ids(cfg)
    return cfg


def _small_object_ids(cfg):
    """With use_small_object_head: cfg.small_object_class_ids (the head's class ids of small_objects, in order) and, with
    use_so_association, cfg.so_person_class_id.  Names resolve through config.classname2id when the caller set it, as the
    reference does (models.py:604-605, 647), else through the merge-prop table the reference's main.py asserts
    (main.py:508-521).  Off: () and 0."""
    from .class_ids import SMALL_OBJECTS, targetClass2id_mergeProp
    cfg.small_object_class_ids = ()
    cfg.so_person_class_id = 0
    if not cfg.use_small_object_head or cfg.is_efficientdet:
        return
    if cfg.small_objects is None:
        cfg.small_objects = list(SMALL_OBJECTS)
    table = getattr(cfg, "classname2id", None) or targetClass2id_mergeProp
    names = list(cfg.small_objects)
    nc = int(cfg.num_class)

    def resolve(n):
        if n == "BG":
            raise ValueError("use_small_object_head: 'BG' cannot be a small object")
        if n not in table:
            raise ValueError("use_small_object_head: %r is not a class name of classname2id" % (n,))
        i = int(table[n])
        if not 1 <= i <= nc - 1:
            raise ValueError("use_small_object_head: %r has id %d, outside 1..num_class-1 (num_class %d)" % (n, i, nc))
        return i

    if not names:
        raise ValueError("use_small_object_head: small_objects is empty")
    dup = sorted({n for n in names if names.count(n) > 1})
    if dup:
        raise ValueError("use_small_object_head: %s listed more than once" % ", ".join(repr(n) for n in dup))
    for flag, why in (("use_frcnn_class_agnostic", "the reference's decode reshapes [N,1,4] box logits against "
                       "[N,num_class-1,4] anchors and fails"),
                      ("use_partial_classes", "the branch reads the full head's class columns"),
                      ("use_conv_frcnn_head", "the branch would need its own fc6 / fc7 next to fastrcnn/fc")):
        if getattr(cfg, flag, False):
            raise ValueError("use_small_object_head cannot be combined with %s: %s" % (flag, why))
    cfg.small_object_class_ids = tuple(resolve(n) for n in names)
    if cfg.use_so_association:
        if "Person" not in table:
            raise ValueError("use_so_association needs a 'Person' class in classname2id (models.py:647)")
        cfg.so_person_class_id = resolve("Person")
        if int(cfg.so_person_topk) < 1:
            raise ValueError("use_so_association: so_person_topk must be >= 1, got %d" % int(cfg.so_person_topk))


def _partial_class_ids(cfg) -> tuple:
    """The COCO class ids the box head keeps with use_partial_classes, in partial_classes order (models.py:807-811); ()
    when it is off.  EfficientDet resolves its own selection (backend.EfficientDet).

    The ids are always coco_obj_class_to_id[name]: what the published frozen partial model computes (main.py:562-566
    packed it with the COCO table).  config.classname2id is not read: the checkpoint driver overwrites it with the partial
    table (obj_detect_tracking.py:287-300), under which the same gather would pick the first len(partial_classes) COCO
    classes instead."""
    from .class_ids import coco_obj_class_to_id, coco_obj_to_actev_obj
    if not cfg.use_partial_classes or cfg.is_efficientdet:
        return ()
    if cfg.partial_classes is None:
        cfg.partial_classes = list(coco_obj_to_actev_obj)
    names = list(cfg.partial_classes)
    if int(cfg.num_class) != 81:
        raise ValueError("use_partial_classes selects classes of a COCO model: num_class must be 81, got %d"
                         % int(cfg.num_class))
    if not names:
        raise ValueError("use_partial_classes: partial_classes is empty")
    for n in names:
        if n == "BG":
            raise ValueError("use_partial_classes: 'BG' cannot be selected (the background column is always kept)")
        if n not in coco_obj_class_to_id:
            raise ValueError("use_partial_classes: %r is not a COCO class name" % (n,))
    dup = sorted({n for n in names if names.count(n) > 1})
    if dup:
        raise ValueError("use_partial_classes: %s selected more than once" % ", ".join(repr(n) for n in dup))
    return tuple(coco_obj_class_to_id[n] for n in names)


def backbone_geometry(h: int, w: int, cfg):
    """Feature-map sizes for an (h, w) input, from the padding rules of
    `nn.py:843-944` (tf_pad_reverse=True) and the crop of `models.py:372-400`.

    Returns dict with c1, pool, c2..c5 (H, W), p2..p6 full sizes and the cropped
    p2..p6 sizes the RPN / ROIAlign see.
    """
    mult = int(cfg.fpn_resolution_requirement)
    ph = int(math.ceil(h / mult) * mult)
    pw = int(math.ceil(w / mult) * mult)
    # pad [3, 2 + pad_to_32], conv 7x7 s2 VALID
    ih, iw = ph + 5, pw + 5
    c1 = ((ih - 7) // 2 + 1, (iw - 7) // 2 + 1)
    # pad [1, 0], maxpool 3x3 s2 VALID
    pool = ((c1[0] + 1 - 3) // 2 + 1, (c1[1] + 1 - 3) // 2 + 1)
    c2 = pool
    def down(s):  # stride-2 group: pad [1,0] + 3x3 s2 VALID (dilated variant pads again)
        return ((s[0] + 1 - 3) // 2 + 1, (s[1] + 1 - 3) // 2 + 1)
    c3 = down(c2)
    c4 = down(c3)
    c5 = down(c4)
    full = [c2, c3, c4, c5, ((c5[0] - 1) // 2 + 1, (c5[1] - 1) // 2 + 1)]
    crop = []
    for i, s in enumerate(cfg.anchor_strides):
        if i < 3:
            crop.append((min(full[i][0], int(math.ceil(h / float(s)))),
                         min(full[i][1], int(math.ceil(w / float(s))))))
        else:
            crop.append(full[i])
    return dict(padded=(ph, pw), c1=c1, pool=pool, c=[c2, c3, c4, c5], p_full=full, p=crop)
