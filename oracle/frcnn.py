"""ORACLE (test infrastructure only -- the product path never imports this).

CPU fp32 restatement of the inference branch of the reference's `Mask_RCNN_FPN`
(models.py:266-1304) and the `nn.py` layers it calls, stage-addressable.  The reference
graph is TensorFlow-1.15 (absent here, see oracle/tf_ops.py) => **parity unpinned** for the
TF op arithmetic; the graph structure, padding rules, constants and orderings below are
restated line by line with citations.  Convolutions run through torch.nn.functional.conv2d
in float32 on the host CPU (this is also the `cpu_baseline` the bench reports).
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

from . import tf_ops
from .anchors import get_all_anchors

BN_EPS = 1e-5            # nn.py:1723


# Arithmetic type of the conv / matmul stack.  float32 is the reference's (and the default).  `exact()` switches it to
# float64: the same graph evaluated without fp32 rounding noise -- the centre any two float32 implementations (TF's Eigen
# kernels, this torch port, the GPU path) scatter around.  Tests use it to split |GPU - oracle32| into the GPU's own
# error and the oracle's.  Post-processing (decode, top-k, NMS, ROIAlign) stays float32 in both modes: the stack's
# outputs are rounded once to float32 at the hand-over (`_np`).
_DT = [torch.float32]


class exact(object):
    def __enter__(self):
        _DT.append(torch.float64)

    def __exit__(self, *a):
        _DT.pop()


def _t(a):
    t = torch.from_numpy(np.ascontiguousarray(a))
    return t.to(_DT[-1]) if t.is_floating_point() else t


def _np(t):
    return t.to(torch.float32).numpy()


def _conv(x, w_hwio, stride=1, dilation=1, pad=(0, 0, 0, 0), bias=None):
    """nn.conv2d (nn.py:337-381): HWIO kernel, explicit pad = (top, bottom, left, right)."""
    wt = _t(w_hwio).permute(3, 2, 0, 1).contiguous()
    if any(pad):
        x = F.pad(x, (pad[2], pad[3], pad[0], pad[1]))
    return F.conv2d(x, wt, None if bias is None else _t(bias), stride=stride, dilation=dilation)


def _same_pad(k, dil):
    p = (k - 1) * dil // 2          # stride-1 SAME: symmetric (Appendix B)
    return (p, p, p, p)


def _bn(x, W, name):
    """BatchNorm inference (nn.py:1771-1774): tf.nn.batch_normalization =
    (x - mean) * rsqrt(var + eps) * gamma + beta."""
    g = _t(W[name + "/bn/gamma"]); b = _t(W[name + "/bn/beta"])
    m = _t(W[name + "/bn/mean/EMA"]); v = _t(W[name + "/bn/variance/EMA"])
    inv = torch.rsqrt(v + BN_EPS) * g
    return x * inv.view(1, -1, 1, 1) + (b - m * inv).view(1, -1, 1, 1)


def preprocess(img_hwc_f32: np.ndarray) -> torch.Tensor:
    """models.py:337-357: /255, -mean[::-1], /std[::-1] (BGR), HWC->NCHW."""
    x = _t(np.asarray(img_hwc_f32, dtype=np.float32)).unsqueeze(0)
    mean = torch.tensor([0.485, 0.456, 0.406][::-1], dtype=torch.float32).to(_DT[-1])
    std = torch.tensor([0.229, 0.224, 0.225][::-1], dtype=torch.float32).to(_DT[-1])
    x = x * (1.0 / 255)
    x = (x - mean) / std
    return x.permute(0, 3, 1, 2).contiguous()


def bottleneck(x, W, p, ch, stride, dil):
    """resnet_bottleneck (nn.py:459-521) with tf_pad_reverse=True, + shortcut (nn.py:551-566),
    + trailing relu (resnet_group nn.py:586-587)."""
    sc = x
    l = torch.relu(_bn(_conv(x, W[p + "/conv1/W"]), W, p + "/conv1"))
    if stride == 2:
        # pad [1,0] (reverse of [0,1]) then 3x3 stride-2 VALID (nn.py:487-492)
        l = _conv(l, W[p + "/conv2/W"], stride=2, dilation=dil, pad=(1, 0, 1, 0))
        l = torch.relu(_bn(l, W, p + "/conv2"))
        if dil != 1:
            l = F.pad(l, (1, 0, 1, 0))           # nn.py:493-497 pads again after the conv
    else:
        l = _conv(l, W[p + "/conv2/W"], dilation=dil, pad=_same_pad(3, dil))
        l = torch.relu(_bn(l, W, p + "/conv2"))
    l = _bn(_conv(l, W[p + "/conv3/W"]), W, p + "/conv3")
    if (p + "/convshortcut/W") in W:
        if stride == 2:
            sc = sc[:, :, :-1, :-1]              # nn.py:555-556
            sc = _conv(sc, W[p + "/convshortcut/W"], stride=2)
        else:
            sc = _conv(sc, W[p + "/convshortcut/W"])
        sc = _bn(sc, W, p + "/convshortcut")
    return torch.relu(l + sc)


def backbone(x, W, cfg):
    """resnet_fpn_backbone (nn.py:843-944)."""
    h, w = x.shape[2:]
    mult = cfg.fpn_resolution_requirement
    ph = int(math.ceil(h / mult) * mult) - h
    pw = int(math.ceil(w / mult) * mult) - w
    l = F.pad(x, (3, 2 + pw, 3, 2 + ph))          # pad_base reversed = [3,2] (nn.py:871-877)
    l = torch.relu(_bn(_conv(l, W["conv0/W"], stride=2), W, "conv0"))
    l = F.pad(l, (1, 0, 1, 0))                     # nn.py:892-894
    l = F.max_pool2d(l, 3, 2)                      # VALID
    feats = []
    for g, (ch, count) in enumerate(zip((64, 128, 256, 512), cfg.resnet_num_block)):
        for i in range(count):
            stride = 2 if (g > 0 and i == 0) else 1
            # dilation only in group3, on its last 3 blocks (nn.py:577-581, 932-936)
            dil = 2 if (g == 3 and cfg.use_dilations and i in range(count)[-3:]) else 1
            l = bottleneck(l, W, "group%d/block%d" % (g, i), ch, stride, dil)
        feats.append(l)
    return feats


def fpn(c2345, W):
    """fpn_model (nn.py:947-1014)."""
    lat = [_conv(c, W["fpn/lateral_1x1_c%d/W" % (i + 2)], bias=W["fpn/lateral_1x1_c%d/b" % (i + 2)])
           for i, c in enumerate(c2345)]
    sums = []
    for idx, l in enumerate(lat[::-1]):
        if idx > 0:
            up = sums[-1].repeat_interleave(2, dim=2).repeat_interleave(2, dim=3)
            l = l + up
        sums.append(l)
    p2345 = [_conv(c, W["fpn/posthoc_3x3_p%d/W" % (i + 2)], pad=(1, 1, 1, 1),
                   bias=W["fpn/posthoc_3x3_p%d/b" % (i + 2)])
             for i, c in enumerate(sums[::-1])]
    p6 = p2345[-1][:, :, ::2, ::2]                 # 1x1 max-pool stride 2 VALID (nn.py:1010-1012)
    return p2345 + [p6]


def rpn_head(p, W, na):
    """rpn_head (models.py:979-1009) -> logits [H,W,A], box [H,W,A,4]."""
    h = torch.relu(_conv(p, W["rpn/conv0/W"], pad=(1, 1, 1, 1), bias=W["rpn/conv0/b"]))
    cls = _conv(h, W["rpn/class/W"], bias=W["rpn/class/b"])
    box = _conv(h, W["rpn/box/W"], bias=W["rpn/box/b"])
    cls = _np(cls[0].permute(1, 2, 0).contiguous())
    box = _np(box[0].permute(1, 2, 0).contiguous())
    return cls, box.reshape(box.shape[0], box.shape[1], na, 4)


def decode_bbox_target(box_pred, anchors, decode_clip=np.log(1333 / 16.0)):
    """decode_bbox_target (nn.py:1518-1538), float32."""
    f32 = np.float32
    bp = np.asarray(box_pred, dtype=f32).reshape(-1, 4)
    an = np.asarray(anchors, dtype=f32).reshape(-1, 4)
    waha = (an[:, 2:] - an[:, :2]).astype(f32)
    xaya = ((an[:, 2:] + an[:, :2]).astype(f32) * f32(0.5)).astype(f32)
    wbhb = (np.exp(np.minimum(bp[:, 2:], f32(decode_clip)).astype(f32)).astype(f32) * waha).astype(f32)
    xbyb = ((bp[:, :2] * waha).astype(f32) + xaya).astype(f32)
    x1y1 = (xbyb - (wbhb * f32(0.5)).astype(f32)).astype(f32)
    x2y2 = (xbyb + (wbhb * f32(0.5)).astype(f32)).astype(f32)
    return np.concatenate([x1y1, x2y2], axis=-1).reshape(np.asarray(anchors).shape)


def clip_boxes(boxes, hw):
    """clip_boxes (nn.py:1339-1346): max(.,0) then min(., [W,H,W,H])."""
    m = np.array([hw[1], hw[0], hw[1], hw[0]], dtype=np.float32)
    return np.minimum(np.maximum(boxes, np.float32(0)), m).astype(np.float32)


def generate_rpn_proposals(boxes, scores, hw, cfg, topk):
    """generate_rpn_proposals (nn.py:1353-1400) for one FPN level."""
    sc, idx = tf_ops.top_k(scores, min(topk, scores.shape[0]))
    b = clip_boxes(boxes[idx], hw)
    wh = b[:, 2:] - b[:, :2]
    valid = np.all(wh > cfg.rpn_min_size, axis=1)
    b = b[valid]; sc = sc[valid]
    keep = tf_ops.non_max_suppression(b[:, [1, 0, 3, 2]], sc, topk, cfg.rpn_proposal_nms_thres)
    return b[keep], sc[keep]


def level_proposals(cfg, level, cls, box, hw, multi=False):
    """The proposals of one FPN level from its RPN outputs cls [fh,fw,A], box [fh,fw,A,4]: anchors, decode, then
    generate_rpn_proposals (single-image graph) or, with `multi`, the batch graph's top-k + clip + hard NMS without the
    min-size filter (nn.py:1431-1474).  Returns the kept (boxes [n,4], scores [n]) in selection order."""
    fh, fw = cls.shape[:2]
    anchors = get_all_anchors(cfg.anchor_strides[level], [cfg.anchor_sizes[level]], cfg.anchor_ratios,
                              cfg.max_size)[:fh, :fw]
    dec = decode_bbox_target(box, anchors, cfg.bbox_decode_clip).reshape(-1, 4)     # nn.py:1486-1514
    K = cfg.rpn_test_post_nms_topk
    if not multi:
        return generate_rpn_proposals(dec, cls.reshape(-1), hw, cfg, K)
    sc, idx = tf_ops.top_k(cls.reshape(-1), min(K, cls.size))                        # nn.py:1431
    bx = clip_boxes(dec[idx], hw)                                                      # no min-size filter (:1441-1455)
    ob, os_, n = combined_nms_single_class(bx, sc, K, cfg.rpn_proposal_nms_thres)
    return ob[:n], os_[:n]


def merge_level_proposals(levels, topk):
    """generate_fpn_proposals (models.py:425-434), single-image graph: concatenate the levels' (boxes, scores) in level
    order and keep the top-k by score (ties -> lower concatenated position)."""
    pb = np.concatenate([b for b, _ in levels], 0); ps = np.concatenate([s for _, s in levels], 0)
    ps, ti = tf_ops.top_k(ps, min(ps.shape[0], topk))
    return pb[ti], ps


def merge_level_proposals_multi(levels, topk):
    """The batch graph's merge (models.py:2490-2520): every level zero-padded to topk (box 0, score 0), top-k by score --
    so the padding outranks negative logits --, then zero-area boxes dropped."""
    cb = np.zeros((len(levels) * topk, 4), np.float32); cs = np.zeros((len(levels) * topk,), np.float32)
    for i, (b, s) in enumerate(levels):
        cb[i * topk:i * topk + len(s)] = b; cs[i * topk:i * topk + len(s)] = s
    ps, ti = tf_ops.top_k(cs, min(cs.shape[0], topk))
    pb = cb[ti]
    area = ((pb[:, 3] - pb[:, 1]) * (pb[:, 2] - pb[:, 0])).astype(np.float32)
    keep = area > 0                                                                    # models.py:2516-2520
    return pb[keep], ps[keep]


def fpn_map_rois_to_levels(boxes):
    """models.py:439-461: level = floor(4 + log(sqrt(area)/224 + 1e-6)/log 2), clamp 2..5."""
    f32 = np.float32
    area = ((boxes[:, 3] - boxes[:, 1]).astype(f32) * (boxes[:, 2] - boxes[:, 0]).astype(f32)).astype(f32)
    sq = np.sqrt(area).astype(f32)
    lvl = np.floor(f32(4) + (np.log((sq * f32(1.0 / 224)).astype(f32) + f32(1e-6)).astype(f32)
                             * f32(1.0 / np.log(2))).astype(f32)).astype(np.int32)
    return np.clip(lvl, 2, 5)


def roi_align(feat_chw: np.ndarray, boxes_fm: np.ndarray, out: int) -> np.ndarray:
    """roi_align (nn.py:1326-1335) = crop_and_resize(2*out) with transform_fpcoor_for_tf
    (nn.py:1229-1280) + 2x2 avg-pool.  Returns [K, C, out, out]."""
    f32 = np.float32
    C, H, W = feat_chw.shape
    crop = out * 2
    x0, y0, x1, y1 = [boxes_fm[:, i].astype(f32) for i in range(4)]
    # a 1-pixel level divides by W - 1 = 0 here (NaN / inf box): tf_ops.crop_and_resize defines that axis
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        sw = ((x1 - x0) / f32(crop)).astype(f32)
        sh = ((y1 - y0) / f32(crop)).astype(f32)
        nx0 = ((x0 + sw / f32(2) - f32(0.5)) / f32(W - 1)).astype(f32)
        ny0 = ((y0 + sh / f32(2) - f32(0.5)) / f32(H - 1)).astype(f32)
        nw = (sw * f32(crop - 1) / f32(W - 1)).astype(f32)
        nh = (sh * f32(crop - 1) / f32(H - 1)).astype(f32)
        nb = np.stack([ny0, nx0, ny0 + nh, nx0 + nw], axis=1).astype(f32)
    r = tf_ops.crop_and_resize(np.ascontiguousarray(feat_chw.transpose(1, 2, 0)), nb, crop)
    r = r.reshape(r.shape[0], out, 2, out, 2, C)
    # tf.nn.avg_pool 2x2: sum of 4 * 0.25 (Eigen mean reducer: sum then divide)
    r = ((r[:, :, 0, :, 0] + r[:, :, 0, :, 1] + r[:, :, 1, :, 0] + r[:, :, 1, :, 1]) / f32(4)).astype(f32)
    return np.ascontiguousarray(r.transpose(0, 3, 1, 2))


def multilevel_roi_align(p2345, boxes, out, strides):
    """multilevel_roi_align (models.py:465-485); p2345 are numpy [C,H,W] (cropped levels)."""
    lvl = fpn_map_rois_to_levels(boxes)
    res = np.zeros((boxes.shape[0], p2345[0].shape[0], out, out), dtype=np.float32)
    for i in range(4):
        ids = np.where(lvl == i + 2)[0]
        if len(ids):
            bf = (boxes[ids] * np.float32(1.0 / strides[i])).astype(np.float32)
            res[ids] = roi_align(p2345[i], bf, out)
    return res, lvl


def fastrcnn_head(feat, W, cfg):
    """fastrcnn_2fc_head (models.py:1030-1108): NCHW flatten -> fc6 relu -> fc7 relu ->
    class [K,C], box [K,C,4][:,1:]."""
    x = _t(feat.reshape(feat.shape[0], -1))
    h = torch.relu(x @ _t(W["fastrcnn/fc6/W"]) + _t(W["fastrcnn/fc6/b"]))
    h = torch.relu(h @ _t(W["fastrcnn/fc7/W"]) + _t(W["fastrcnn/fc7/b"]))
    cls = _np(h @ _t(W["fastrcnn/outputs/class/W"]) + _t(W["fastrcnn/outputs/class/b"]))
    box = _np(h @ _t(W["fastrcnn/outputs/box/W"]) + _t(W["fastrcnn/outputs/box/b"]))
    box = box.reshape(box.shape[0], -1, 4)
    if not cfg.use_frcnn_class_agnostic:
        box = box[:, 1:, :]
    else:
        box = np.tile(box, (1, cfg.num_class - 1, 1))     # models.py:799-802
    return cls, np.ascontiguousarray(box), _np(h)


def softmax(x):
    m = x.max(axis=1, keepdims=True)
    e = np.exp((x - m).astype(np.float32)).astype(np.float32)
    return (e / e.sum(axis=1, keepdims=True, dtype=np.float32)).astype(np.float32)


def fastrcnn_predictions(boxes, probs, cfg):
    """fastrcnn_predictions (models.py:1258-1304) + nms_return_masks (:1202-1223).
    boxes [K,C-1,4], probs [K,C].  Returns (pred_indices [R,2]=(box_id, class_id), probs [R])
    in canonical order (prob descending; ties -> (class, box) ascending, i.e. the order of
    tf.where(masks) on the [C-1,K] mask)."""
    K = boxes.shape[0]
    nc1 = boxes.shape[1]
    sel = []
    for c in range(nc1):
        p = probs[:, c + 1]
        ids = np.where(p > np.float32(cfg.result_score_thres))[0]
        keep = tf_ops.non_max_suppression(boxes[ids, c], p[ids], cfg.result_per_im,
                                          cfg.fastrcnn_nms_iou_thres)
        for k in sorted(ids[keep].tolist()):
            sel.append((c, k))
    if not sel:
        return np.zeros((0, 2), np.int64), np.zeros((0,), np.float32)
    sel = np.asarray(sel, dtype=np.int64)
    pr = probs[sel[:, 1], sel[:, 0] + 1]
    tp, ti = tf_ops.top_k(pr, min(cfg.result_per_im, pr.shape[0]))
    return sel[ti][:, ::-1].copy(), tp


def fastrcnn_predictions_multi(boxes, probs, cfg):
    """The batch graph's combined NMS over classes (models.py:2924-2976): per class hard NMS (<= result_per_im), no score
    threshold, merge, sort by score, keep result_per_im.  Canonical tie order: (class, selection order).  Same returns
    as fastrcnn_predictions."""
    R = cfg.result_per_im
    cand = []
    for c in range(boxes.shape[1]):
        keep = tf_ops.non_max_suppression(boxes[:, c], probs[:, c + 1], R, cfg.fastrcnn_nms_iou_thres)
        cand += [(int(k), c) for k in keep]
    if not cand:
        return np.zeros((0, 2), np.int64), np.zeros((0,), np.float32)
    cand = np.asarray(cand, dtype=np.int64)
    sc = probs[cand[:, 0], cand[:, 1] + 1].astype(np.float32)
    tp, ti = tf_ops.top_k(sc, min(R, len(cand)))
    return cand[ti], tp


def head_postprocess(cls_logits, box_logits, proposals, hw, cfg, multi=False):
    """Inference decode of the box head (models.py:830-843) + fastrcnn_predictions (or, with `multi`, the batch graph's
    combined NMS).  box_logits [K, num_class-1, 4] (class-agnostic already tiled).  Returns (decoded boxes [K,C-1,4],
    probs [K,C], pred_indices [R,2] = (box_id, class_id), final probs [R])."""
    nc1 = box_logits.shape[1]
    anchors = np.tile(proposals[:, None, :], (1, nc1, 1))
    rw = np.asarray(cfg.fastrcnn_bbox_reg_weights, dtype=np.float32)
    dec = decode_bbox_target((box_logits / rw).astype(np.float32), anchors)   # default clip log(1333/16)
    dec = clip_boxes(dec, hw)
    probs = softmax(cls_logits)
    pred, fprobs = (fastrcnn_predictions_multi if multi else fastrcnn_predictions)(dec, probs, cfg)
    return dec, probs, pred, fprobs


def maskrcnn_head(feat, W, num_class):
    """maskrcnn_up4conv_head (models.py:1173-1199): 4 x [conv3x3 SAME + bias + ReLU] on the [R,256,14,14] ROI features,
    Conv2DTranspose 2x2 stride 2 + bias + ReLU (nn.deconv2d, nn.py:383-413; TF kernel layout [kh, kw, out, in]),
    conv1x1 + bias -> [R, num_class - 1, 28, 28] logits."""
    x = _t(feat)
    with torch.no_grad():
        for k in range(4):
            x = torch.relu(_conv(x, W["maskrcnn/fcn%d/W" % k], pad=(1, 1, 1, 1), bias=W["maskrcnn/fcn%d/b" % k]))
        wd = _t(W["maskrcnn/deconv/W"]).permute(3, 2, 0, 1).contiguous()      # -> torch's [in, out, kh, kw]
        x = torch.relu(F.conv_transpose2d(x, wd, _t(W["maskrcnn/deconv/b"]), stride=2))
        x = _conv(x, W["maskrcnn/conv/W"], bias=W["maskrcnn/conv/b"])
    assert x.shape[1] == num_class - 1
    return _np(x)


def final_masks(cfg, W, feats, fboxes, flabels):
    """models.py:934-961: ROIAlign 14 of the final boxes -> mask head -> the logits of each box's own class ->
    sigmoid -> [R,28,28]."""
    if not len(fboxes):
        return np.zeros((0, 28, 28), np.float32), np.zeros((0, cfg.num_class - 1, 28, 28), np.float32)
    roi14, _ = multilevel_roi_align(feats, fboxes, 14, cfg.anchor_strides)
    logits = maskrcnn_head(roi14, W, cfg.num_class)
    sel = logits[np.arange(len(fboxes)), np.asarray(flabels, dtype=np.int64) - 1]
    return (1.0 / (1.0 + np.exp(-sel.astype(np.float32)))).astype(np.float32), logits


def forward(cfg, W, img_hwc_f32: np.ndarray, stages: bool = True) -> dict:
    """Mask_RCNN_FPN.build_forward inference branch (models.py:488-973) for one image
    (already resized by the caller, float32 HWC BGR as obj_detect_tracking.py:597-610)."""
    out = {}
    x = preprocess(img_hwc_f32)
    H, W_ = x.shape[2:]
    hw = (H, W_)
    with torch.no_grad():
        c2345 = backbone(x, W, cfg)
        p23456 = fpn(c2345, W)
    # slice_feature_and_anchors (models.py:372-400): p2..p4 cropped to ceil(H/stride)
    for i, s in enumerate(cfg.anchor_strides):
        if i < 3:
            th = int(math.ceil(H * (1.0 / s))); tw = int(math.ceil(W_ * (1.0 / s)))
            p23456[i] = p23456[i][:, :, :th, :tw]
    na = len(cfg.anchor_ratios)
    lvl_props = []
    rpn_out = []
    for i in range(len(cfg.anchor_strides)):
        with torch.no_grad():
            cls, box = rpn_head(p23456[i], W, na)
        lvl_props.append(level_proposals(cfg, i, cls, box, hw))
        rpn_out.append((cls, box))
    pb, ps = merge_level_proposals(lvl_props, cfg.rpn_test_post_nms_topk)
    feats = [_np(p[0]) for p in p23456[:4]]
    roi, roi_lvl = multilevel_roi_align(feats, pb, 7, cfg.anchor_strides)
    with torch.no_grad():
        cls_logits, box_logits, hidden = fastrcnn_head(roi, W, cfg)
    dec, probs, pred, fprobs = head_postprocess(cls_logits, box_logits, pb, hw, cfg)
    fboxes = dec[pred[:, 0], pred[:, 1]] if len(pred) else np.zeros((0, 4), np.float32)
    flabels = (pred[:, 1] + 1).astype(np.int64)
    if len(fboxes):
        box_feat, _ = multilevel_roi_align(feats, fboxes, 7, cfg.anchor_strides)
    else:
        box_feat = np.zeros((0, feats[0].shape[0], 7, 7), np.float32)
    out.update(final_boxes=fboxes.astype(np.float32), final_labels=flabels,
               final_probs=fprobs.astype(np.float32), fpn_box_feat=box_feat)
    if getattr(cfg, "add_mask", False):
        out["final_masks"], out["mask_logits"] = final_masks(cfg, W, feats, fboxes.astype(np.float32), flabels)
    if stages:
        out.update(c2345=[_np(c[0]) for c in c2345], p23456=[_np(p[0]) for p in p23456],
                   rpn=rpn_out, level_proposals=lvl_props, proposal_boxes=pb, proposal_scores=ps,
                   roi_feat=roi, roi_level=roi_lvl, cls_logits=cls_logits, box_logits=box_logits,
                   hidden=hidden, decoded_boxes=dec, probs=probs, pred_indices=pred)
    return out


def forward_givenbox(cfg, W, img_hwc_f32: np.ndarray, boxes: np.ndarray) -> np.ndarray:
    """RCNN_FPN_givenbox.build_forward (models.py:1900-1950): backbone + FPN, multilevel_roi_align of the given boxes on
    the UNCROPPED p2..p5 (no slice_feature_and_anchors in that graph), mean over the 7x7 bins -> [n, 256]."""
    x = preprocess(img_hwc_f32)
    with torch.no_grad():
        p23456 = fpn(backbone(x, W, cfg), W)
    feats = [_np(p[0]) for p in p23456[:4]]
    boxes = np.asarray(boxes, dtype=np.float32).reshape(-1, 4)
    if not len(boxes):
        return np.zeros((0, feats[0].shape[0]), np.float32)
    roi, _ = multilevel_roi_align(feats, boxes, 7, cfg.anchor_strides)
    return roi.mean(axis=(2, 3)).astype(np.float32)


# ------------------------------------------------------------------------------------------------
# Batch graph: Mask_RCNN_FPN_multi (models.py:1969-3487).  Same layers; the post-processing differs
# because it is built on tf.image.combined_non_max_suppression (zero-padded, no score threshold).

def combined_nms_single_class(boxes, scores, max_out, iou_thr):
    """tf.image.combined_non_max_suppression with q = 1, one class, score_threshold = -inf,
    pad_per_class=False, clip_boxes=False (call site nn.py:1468-1474): hard NMS, zero-padded outputs.
    Returns (boxes [max_out,4], scores [max_out], valid)."""
    keep = tf_ops.non_max_suppression(boxes[:, [1, 0, 3, 2]], scores, max_out, iou_thr)
    ob = np.zeros((max_out, 4), np.float32); os_ = np.zeros((max_out,), np.float32)
    ob[:len(keep)] = boxes[keep]; os_[:len(keep)] = scores[keep]
    return ob, os_, len(keep)


def forward_multi(cfg, W, imgs, stages=False):
    """Inference branch of Mask_RCNN_FPN_multi.build_forward (models.py:2058-2409) for a batch of equally
    sized frames.  Returns zero-padded [B,100,...] outputs + valid counts + concatenated box features."""
    B = len(imgs)
    K, R = cfg.rpn_test_post_nms_topk, cfg.result_per_im
    out_boxes = np.zeros((B, R, 4), np.float32); out_probs = np.zeros((B, R), np.float32)
    out_labels = np.zeros((B, R), np.float32); valid = np.zeros((B,), np.int32)
    feats_all, per_image = [], []
    na = len(cfg.anchor_ratios)
    for b in range(B):
        x = preprocess(imgs[b])
        H, W_ = x.shape[2:]
        hw = (H, W_)
        with torch.no_grad():
            p23456 = fpn(backbone(x, W, cfg), W)
        for i, s in enumerate(cfg.anchor_strides):
            if i < 3:
                p23456[i] = p23456[i][:, :, :int(math.ceil(H / float(s))), :int(math.ceil(W_ / float(s)))]
        lvl = []
        for i in range(len(cfg.anchor_strides)):
            with torch.no_grad():
                cls, box = rpn_head(p23456[i], W, na)
            lvl.append(level_proposals(cfg, i, cls, box, hw, multi=True))
        pb, ps = merge_level_proposals_multi(lvl, K)
        fmaps = [_np(p[0]) for p in p23456[:4]]
        roi, _ = multilevel_roi_align(fmaps, pb, 7, cfg.anchor_strides)
        with torch.no_grad():
            cls_logits, box_logits, _ = fastrcnn_head(roi, W, cfg)
        dec, probs, pred, _ = head_postprocess(cls_logits, box_logits, pb, hw, cfg, multi=True)
        n = len(pred)
        valid[b] = n
        for j, (k, c) in enumerate(pred):
            out_boxes[b, j] = dec[k, c]; out_probs[b, j] = probs[k, c + 1]; out_labels[b, j] = c + 1
        bf, _ = multilevel_roi_align(fmaps, out_boxes[b, :n], 7, cfg.anchor_strides) if n else (np.zeros((0, 256, 7, 7), np.float32), None)
        feats_all.append(bf)
        per_image.append(dict(proposal_boxes=pb, proposal_scores=ps, probs=probs, decoded_boxes=dec))
    res = dict(final_boxes=out_boxes, final_probs=out_probs, final_labels=out_labels, final_valid_indices=valid,
               fpn_box_feat=np.concatenate(feats_all, 0))
    if stages:
        res["per_image"] = per_image
    return res
