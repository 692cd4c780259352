"""ORACLE (test infrastructure only).  CPU fp32 restatement of the EfficientDet feature network (BiFPN),
class/box nets and post-processing the reference wires up in efficientdet_wrapper.py.

Reference: efficientdet/efficientdet_arch.py (`resample_feature_map` :105-200, `class_net` :227-282,
`box_net` :285-340, `build_class_and_box_outputs` :343-393, `build_feature_network` :440-505,
`build_bifpn_layer` :594-682), efficientdet/utils.py (`batch_norm_act` :252-303 eps 1e-3, swish :35-46),
efficientdet/anchors.py (`_generate_anchor_boxes` :216-257, `decode_box_outputs_tf` :369-396,
`_generate_detections_tf` :399-487), efficientdet_wrapper.py (`add_metric_fn_inputs` :367-474,
`get_results_tf` :304-363, `multilevel_roi_align` :265-301).
The graph is TensorFlow (absent here, google/automl vendored copy) => op arithmetic **parity unpinned**
(tf.layers.separable_conv2d, max_pooling2d SAME, non_max_suppression_with_scores follow TF's documented
semantics, SURVEY Appendix B).  Tensors are NCHW torch fp32; weights use TF variable naming, HWIO kernels.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from . import frcnn, tf_ops

BN_EPS = 1e-3


def _t(a):
    """float32 by default; float64 inside `with oracle.frcnn.exact():` (the rounding-noise-free evaluation, see frcnn.py)."""
    from .frcnn import _DT
    t = torch.from_numpy(np.ascontiguousarray(a))
    return t.to(_DT[-1]) if t.is_floating_point() else t


def _np(t):
    return t.to(torch.float32).numpy()


def swish(x):
    return x * torch.sigmoid(x)


def bn(x, W, name):
    g, b = _t(W[name + "/gamma"]), _t(W[name + "/beta"])
    m, v = _t(W[name + "/moving_mean"]), _t(W[name + "/moving_variance"])
    inv = torch.rsqrt(v + BN_EPS) * g
    return x * inv.view(1, -1, 1, 1) + (b - m * inv).view(1, -1, 1, 1)


def conv1x1(x, W, name):
    k = _t(W[name + "/kernel"]).permute(3, 2, 0, 1).contiguous()
    return F.conv2d(x, k, _t(W[name + "/bias"]))


def sepconv(x, W, name):
    """tf.layers.separable_conv2d(depth_multiplier=1, padding='same'): depthwise 3x3 then pointwise + bias."""
    dw = _t(W[name + "/depthwise_kernel"])            # [3,3,C,1]
    c = dw.shape[2]
    x = F.conv2d(x, dw.permute(2, 3, 0, 1).contiguous(), None, padding=1, groups=c)
    pw = _t(W[name + "/pointwise_kernel"]).permute(3, 2, 0, 1).contiguous()
    return F.conv2d(x, pw, _t(W[name + "/bias"]))


def maxpool_same(x, stride):
    """tf.layers.max_pooling2d(pool=stride+1, strides=stride, padding='SAME') (arch.py:157-163)."""
    k = stride + 1
    h, w = x.shape[2:]
    oh, ow = -(-h // stride), -(-w // stride)
    ph = max((oh - 1) * stride + k - h, 0)
    pw = max((ow - 1) * stride + k - w, 0)
    x = F.pad(x, (pw // 2, pw - pw // 2, ph // 2, ph - ph // 2), value=float("-inf"))
    return F.max_pool2d(x, k, stride)


def resample(feat, W, name, th, tw, tc, apply_bn=True):
    """resample_feature_map (arch.py:105-200), conv_after_downsample=False."""
    _, c, h, w = feat.shape

    def maybe_1x1(f):
        if c != tc:
            f = conv1x1(f, W, name + "/conv2d")
            if apply_bn:
                f = bn(f, W, name + "/bn")
        return f

    if h > th and w > tw:
        feat = maybe_1x1(feat)
        sh, sw = (h - 1) // th + 1, (w - 1) // tw + 1
        assert sh == sw
        feat = maxpool_same(feat, sh)
    elif h <= th and w <= tw:
        feat = maybe_1x1(feat)
        if h < th or w < tw:
            feat = feat.repeat_interleave(th // h, dim=2).repeat_interleave(tw // w, dim=3)   # nearest_upsampling
    else:
        raise ValueError("incompatible sizes")
    return feat


def build_feature_network(features, W, cfg, nodes, fsizes):
    """build_feature_network + build_bifpn_layer (arch.py:440-505, 594-682).  features: {3,4,5: NCHW}."""
    feats = [features[l] for l in (3, 4, 5)]
    for level in (6, 7):
        h, w = feats[-1].shape[2:]
        feats.append(resample(feats[-1], W, "resample_p%d" % level, (h - 1) // 2 + 1, (w - 1) // 2 + 1,
                              cfg.fpn_num_filters))
    for rep in range(cfg.fpn_cell_repeats):
        feats = list(feats)
        for i, (lvl, offsets) in enumerate(nodes):
            th, tw = fsizes[lvl]
            pre = "fpn_cells/cell_%d/fnode%d" % (rep, i)
            ins = [resample(feats[o], W, "%s/resample_%d_%d_%d" % (pre, idx, o, len(feats)), th, tw,
                            cfg.fpn_num_filters) for idx, o in enumerate(offsets)]
            if cfg.fpn_weight_method == "sum":
                node = ins[0]
                for t in ins[1:]:
                    node = node + t                                  # tf.add_n
            elif cfg.fpn_weight_method == "fastattn":
                ws = [torch.relu(_t(W["%s/WSM%s" % (pre, "" if k == 0 else "_%d" % k)])) for k in range(len(ins))]
                tot = ws[0]
                for t in ws[1:]:
                    tot = tot + t
                parts = [ins[k] * ws[k] / (tot + 0.0001) for k in range(len(ins))]
                node = parts[0]
                for t in parts[1:]:
                    node = node + t
            else:
                raise ValueError(cfg.fpn_weight_method)
            op = "%s/op_after_combine%d" % (pre, len(feats))
            node = bn(sepconv(swish(node), W, op + "/conv"), W, op + "/bn")
            feats.append(node)
        out = {}
        for l in range(cfg.min_level, cfg.max_level + 1):
            for i, (lvl, _) in enumerate(reversed(nodes)):
                if lvl == l:
                    out[l] = feats[-1 - i]
                    break
        feats = [out[l] for l in range(cfg.min_level, cfg.max_level + 1)]
    return out


def head_net(x, W, level, cfg, kind):
    """class_net / box_net (arch.py:227-340): shared sepconvs, per-level BN, swish; then *-predict."""
    for i in range(cfg.box_class_repeats):
        x = sepconv(x, W, "%s_net/%s-%d" % (kind, kind, i))
        x = swish(bn(x, W, "%s_net/%s-%d-bn-%d" % (kind, kind, i, level)))
    return sepconv(x, W, "%s_net/%s-predict" % (kind, kind))


def anchor_boxes(cfg, fsizes):
    """anchors.py:182-257 -> float32 [N,4] (ymin, xmin, ymax, xmax), levels min..max, [h, w, anchor] order."""
    out = []
    for level in range(cfg.min_level, cfg.max_level + 1):
        stride = (fsizes[0][0] / float(fsizes[level][0]), fsizes[0][1] / float(fsizes[level][1]))
        per = []
        for octave in range(cfg.num_scales):
            for aspect in cfg.aspect_ratios:
                sx = cfg.anchor_scale * stride[1] * 2 ** (octave / float(cfg.num_scales))
                sy = cfg.anchor_scale * stride[0] * 2 ** (octave / float(cfg.num_scales))
                ax2, ay2 = sx * aspect[0] / 2.0, sy * aspect[1] / 2.0
                x = np.arange(stride[1] / 2, cfg.image_size[1], stride[1])
                y = np.arange(stride[0] / 2, cfg.image_size[0], stride[0])
                xv, yv = np.meshgrid(x, y)
                xv, yv = xv.reshape(-1), yv.reshape(-1)
                b = np.vstack((yv - ay2, xv - ax2, yv + ay2, xv + ax2)).swapaxes(0, 1)
                per.append(np.expand_dims(b, axis=1))
        out.append(np.concatenate(per, axis=1).reshape([-1, 4]))
    return np.vstack(out).astype(np.float32)


def sigmoid(logits):
    """anchors.py:51-53 in float32 (tf.sigmoid of float32 logits at :443)."""
    f32 = np.float32
    return (f32(1) / (f32(1) + np.exp(-np.asarray(logits, f32)))).astype(f32)


def decode_boxes(rel_codes, anchors):
    """decode_box_outputs_tf (anchors.py:369-396; numpy twin :56-84): [N,4] (ty,tx,th,tw) x anchors [N,4]
    (ymin,xmin,ymax,xmax) -> [N,4] (ymin,xmin,ymax,xmax), float32 op by op."""
    f32 = np.float32
    t = np.asarray(rel_codes, f32)
    anchors = np.asarray(anchors, f32)
    yca = ((anchors[:, 0] + anchors[:, 2]) / f32(2)).astype(f32); xca = ((anchors[:, 1] + anchors[:, 3]) / f32(2)).astype(f32)
    ha = (anchors[:, 2] - anchors[:, 0]).astype(f32); wa = (anchors[:, 3] - anchors[:, 1]).astype(f32)
    w = (np.exp(t[:, 3]).astype(f32) * wa).astype(f32); h = (np.exp(t[:, 2]).astype(f32) * ha).astype(f32)
    yc = ((t[:, 0] * ha).astype(f32) + yca).astype(f32); xc = ((t[:, 1] * wa).astype(f32) + xca).astype(f32)
    return np.stack([yc - h / f32(2), xc - w / f32(2), yc + h / f32(2), xc + w / f32(2)], 1).astype(f32)


def postprocess(cls_out, box_out, cfg, fsizes, image_scale, partial_class_idxs=None):
    """add_metric_fn_inputs (wrapper:367-474) + _generate_detections_tf (anchors.py:399-487).
    cls_out/box_out: {level: [H,W,A*C] / [H,W,A*4]} numpy.  Returns boxes x1y1x2y2 (scaled), scores, classes 1..90,
    level indexes -- canonical order = NMS selection order."""
    return nms_select(*topk_candidates(cls_out, box_out, cfg, fsizes, partial_class_idxs), cfg, image_scale)


def topk_candidates(cls_out, box_out, cfg, fsizes, partial_class_idxs=None, top_k=tf_ops.top_k):
    """add_metric_fn_inputs' global top-k over all class logits, then sigmoid and the anchor decode.  Returns the
    candidates in top-k order (logit descending, then flat index): boxes [K,4] (ymin, xmin, ymax, xmax) in network
    pixels, scores [K], classes [K] (1-based), levels [K].  top_k: any exact equivalent of tf_ops.top_k."""
    nc = cfg.num_classes
    na = cfg.num_scales * len(cfg.aspect_ratios)
    cls_all = np.concatenate([cls_out[l].reshape(-1, nc) for l in range(cfg.min_level, cfg.max_level + 1)], 0)
    if partial_class_idxs:                                            # wrapper :398-411: tf.gather on the class axis
        cls_all = np.ascontiguousarray(cls_all[:, list(partial_class_idxs)])
        nc = len(partial_class_idxs)
    box_all = np.concatenate([box_out[l].reshape(-1, 4) for l in range(cfg.min_level, cfg.max_level + 1)], 0)
    lvl_all = np.concatenate([np.full(fsizes[l][0] * fsizes[l][1] * na, l, np.int32)
                              for l in range(cfg.min_level, cfg.max_level + 1)])
    flat = cls_all.reshape(-1)
    k = min(cfg.max_detection_topk, flat.shape[0])
    _, ti = top_k(flat, k)
    idx, cls = ti // nc, ti % nc
    logits = cls_all[idx, cls]
    anchors = anchor_boxes(cfg, fsizes)[idx]
    scores = sigmoid(logits)
    with np.errstate(over="ignore"):                                  # exp(th) may overflow to an infinite side
        boxes = decode_boxes(box_all[idx], anchors)
    return boxes, scores, (cls + 1).astype(np.int32), lvl_all[idx]


def nms_select(boxes, scores, classes, levels, cfg, image_scale):
    """_generate_detections_tf's class-agnostic non_max_suppression_with_scores over topk_candidates' output (visited by
    score descending, then candidate rank).  Returns the kept boxes x1y1x2y2 * image_scale, scores, classes, levels."""
    f32 = np.float32
    keep = tf_ops.non_max_suppression(boxes, scores, cfg.result_per_im, cfg.nms_iou_threshold,
                                      score_threshold=cfg.result_score_thres)
    b = (np.asarray(boxes, f32).reshape(-1, 4)[keep] * f32(image_scale)).astype(f32)
    return b[:, [1, 0, 3, 2]], scores[keep], classes[keep], levels[keep]


def box_features(fpn_feats, boxes, levels, cfg):
    """wrapper multilevel_roi_align (:265-301): ROIAlign 7x7 on the box's own level, mean -> [R, C]."""
    out = np.zeros((boxes.shape[0], cfg.fpn_num_filters), np.float32)
    for l in range(cfg.min_level, cfg.max_level + 1):
        ids = np.where(levels == l)[0]
        if len(ids):
            bf = (boxes[ids] * np.float32(1.0 / (2.0 ** l))).astype(np.float32)
            r = frcnn.roi_align(_np(fpn_feats[l][0]), bf, 7)          # [K,C,7,7]
            out[ids] = r.mean(axis=(2, 3), dtype=np.float32)
    return out


def forward_from_features(cfg, W, features, image_scale=1.0, stages=False, partial_class_idxs=None):
    """BiFPN + heads + post-processing from backbone features {3,4,5: numpy [C,H,W]}."""
    from object_detection_tracking_b200.effdet_config import BIFPN_NODES, feat_sizes
    fs = feat_sizes(cfg)
    with torch.no_grad():
        feats = build_feature_network({l: _t(features[l])[None] for l in (3, 4, 5)}, W, cfg, BIFPN_NODES, fs)
        cls_out = {l: _np(head_net(feats[l], W, l, cfg, "class")[0].permute(1, 2, 0).contiguous()) for l in feats}
        box_out = {l: _np(head_net(feats[l], W, l, cfg, "box")[0].permute(1, 2, 0).contiguous()) for l in feats}
    boxes, scores, classes, levels = postprocess(cls_out, box_out, cfg, fs, image_scale, partial_class_idxs)
    res = dict(final_boxes=boxes, final_probs=scores, final_labels=classes, levels=levels,
               fpn_box_feat=box_features(feats, boxes, levels, cfg))
    if stages:
        res.update(fpn={l: _np(feats[l][0]) for l in feats}, cls_out=cls_out, box_out=box_out)
    return res
