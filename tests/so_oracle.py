"""CPU oracle of the small-object branch, `--use_small_object_head` (test infrastructure; the product path never imports
this).

The branch (models.py:590-692, 845-897) reads the box head's logits and the FPN levels; it changes nothing the main
outputs depend on.  `branch(cfg, W, out)` evaluates it after a forward of `att_oracle` (so GroupNorm, the relation
modules and the attention head compose) with stages=True:

  boxes   decode_bbox_target of every class, unclipped; probs = softmax(label logits)
  select  per small class: tf.image.non_max_suppression(boxes, probs, result_per_im, nms_thres), no score threshold,
          selection order kept; unequal counts raise SoCountError (tf.map_fn cannot stack them)
  hidden  ROIAlign 7 of the selected boxes (unclipped) -> the head's fc6 -> fc7 (plain: no relation / attention)
  assoc   with use_so_association: Person's NMS (so_person_topk) -> ref rows; hidden[i] += person_object_relation
  logits  per class dense [D, 2]; rebuilt [K, C + 1]: column 0 the mean of the classes' column 0, column i + 1 class i's
          column 1
  final   fastrcnn_predictions over the clipped [K, C, 4] boxes and those LOGITS, score-filtered only with
          use_so_score_thres

With one key row the softmax weight is 1 (the reference's tf.squeeze fails there).  The arithmetic type follows
`oracle.frcnn.exact()`."""
from __future__ import annotations

import copy
import math

import numpy as np
import torch

from oracle import frcnn, tf_ops

GROUPS = 16
GEO_DIM = 64
REL = "fastrcnn/small_objects/person_object_relation"


class SoCountError(RuntimeError):
    def __init__(self, counts):
        super().__init__("small classes kept different counts: %s" % (counts,))
        self.counts = counts


def geometric_encoding_pair(b1, b2):
    """nn.py:301-332 on [K, 4] and [R, 4] x1y1x2y2 boxes: [K, R, 4]; both centre offsets over the width of box 2."""
    x11, y11, x12, y12 = b1.unbind(1)
    x21, y21, x22, y22 = b2.unbind(1)
    w1, h1, w2, h2 = x12 - x11, y12 - y11, x22 - x21, y22 - y21
    cx1, cy1, cx2, cy2 = 0.5 * (x11 + x12), 0.5 * (y11 + y12), 0.5 * (x21 + x22), 0.5 * (y21 + y22)
    dx = torch.log(torch.clamp(torch.abs((cx1[:, None] - cx2[None, :]) / w2[None, :]), min=1e-3))
    dy = torch.log(torch.clamp(torch.abs((cy1[:, None] - cy2[None, :]) / w2[None, :]), min=1e-3))
    dw = torch.log(w1[:, None] / w2[None, :])
    dh = torch.log(h1[:, None] / h2[None, :])
    return torch.stack([dx, dy, dw, dh], dim=2)


def person_object_relation(h, boxes, ref_boxes, ref, W, scope=REL):
    """nn.py:194-270: output_linear(P . ref) [K, D] (without the residual) for query rows h [K, D], key rows ref [R, D]."""
    t = frcnn._t
    h, ref = t(h), t(ref)
    K, D = h.shape
    R = ref.shape[0]
    if K == 0 or R == 0:
        return torch.zeros_like(h)
    enc = geometric_encoding_pair(t(boxes), t(ref_boxes))
    e = torch.tanh(enc @ t(W[scope + "/geo_emb/W"]) + t(W[scope + "/geo_emb/b"]))                # [K, R, 64]
    wg = torch.relu(e @ t(W[scope + "/geo_conv/W"]).reshape(GEO_DIM, GROUPS) + t(W[scope + "/geo_conv/b"]))
    wg = wg.permute(0, 2, 1)                                                                      # [K, 16, R]
    dg = D // GROUPS
    q = (h @ t(W[scope + "/query_linear/W"])).reshape(K, GROUPS, dg).permute(1, 0, 2)
    k = (ref @ t(W[scope + "/key_linear/W"])).reshape(R, GROUPS, dg).permute(1, 0, 2)
    logits = ((1.0 / math.sqrt(float(dg))) * (q @ k.transpose(1, 2))).permute(1, 0, 2)           # [K, 16, R]
    p = torch.softmax(torch.log(torch.clamp(wg, min=1e-6)) + logits, dim=-1)
    o = (p.reshape(K * GROUPS, R) @ ref).reshape(K, GROUPS * D)
    return o @ t(W[scope + "/output_linear/W"])


def _fc67(feat, W):
    t = frcnn._t
    x = t(feat.reshape(feat.shape[0], -1))
    h = torch.relu(x @ t(W["fastrcnn/fc6/W"]) + t(W["fastrcnn/fc6/b"]))
    return torch.relu(h @ t(W["fastrcnn/fc7/W"]) + t(W["fastrcnn/fc7/b"]))


def branch(cfg, W, out, hw):
    """The branch from a forward's stages (`out`: att_oracle / oracle.frcnn forward with stages=True) of an image of
    size hw.  Returns a dict with so_final_boxes [n, 4], so_final_labels [n] int64, so_final_probs [n] (logits) and the
    stages."""
    t = frcnn._t
    H, W_img = hw
    pb, cls_logits, box_logits = out["proposal_boxes"], out["cls_logits"], out["box_logits"]
    nc1 = box_logits.shape[1]
    rw = np.asarray(cfg.fastrcnn_bbox_reg_weights, dtype=np.float32)
    dec = frcnn.decode_bbox_target((box_logits / rw).astype(np.float32), np.tile(pb[:, None, :], (1, nc1, 1)))
    probs = frcnn.softmax(cls_logits)
    R, thr = int(cfg.result_per_im), float(cfg.fastrcnn_nms_iou_thres)
    ids = list(cfg.small_object_class_ids)
    keeps = [tf_ops.non_max_suppression(dec[:, i - 1], probs[:, i], R, thr) for i in ids]
    counts = [len(k) for k in keeps]
    res = dict(class_counts=counts)
    if len(set(counts)) != 1:
        raise SoCountError(counts)
    K = counts[0]
    so_boxes = np.stack([dec[k, i - 1] for k, i in zip(keeps, ids)]).astype(np.float32).reshape(len(ids), K, 4)
    feats = out["p23456"][:4]
    roi, _ = frcnn.multilevel_roi_align(feats, so_boxes.reshape(-1, 4), 7, cfg.anchor_strides)
    with torch.no_grad():
        hidden = _fc67(roi, W).reshape(len(ids), K, -1)
        res["so_fc7"] = frcnn._np(hidden).reshape(len(ids) * K, -1)
        if cfg.use_so_association:
            pid = cfg.so_person_class_id
            pk = tf_ops.non_max_suppression(dec[:, pid - 1], probs[:, pid], int(cfg.so_person_topk), thr)
            ref_boxes = dec[pk, pid - 1].astype(np.float32).reshape(-1, 4)
            rroi, _ = frcnn.multilevel_roi_align(feats, ref_boxes, 7, cfg.anchor_strides)
            ref = _fc67(rroi, W)
            hidden = torch.stack([hidden[i] + person_object_relation(hidden[i], so_boxes[i], ref_boxes, ref, W)
                                  for i in range(len(ids))])
            res.update(ref_boxes=ref_boxes, so_asso=frcnn._np(hidden).reshape(len(ids) * K, -1))
        lg = [hidden[i] @ t(W["fastrcnn/small_objects/small_object_classification_c%d/W" % (i + 1)])
              + t(W["fastrcnn/small_objects/small_object_classification_c%d/b" % (i + 1)]) for i in range(len(ids))]
        lg = torch.stack(lg)                                                                    # [C, K, 2]
        logits = frcnn._np(torch.cat([lg[:, :, 0].mean(dim=0)[:, None], lg[:, :, 1].transpose(0, 1)], dim=1))
    boxes = frcnn.clip_boxes(so_boxes.transpose(1, 0, 2), (H, W_img))                          # [K, C, 4]
    fcfg = copy.copy(cfg)
    if not cfg.use_so_score_thres:
        fcfg.result_score_thres = -np.inf
    pred, fprobs = frcnn.fastrcnn_predictions(boxes, logits, fcfg)
    fb = boxes[pred[:, 0], pred[:, 1]] if len(pred) else np.zeros((0, 4), np.float32)
    res.update(so_boxes=so_boxes, so_logits=logits, so_cls_logits=frcnn._np(lg), so_final_boxes=fb.astype(np.float32),
               so_final_labels=(pred[:, 1] + 1).astype(np.int64), so_final_probs=fprobs.astype(np.float32))
    return res


def forward(cfg, W, img):
    """The main outputs (att_oracle.forward, stages) and the branch's, for one resized float32 image."""
    import att_oracle
    out = att_oracle.forward(cfg, W, img, stages=True)
    out["so"] = branch(cfg, W, out, img.shape[:2])
    return out
