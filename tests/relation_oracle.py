"""CPU oracle of the relation-network box head, `--add_relation_nn` (test infrastructure; the product path never imports
this).

`oracle.frcnn` restates the plain 2fc head.  This module restates the head `fastrcnn_2fc_head` builds instead when
`add_relation_nn` is set (models.py:1044-1054; the class-agnostic head models.py:1139-1148 is the same) and evaluates the
whole graph through `oracle.frcnn`'s own `forward` and `forward_multi`:

  h1 = relu(fc6(x));  h1 = h1 + RM_r1(h1, boxes)
  h2 = relu(fc7(h1)); h2 = h2 + RM_r2(h2, boxes)          no ReLU after either sum; class / box outputs read h2

  relation_network     nn.py:115-190   group 16, geo_feat_dim 64, value = h itself, output_linear over the
                                       [K, 16 * D] flatten (index g * D + c)
  geometric_encoding   nn.py:273-298   dx = log(max(|cx_i - cx_j| / w_i, 1e-3)), dy = log(max(|cy_i - cy_j| / w_i, 1e-3))
                                       (the width, for dy too), dw = log(w_i / w_j), dh = log(h_i / h_j)

`boxes` are the image's proposals.  `oracle.frcnn`'s head has no boxes argument, so `graph(cfg)` captures them by wrapping
`merge_level_proposals` and `merge_level_proposals_multi`, whose outputs are exactly the rows the head sees, in `forward`
and in `forward_multi`.  The batch graph cannot build this head (Mask_RCNN_FPN_multi calls it without boxes,
models.py:2155-2160); here batch mode is the single-image head applied to each image on its own.  With K = 1 the weight
is 1 on the ROI itself (the reference's tf.squeeze fails there).  `use_conv_frcnn_head` takes precedence: with both flags
there is no relation module.  The arithmetic type follows `oracle.frcnn.exact()`; the stack on `resnext_oracle.graph`
covers GroupNorm, squeeze-excite and ResNeXt too."""
from __future__ import annotations

import contextlib
import math

import torch

import resnext_oracle
from oracle import frcnn

GROUPS = 16               # relation_network(group=16) at models.py:1049, 1054
GEO_DIM = 64              # geo_feat_dim
MODULES = ("RM_r1", "RM_r2")

# the last head evaluation's module outputs (float32 numpy [K, D]), for stage comparisons
LAST = {}


def use_relation(cfg):
    return getattr(cfg, "add_relation_nn", False) and not getattr(cfg, "use_conv_frcnn_head", False)


def geometric_encoding(boxes):
    """nn.py:273-298 on [K, 4] x1y1x2y2 boxes (a tensor of the oracle's type): [K, K, 4] (dx, dy, dw, dh)."""
    x1, y1, x2, y2 = boxes.unbind(1)
    w = x2 - x1
    h = y2 - y1
    cx = 0.5 * (x1 + x2)
    cy = 0.5 * (y1 + y2)
    dx = torch.log(torch.clamp(torch.abs((cx[:, None] - cx[None, :]) / w[:, None]), min=1e-3))
    dy = torch.log(torch.clamp(torch.abs((cy[:, None] - cy[None, :]) / w[:, None]), min=1e-3))
    dw = torch.log(w[:, None] / w[None, :])
    dh = torch.log(h[:, None] / h[None, :])
    return torch.stack([dx, dy, dw, dh], dim=2)


def attention(h, boxes, W, scope):
    """The softmax weights P [K, 16, K] of relation_network `scope` (nn.py:123-172)."""
    t = frcnn._t
    K, D = h.shape
    enc = geometric_encoding(t(boxes))
    e = torch.tanh(enc @ t(W[scope + "/geo_emb/W"]) + t(W[scope + "/geo_emb/b"]))              # [K, K, 64]
    wg = torch.relu(e @ t(W[scope + "/geo_conv/W"]).reshape(GEO_DIM, GROUPS) + t(W[scope + "/geo_conv/b"]))
    wg = wg.permute(0, 2, 1)                                                                      # [K, 16, K]
    dg = D // GROUPS
    q = (h @ t(W[scope + "/query_linear/W"])).reshape(K, GROUPS, dg).permute(1, 0, 2)
    k = (h @ t(W[scope + "/key_linear/W"])).reshape(K, GROUPS, dg).permute(1, 0, 2)
    logits = ((1.0 / math.sqrt(float(dg))) * (q @ k.transpose(1, 2))).permute(1, 0, 2)          # [K, 16, K]
    return torch.softmax(torch.log(torch.clamp(wg, min=1e-6)) + logits, dim=-1)


def relation(h, boxes, W, scope):
    """relation_network (nn.py:115-190): output_linear(P . h) [K, D] for head rows h [K, D] and boxes [K, 4]."""
    K, D = h.shape
    if K == 0:
        return torch.zeros_like(h)
    p = attention(h, boxes, W, scope)
    o = (p.reshape(K * GROUPS, K) @ h).reshape(K, GROUPS * D)
    return o @ frcnn._t(W[scope + "/output_linear/W"])


_PREV = {}
_BOXES = []


def fastrcnn_head(feat, W, cfg):
    """fastrcnn_2fc_head with add_relation_nn (models.py:1044-1054); the head of the enclosing graph otherwise."""
    if not use_relation(cfg):
        return _PREV["fastrcnn_head"](feat, W, cfg)
    t = frcnn._t
    boxes = _BOXES[-1]
    assert len(boxes) == feat.shape[0], (len(boxes), feat.shape)
    x = t(feat.reshape(feat.shape[0], -1))
    h = torch.relu(x @ t(W["fastrcnn/fc6/W"]) + t(W["fastrcnn/fc6/b"]))
    h = h + relation(h, boxes, W, "fastrcnn/RM_r1")
    LAST["rm_r1"] = frcnn._np(h)
    h = torch.relu(h @ t(W["fastrcnn/fc7/W"]) + t(W["fastrcnn/fc7/b"]))
    h = h + relation(h, boxes, W, "fastrcnn/RM_r2")
    LAST["rm_r2"] = frcnn._np(h)
    cls = frcnn._np(h @ t(W["fastrcnn/outputs/class/W"]) + t(W["fastrcnn/outputs/class/b"]))
    box = frcnn._np(h @ t(W["fastrcnn/outputs/box/W"]) + t(W["fastrcnn/outputs/box/b"]))
    box = box.reshape(box.shape[0], -1, 4)
    if not cfg.use_frcnn_class_agnostic:
        box = box[:, 1:, :]
    else:
        box = box.repeat(cfg.num_class - 1, axis=1)         # models.py:799-802
    return cls, box.copy(), frcnn._np(h)


def _capturing(merge):
    def wrapped(levels, topk):
        pb, ps = merge(levels, topk)
        _BOXES.append(pb)
        return pb, ps
    return wrapped


@contextlib.contextmanager
def graph(cfg):
    """Within the block, oracle.frcnn evaluates the graph `cfg` describes: GroupNorm, conv head, squeeze-excite, ResNeXt
    blocks and the relation head."""
    names = ("fastrcnn_head", "merge_level_proposals", "merge_level_proposals_multi")
    with resnext_oracle.graph(cfg):
        saved = {n: getattr(frcnn, n) for n in names}
        _PREV["fastrcnn_head"] = saved["fastrcnn_head"]
        frcnn.merge_level_proposals = _capturing(saved["merge_level_proposals"])
        frcnn.merge_level_proposals_multi = _capturing(saved["merge_level_proposals_multi"])
        frcnn.fastrcnn_head = fastrcnn_head
        try:
            yield
        finally:
            for n, f in saved.items():
                setattr(frcnn, n, f)
            del _BOXES[:]


def forward(cfg, W, img, stages=True):
    with graph(cfg):
        return frcnn.forward(cfg, W, img, stages=stages)


def forward_multi(cfg, W, imgs, stages=False):
    with graph(cfg):
        return frcnn.forward_multi(cfg, W, imgs, stages=stages)
