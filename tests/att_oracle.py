"""CPU oracle of the attention box head, `--use_att_frcnn_head` (test infrastructure; the product path never imports this).

fastrcnn_2fc_head (models.py:1064-1089; the batch graph's copy :2682-2707 is identical) adds, after the hidden rows are
computed (fc6 / fc7, the relation modules or the conv head):

  feature   = transpose(roi_feature, NCHW -> NHWC)                                   [K, 7, 7, 256]
  attention = conv2d(feature, 1, kernel 3, SAME, bias, activation=softmax)           [K, 7, 7, 1]   scope fastrcnn/attention
  attended  = reduce_sum(feature * attention over the 49 cells)                      [K, 256]
  hidden    = hidden + dense(attended, fc_head_dim, relu)                            scope fastrcnn/att_trans

The softmax runs over the conv's single output channel, so a cell's weight is exactly 1 when its logit is finite and NaN
otherwise; with finite attention weights whose logits cannot overflow (the engine's load check), a logit is non-finite
exactly when its ROI has a non-finite feature (the centre tap reads every channel of its own cell).  `attended` here is
therefore the sum of the ROI's 49 cells, NaN in every channel for an ROI with a non-finite feature; test_att_head_cpu
checks that against the literal conv + softmax.  The class-agnostic heads (models.py:1126-1170) have no attention branch:
with use_frcnn_class_agnostic the wrapper passes the enclosing head's outputs through.

`graph(cfg)` evaluates oracle.frcnn's `forward` and `forward_multi` with the head `relation_oracle.graph` builds (so
GroupNorm, the conv head, squeeze-excite, ResNeXt and the relation modules compose) plus this branch; partial_oracle's
`partial_classes` composes outside it, as its gather runs on this head's logits."""
from __future__ import annotations

import contextlib

import torch

import relation_oracle
from oracle import frcnn

# the last head evaluation's branch rows (float32 numpy), for stage comparisons
LAST = {}


def use_att(cfg):
    return getattr(cfg, "use_att_frcnn_head", False) and not cfg.use_frcnn_class_agnostic


def attended(feat):
    """[K, C, 7, 7] ROI features -> [K, C] (a tensor of the oracle's type): the sum over the 49 cells, all NaN for an ROI
    with a non-finite feature."""
    x = frcnn._t(feat)
    s = x.sum(dim=(2, 3))
    bad = ~torch.isfinite(x).flatten(1).all(dim=1)
    s[bad] = float("nan")
    return s


def head(inner):
    """The box head `inner` (feat, W, cfg) -> (cls, box, hidden) with the attention branch added when cfg asks for it."""
    def fastrcnn_head(feat, W, cfg):
        cls, box, hidden = inner(feat, W, cfg)
        if not use_att(cfg):
            return cls, box, hidden
        t = frcnn._t
        pooled = attended(feat)
        att = torch.relu(pooled @ t(W["fastrcnn/att_trans/W"]) + t(W["fastrcnn/att_trans/b"]))
        h = t(hidden) + att
        LAST["att_pool"], LAST["att_trans"], LAST["att_sum"] = frcnn._np(pooled), frcnn._np(att), frcnn._np(h)
        cls = frcnn._np(h @ t(W["fastrcnn/outputs/class/W"]) + t(W["fastrcnn/outputs/class/b"]))
        box = frcnn._np(h @ t(W["fastrcnn/outputs/box/W"]) + t(W["fastrcnn/outputs/box/b"]))
        box = box.reshape(box.shape[0], -1, 4)[:, 1:, :]       # class-specific only (use_att)
        return cls, box.copy(), frcnn._np(h)
    return fastrcnn_head


@contextlib.contextmanager
def graph(cfg):
    """Within the block, oracle.frcnn evaluates the graph `cfg` describes, attention branch included."""
    with relation_oracle.graph(cfg):
        saved = frcnn.fastrcnn_head
        frcnn.fastrcnn_head = head(saved)
        try:
            yield
        finally:
            frcnn.fastrcnn_head = saved


def forward(cfg, W, img, stages=True):
    with graph(cfg):
        return frcnn.forward(cfg, W, img, stages=stages)


def forward_multi(cfg, W, imgs, stages=False):
    with graph(cfg):
        return frcnn.forward_multi(cfg, W, imgs, stages=stages)
