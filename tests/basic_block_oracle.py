"""CPU oracle of the ResNet-18 / ResNet-34 detectors, `--resnet18` / `--resnet34` (`use_basic_block`) (test infrastructure;
the product path never imports this).

`oracle.frcnn` restates the ResNet bottleneck.  This module restates the block `resnet_fpn_backbone` picks instead when
`use_basic_block` is set (nn.py:864-868) and evaluates the whole graph through `oracle.frcnn`'s own `forward`,
`forward_multi` and `forward_givenbox`, as the other family oracles do:

  resnet_basicblock   nn.py:439-456   conv1 3x3 cin -> ch, stride of the block, padding SAME (the conv2d default,
                                      nn.py:337): at stride 2 the odd pad goes bottom / right, NormReLU
                                      conv2 3x3 ch -> ch, stride 1 SAME, norm (get_bn, zero_init only at training)
                                      + resnet_shortcut(x, ch, stride)
  resnet_shortcut     nn.py:551-566   n_out = ch (not 4 * ch): the identity when the input already has ch channels (group0
                                      block0, after the 64-channel pool), else drop the last row / column and a 1x1
                                      stride-2 VALID conv + norm
  resnet_group        nn.py:586-587   relu after every block

The block takes the `dilations`, `deformable` and `use_se` arguments and ignores them.  `use_resnext` reassigns block_func
after it, so ResNeXt wins.  `graph(cfg)` selects the block from `cfg.use_basic_block` on top of `deform_oracle.graph`, so
GroupNorm, the conv head and the relation head are covered too.  The given-box graph passes `use_basic_block`
(models.py:1935), so `forward_givenbox` runs the basic backbone.  The arithmetic type follows `oracle.frcnn.exact()`."""
from __future__ import annotations

import contextlib
import math

import torch
import torch.nn.functional as F

import deform_oracle
import gn_oracle
from oracle import frcnn
from resnext_oracle import same_pads


def use_basic(cfg):
    return getattr(cfg, "use_basic_block", False) and not getattr(cfg, "use_resnext", False)


def shortcut(x, W, p, ch, stride, use_gn):
    """resnet_shortcut (nn.py:551-566) with n_out = ch."""
    if x.shape[1] == ch:
        return x
    if stride == 2:
        x = x[:, :, :-1, :-1]                    # nn.py:555-556
    return gn_oracle._norm(frcnn._conv(x, W[p + "/convshortcut/W"], stride=stride), W, p + "/convshortcut", use_gn)


def basic_block(x, W, p, ch, stride, use_gn):
    """resnet_basicblock (nn.py:439-456) + shortcut + the group's trailing relu (nn.py:586-587)."""
    conv = frcnn._conv
    norm = gn_oracle._norm
    pad = same_pads(x.shape[2], 3, stride, 1) + same_pads(x.shape[3], 3, stride, 1)
    l = torch.relu(norm(conv(x, W[p + "/conv1/W"], stride=stride, pad=pad), W, p + "/conv1", use_gn))
    l = norm(conv(l, W[p + "/conv2/W"], pad=(1, 1, 1, 1)), W, p + "/conv2", use_gn)
    return torch.relu(l + shortcut(x, W, p, ch, stride, use_gn))


def backbone(x, W, cfg):
    """resnet_fpn_backbone (nn.py:843-944) with block_func = resnet_basicblock."""
    use_gn = getattr(cfg, "use_gn", False)
    h, w = x.shape[2:]
    mult = cfg.fpn_resolution_requirement
    ph = int(math.ceil(h / mult) * mult) - h
    pw = int(math.ceil(w / mult) * mult) - w
    l = F.pad(x, (3, 2 + pw, 3, 2 + ph))
    l = torch.relu(gn_oracle._norm(frcnn._conv(l, W["conv0/W"], stride=2), W, "conv0", use_gn))
    l = F.max_pool2d(F.pad(l, (1, 0, 1, 0)), 3, 2)
    feats = []
    for g, (ch, count) in enumerate(zip((64, 128, 256, 512), cfg.resnet_num_block)):
        for i in range(count):
            l = basic_block(l, W, "group%d/block%d" % (g, i), ch, 2 if (g > 0 and i == 0) else 1, use_gn)
        feats.append(l)
    return feats


@contextlib.contextmanager
def graph(cfg):
    """Within the block, oracle.frcnn evaluates the graph `cfg` describes: GroupNorm, conv head, squeeze-excite, ResNeXt,
    the relation head, deformable and basic blocks."""
    with deform_oracle.graph(cfg):               # restores every oracle.frcnn entry point on exit, backbone included
        if use_basic(cfg):
            frcnn.backbone = backbone
        yield


def forward(cfg, W, img, stages=True):
    with graph(cfg):
        return frcnn.forward(cfg, W, img, stages=stages)


def forward_multi(cfg, W, imgs, stages=False):
    with graph(cfg):
        return frcnn.forward_multi(cfg, W, imgs, stages=stages)


def forward_givenbox(cfg, W, img, boxes):
    with graph(cfg):
        return frcnn.forward_givenbox(cfg, W, img, boxes)
