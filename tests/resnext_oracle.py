"""CPU oracle of the ResNeXt detector, `--use_resnext` (test infrastructure; the product path never imports this).

`oracle.frcnn` restates the ResNet bottleneck.  This module restates the block `resnet_fpn_backbone` picks instead when
`use_resnext` is set (nn.py:864-868) and evaluates the whole graph through `oracle.frcnn`'s own `forward`,
`forward_multi` and `forward_givenbox`, as `se_oracle` does for squeeze-excite:

  resnext_32x4d_bottleneck  nn.py:524-549   conv1 1x1 -> 2*ch, NormReLU
                                            conv2 3x3 2*ch -> 2*ch, split=32, stride / dilation of the block, padding
                                                  SAME (no explicit pad, no [1,0] pad after a dilated stride-2 conv),
                                                  NormReLU
                                            conv3 1x1 -> 4*ch, norm; + shortcut (nn.py:551-566); relu (nn.py:586-587)
  conv2d split != 1         nn.py:352-355   W [k, k, Cin / split, Cout]: TF's grouped conv2d, output group g reading
                                            input channels [g * Cin / split, (g + 1) * Cin / split)
  padding SAME              SURVEY App. B   total = max((ceil(n / s) - 1) * s + (k - 1) * d + 1 - n, 0), the odd
                                            element at the bottom / right

The block has no squeeze-excite branch: `use_se` is ignored with `use_resnext`.  `graph(cfg)` selects the block from
`cfg.use_resnext` on top of `se_oracle.graph`, so GroupNorm and the conv head are covered too.  The reference's
`RCNN_FPN_givenbox` never passes `use_resnext` (models.py:1930-1936); here the given-box entry runs the backbone the
configuration describes.  The arithmetic type follows `oracle.frcnn.exact()`."""
from __future__ import annotations

import contextlib
import math

import torch
import torch.nn.functional as F

import gn_oracle
import se_oracle
from oracle import frcnn

GROUPS = 32              # resnext_32x4d_bottleneck's split (nn.py:539)


def same_pads(n, k, stride, dil):
    """TF padding SAME along one axis of size n: (before, after)."""
    out = -(-n // stride)
    total = max((out - 1) * stride + (k - 1) * dil + 1 - n, 0)
    return total // 2, total - total // 2


def group_conv(x, w_hwio, groups, stride=1, dilation=1, pad=(0, 0, 0, 0)):
    """nn.conv2d with split = groups (nn.py:337-381): HWIO kernel [k, k, Cin / groups, Cout], pad = (top, bottom, left,
    right)."""
    wt = frcnn._t(w_hwio).permute(3, 2, 0, 1).contiguous()
    x = F.pad(x, (pad[2], pad[3], pad[0], pad[1]))
    return F.conv2d(x, wt, stride=stride, dilation=dilation, groups=groups)


def bottleneck(x, W, p, stride, dil, use_gn):
    """resnext_32x4d_bottleneck (nn.py:524-549) + shortcut (nn.py:551-566) + trailing relu (nn.py:586-587)."""
    conv = frcnn._conv
    norm = gn_oracle._norm
    sc = x
    l = torch.relu(norm(conv(x, W[p + "/conv1/W"]), W, p + "/conv1", use_gn))
    pad = same_pads(l.shape[2], 3, stride, dil) + same_pads(l.shape[3], 3, stride, dil)
    l = group_conv(l, W[p + "/conv2/W"], GROUPS, stride=stride, dilation=dil, pad=pad)
    l = torch.relu(norm(l, W, p + "/conv2", use_gn))
    l = norm(conv(l, W[p + "/conv3/W"]), W, p + "/conv3", use_gn)
    if (p + "/convshortcut/W") in W:
        if stride == 2:
            sc = conv(sc[:, :, :-1, :-1], W[p + "/convshortcut/W"], stride=2)          # nn.py:555-556
        else:
            sc = conv(sc, W[p + "/convshortcut/W"])
        sc = norm(sc, W, p + "/convshortcut", use_gn)
    return torch.relu(l + sc)


def backbone(x, W, cfg):
    """resnet_fpn_backbone (nn.py:843-944) with block_func = resnext_32x4d_bottleneck."""
    use_gn = getattr(cfg, "use_gn", False)
    h, w = x.shape[2:]
    mult = cfg.fpn_resolution_requirement
    ph = int(math.ceil(h / mult) * mult) - h
    pw = int(math.ceil(w / mult) * mult) - w
    l = F.pad(x, (3, 2 + pw, 3, 2 + ph))
    l = torch.relu(gn_oracle._norm(frcnn._conv(l, W["conv0/W"], stride=2), W, "conv0", use_gn))
    l = F.max_pool2d(F.pad(l, (1, 0, 1, 0)), 3, 2)
    feats = []
    for g, count in enumerate(cfg.resnet_num_block):
        for i in range(count):
            stride = 2 if (g > 0 and i == 0) else 1
            dil = 2 if (g == 3 and cfg.use_dilations and i in range(count)[-3:]) else 1
            l = bottleneck(l, W, "group%d/block%d" % (g, i), stride, dil, use_gn)
        feats.append(l)
    return feats


@contextlib.contextmanager
def graph(cfg):
    """Within the block, oracle.frcnn evaluates the graph `cfg` describes: GroupNorm, conv head, squeeze-excite and
    ResNeXt blocks."""
    with se_oracle.graph(cfg):                   # restores every oracle.frcnn entry point on exit, backbone included
        if getattr(cfg, "use_resnext", False):
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
