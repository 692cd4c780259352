"""CPU oracle of the SE-ResNet detector, `--use_se` (`--version 6`) (test infrastructure; the product path never imports this).

`oracle.frcnn` restates the plain ResNet bottleneck.  This module restates what `use_se` adds to it and evaluates the whole
graph through `oracle.frcnn`'s own `forward`, `forward_multi` and `forward_givenbox`, as `gn_oracle` does for GroupNorm:

  resnet_bottleneck   nn.py:459-521   after conv3 and its norm, before the shortcut:
                                        s = GlobalAvgPooling(l)              (nn.py:333-335, per image)
                                        s = relu(dense fc1(s))               [4*ch_out -> ch_out // 4]
                                        s = sigmoid(dense fc2(s))            [ch_out // 4 -> 4*ch_out]
                                        l = l * s[:, :, None, None]
                      nn.py:520-521, 586-587   relu(l + shortcut)
  dense               nn.py:730-774   W [in, out], b [out]: x @ W + b

`graph(cfg)` selects the SE bottleneck from `cfg.use_se` (not from the weight names present) on top of `gn_oracle.graph`,
so `use_gn` + `use_se` is covered too.  The arithmetic type follows `oracle.frcnn.exact()`."""
from __future__ import annotations

import contextlib
import math

import torch
import torch.nn.functional as F

import gn_oracle
from oracle import frcnn


def squeeze_excite(l, W, p):
    """The use_se branch of resnet_bottleneck (nn.py:506-519) on l [N, C, H, W]; returns (l * gate, gate [N, C])."""
    t = frcnn._t
    s = l.mean(dim=(2, 3))
    s = torch.relu(s @ t(W[p + "/fc1/W"]) + t(W[p + "/fc1/b"]))
    s = torch.sigmoid(s @ t(W[p + "/fc2/W"]) + t(W[p + "/fc2/b"]))
    return l * s[:, :, None, None], s


def bottleneck(x, W, p, stride, dil, use_gn, use_se, gates=None):
    """resnet_bottleneck (nn.py:459-521) + shortcut (nn.py:551-566) + trailing relu, as gn_oracle.bottleneck with the
    squeeze-excite gate between conv3's norm and the shortcut sum.  `gates`, when given, collects (scope, gate)."""
    conv = frcnn._conv
    norm = gn_oracle._norm
    sc = x
    l = torch.relu(norm(conv(x, W[p + "/conv1/W"]), W, p + "/conv1", use_gn))
    if stride == 2:
        l = conv(l, W[p + "/conv2/W"], stride=2, dilation=dil, pad=(1, 0, 1, 0))      # nn.py:487-492
        l = torch.relu(norm(l, W, p + "/conv2", use_gn))
        if dil != 1:
            l = F.pad(l, (1, 0, 1, 0))           # nn.py:493-497
    else:
        l = conv(l, W[p + "/conv2/W"], dilation=dil, pad=frcnn._same_pad(3, dil))
        l = torch.relu(norm(l, W, p + "/conv2", use_gn))
    l = norm(conv(l, W[p + "/conv3/W"]), W, p + "/conv3", use_gn)
    if use_se:
        l, g = squeeze_excite(l, W, p)
        if gates is not None:
            gates.append((p, g))
    if (p + "/convshortcut/W") in W:
        if stride == 2:
            sc = conv(sc[:, :, :-1, :-1], W[p + "/convshortcut/W"], stride=2)          # nn.py:555-556
        else:
            sc = conv(sc, W[p + "/convshortcut/W"])
        sc = norm(sc, W, p + "/convshortcut", use_gn)
    return torch.relu(l + sc)


def backbone(x, W, cfg, gates=None):
    """resnet_fpn_backbone (nn.py:843-944) with the bottlenecks above (use_gn and use_se from cfg)."""
    use_gn, use_se = getattr(cfg, "use_gn", False), getattr(cfg, "use_se", False)
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
            l = bottleneck(l, W, "group%d/block%d" % (g, i), stride, dil, use_gn, use_se, gates)
        feats.append(l)
    return feats


@contextlib.contextmanager
def graph(cfg):
    """Within the block, oracle.frcnn evaluates the graph `cfg` describes: GroupNorm, conv head and squeeze-excite."""
    with gn_oracle.graph(cfg):                   # restores every oracle.frcnn entry point on exit, backbone included
        if getattr(cfg, "use_se", False):
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
