"""CPU oracle of the GroupNorm model family (test infrastructure; the product path never imports this).

`oracle.frcnn` restates the BatchNorm graph with the 2fc box head.  This module restates what `--use_gn` and
`--use_conv_frcnn_head` change in it and evaluates the whole graph through `oracle.frcnn`'s own `forward`,
`forward_multi` and `forward_givenbox`:

  group_norm               nn.py:81-108     32 groups, tf.nn.moments statistics per sample, eps 1e-5
  GNReLU / get_bn          nn.py:591-623    `<conv scope>/gn/{gamma,beta}` replaces `<conv scope>/bn/...`
  resnet_bottleneck        nn.py:459-521    GN + ReLU before the dilated block's [1, 0] pad
  fpn_model                nn.py:987-1009   gn_c* before the top-down sum, gn_p* after the post-hoc 3x3
  conv_frcnn_head          models.py:1110-1125  4 x [conv 3x3 + bias, ReLU, then GN per ROI], then dense "fc" + ReLU

`graph(cfg)` binds `oracle.frcnn`'s backbone / fpn / box-head entry points to the versions below for the duration of a
`with` block; the stages, proposals, ROIAlign and post-processing stay exactly `oracle.frcnn`'s.  The arithmetic type
follows `oracle.frcnn.exact()`."""
from __future__ import annotations

import contextlib
import math

import torch
import torch.nn.functional as F

from oracle import frcnn

GN_GROUPS = 32           # group_norm(x, group=32) (nn.py:81)


def gn(x, W, name):
    """group_norm (nn.py:81-108): statistics per sample over (C/32, H, W) from tf.nn.moments (the mean, then the mean of
    squared deviations from it), then tf.nn.batch_normalization with eps 1e-5:
    inv = rsqrt(var + eps) * gamma, y = x * inv + (beta - mean * inv)."""
    n, c, h, w = x.shape
    assert c % GN_GROUPS == 0, c
    xg = x.reshape(n, GN_GROUPS, c // GN_GROUPS, h, w)
    mean = xg.mean(dim=(2, 3, 4), keepdim=True)
    var = ((xg - mean) ** 2).mean(dim=(2, 3, 4), keepdim=True)
    g = frcnn._t(W[name + "/gamma"]).view(1, GN_GROUPS, c // GN_GROUPS, 1, 1)
    b = frcnn._t(W[name + "/beta"]).view(1, GN_GROUPS, c // GN_GROUPS, 1, 1)
    inv = torch.rsqrt(var + frcnn.BN_EPS) * g
    return (xg * inv + (b - mean * inv)).reshape(n, c, h, w)


def _norm(x, W, scope, use_gn):
    """get_bn / NormReLU's norm (nn.py:591-623): `<scope>/gn` with use_gn, else `<scope>/bn`."""
    return gn(x, W, scope + "/gn") if use_gn else frcnn._bn(x, W, scope)


def bottleneck(x, W, p, stride, dil, use_gn):
    """resnet_bottleneck (nn.py:459-521) + shortcut (nn.py:551-566) + trailing relu, as oracle.frcnn.bottleneck with the
    norm chosen by use_gn."""
    conv = frcnn._conv
    sc = x
    l = torch.relu(_norm(conv(x, W[p + "/conv1/W"]), W, p + "/conv1", use_gn))
    if stride == 2:
        l = conv(l, W[p + "/conv2/W"], stride=2, dilation=dil, pad=(1, 0, 1, 0))      # nn.py:487-492
        l = torch.relu(_norm(l, W, p + "/conv2", use_gn))
        if dil != 1:
            l = F.pad(l, (1, 0, 1, 0))           # nn.py:493-497: the pad follows the norm + ReLU
    else:
        l = conv(l, W[p + "/conv2/W"], dilation=dil, pad=frcnn._same_pad(3, dil))
        l = torch.relu(_norm(l, W, p + "/conv2", use_gn))
    l = _norm(conv(l, W[p + "/conv3/W"]), W, p + "/conv3", use_gn)
    if (p + "/convshortcut/W") in W:
        if stride == 2:
            sc = conv(sc[:, :, :-1, :-1], W[p + "/convshortcut/W"], stride=2)          # nn.py:555-556
        else:
            sc = conv(sc, W[p + "/convshortcut/W"])
        sc = _norm(sc, W, p + "/convshortcut", use_gn)
    return torch.relu(l + sc)


def backbone(x, W, cfg):
    """resnet_fpn_backbone (nn.py:843-944) with use_gn: conv0 -> GN -> ReLU (GNReLU, :616-623), GN bottlenecks."""
    use_gn = getattr(cfg, "use_gn", False)
    h, w = x.shape[2:]
    mult = cfg.fpn_resolution_requirement
    ph = int(math.ceil(h / mult) * mult) - h
    pw = int(math.ceil(w / mult) * mult) - w
    l = F.pad(x, (3, 2 + pw, 3, 2 + ph))
    l = torch.relu(_norm(frcnn._conv(l, W["conv0/W"], stride=2), W, "conv0", use_gn))
    l = F.max_pool2d(F.pad(l, (1, 0, 1, 0)), 3, 2)
    feats = []
    for g, count in enumerate(cfg.resnet_num_block):
        for i in range(count):
            stride = 2 if (g > 0 and i == 0) else 1
            dil = 2 if (g == 3 and cfg.use_dilations and i in range(count)[-3:]) else 1
            l = bottleneck(l, W, "group%d/block%d" % (g, i), stride, dil, use_gn)
        feats.append(l)
    return feats


def fpn(c2345, W, use_gn):
    """fpn_model (nn.py:947-1014) with use_gn: GN of every lateral before the top-down sum (gn_c*, :987-990) and of every
    post-hoc output (gn_p*, :1007-1009); p6 is subsampled from the normalised p5."""
    conv = frcnn._conv
    lat = [conv(c, W["fpn/lateral_1x1_c%d/W" % (i + 2)], bias=W["fpn/lateral_1x1_c%d/b" % (i + 2)])
           for i, c in enumerate(c2345)]
    if use_gn:
        lat = [gn(c, W, "fpn/gn_c%d" % (i + 2)) for i, c in enumerate(lat)]
    sums = []
    for idx, l in enumerate(lat[::-1]):
        if idx > 0:
            l = l + sums[-1].repeat_interleave(2, dim=2).repeat_interleave(2, dim=3)
        sums.append(l)
    p2345 = [conv(c, W["fpn/posthoc_3x3_p%d/W" % (i + 2)], pad=(1, 1, 1, 1), bias=W["fpn/posthoc_3x3_p%d/b" % (i + 2)])
             for i, c in enumerate(sums[::-1])]
    if use_gn:
        p2345 = [gn(c, W, "fpn/gn_p%d" % (i + 2)) for i, c in enumerate(p2345)]
    return p2345 + [p2345[-1][:, :, ::2, ::2]]


def conv_frcnn_head(feat, W, use_gn):
    """conv_frcnn_head (models.py:1110-1125) on the [K,C,7,7] ROI features: 4 x [conv 3x3 SAME + bias, ReLU, then
    GroupNorm per ROI if use_gn] -- the reference's order is ReLU first, GN second, no ReLU after the GN (Tensorpack's own
    GN head normalises first) -- then dense "fc" + ReLU over the NCHW flatten."""
    x = frcnn._t(feat)
    for k in range(4):
        x = torch.relu(frcnn._conv(x, W["fastrcnn/conv%d/W" % k], pad=(1, 1, 1, 1), bias=W["fastrcnn/conv%d/b" % k]))
        if use_gn:
            x = gn(x, W, "fastrcnn/gn%d" % k)
    x = x.reshape(x.shape[0], -1)
    return torch.relu(x @ frcnn._t(W["fastrcnn/fc/W"]) + frcnn._t(W["fastrcnn/fc/b"]))


def fastrcnn_head(feat, W, cfg):
    """oracle.frcnn.fastrcnn_head with the conv head in place of fc6 / fc7 when use_conv_frcnn_head."""
    if not getattr(cfg, "use_conv_frcnn_head", False):
        return _FRCNN["fastrcnn_head"](feat, W, cfg)
    t = frcnn._t
    h = conv_frcnn_head(feat, W, getattr(cfg, "use_gn", False))
    cls = frcnn._np(h @ t(W["fastrcnn/outputs/class/W"]) + t(W["fastrcnn/outputs/class/b"]))
    box = frcnn._np(h @ t(W["fastrcnn/outputs/box/W"]) + t(W["fastrcnn/outputs/box/b"]))
    box = box.reshape(box.shape[0], -1, 4)
    if not cfg.use_frcnn_class_agnostic:
        box = box[:, 1:, :]
    else:
        box = box.repeat(cfg.num_class - 1, axis=1)         # models.py:799-802
    return cls, box.copy(), frcnn._np(h)


_FRCNN = {n: getattr(frcnn, n) for n in ("backbone", "fpn", "fastrcnn_head")}


@contextlib.contextmanager
def graph(cfg):
    """Within the block, oracle.frcnn evaluates the graph `cfg` describes, GroupNorm and conv head included."""
    use_gn = getattr(cfg, "use_gn", False)
    frcnn.backbone = backbone
    frcnn.fpn = lambda c2345, W: fpn(c2345, W, use_gn)
    frcnn.fastrcnn_head = fastrcnn_head
    try:
        yield
    finally:
        for n, f in _FRCNN.items():
            setattr(frcnn, n, f)


def forward(cfg, W, img, stages=True):
    with graph(cfg):
        return frcnn.forward(cfg, W, img, stages=stages)


def forward_multi(cfg, W, imgs, stages=False):
    with graph(cfg):
        return frcnn.forward_multi(cfg, W, imgs, stages=stages)


def forward_givenbox(cfg, W, img, boxes):
    with graph(cfg):
        return frcnn.forward_givenbox(cfg, W, img, boxes)
