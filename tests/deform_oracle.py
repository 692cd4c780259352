"""CPU oracle of the deformable-conv detector, `--use_deformable` (test infrastructure; the product path never imports this).

`oracle.frcnn` restates the plain ResNet bottleneck.  This module restates the deformable branch `resnet_bottleneck` takes
instead (nn.py:470-486) and evaluates the whole graph through `oracle.frcnn`'s own `forward`, `forward_multi` and
`forward_givenbox`:

  which blocks          nn.py:470, 577-581   deformable iff use_deformable, stride 2 and among the last 3 blocks of the
                                             group: res5 block 0 for R50 / R101, block 0 of res3-res5 for (1, 1, 2, 1)
  conv2_offset          nn.py:474-476        3x3 SAME stride-1 conv of conv1's output, bias, no norm, no activation:
                                             [N, 18, H, W], channel 2k the y and 2k + 1 the x offset of tap k
  deformable_conv2d     nn.py:1642-1712      tap k starts at base (2i - 1, 2j - 1) + TAP_BASE[k] and is multiplied by
                                             W[k // 3][k % 3]; the stride-2 conv3d keeps output (i, j) = centre (2i, 2j),
                                             ceil(h / 2) rows; no bias, no norm, no ReLU (activation tf.identity)
  _tf_batch_map_offsets deformable_helper.py:42-137   y = base + dy, clamped to [0, h - 1] (border replication), then
                                             bilinear with floor / ceil corners, y first then x, each op rounded

Batch: each image is sampled at its own offsets, as the single-image graph does.  The reference's batch graph tiles the
coordinates channel-major and samples channel c of image b at the offsets of image (b * C + c) mod B; test_deform_cpu pins
that deviation.  With use_dilations the reference cannot build the graph (the [1, 0] pad after the dilated stride-2 conv
makes the branch one row and column larger than the shortcut): `backbone` raises.  `use_resnext` ignores the flag.  The
arithmetic type follows `oracle.frcnn.exact()`; the stack on `relation_oracle.graph` covers GroupNorm, squeeze-excite and
the relation head too."""
from __future__ import annotations

import contextlib
import math

import torch
import torch.nn.functional as F

import gn_oracle
import relation_oracle
import se_oracle
from oracle import frcnn

# (by, bx) of tap k: reshape(stack(meshgrid(range(3), range(3), "ij")), (-1, 2)) pairs up the [2, 3, 3] stack row-major
TAP_BASE = ((0, 0), (0, 1), (1, 1), (2, 2), (2, 0), (1, 2), (0, 1), (2, 0), (1, 2))

# the last evaluation's offsets [N, Ho, Wo, 18] and samples [N, Ho, Wo, 9, C] per block (float32 numpy), for stage checks
LAST = {}


def use_deformable(cfg):
    return getattr(cfg, "use_deformable", False) and not getattr(cfg, "use_resnext", False)


def is_deformable(cfg, g, i, count):
    stride = 2 if (g > 0 and i == 0) else 1
    return use_deformable(cfg) and stride == 2 and i in range(count)[-3:]


def sample(l, off):
    """The bilinear samples [N, 9, C, Ho, Wo] of l [N, C, H, W] at the offsets off [N, 18, Ho, Wo] of the centres
    (2i, 2j), per image."""
    N, C, H, W = l.shape
    Ho, Wo = off.shape[2:]
    i = torch.arange(Ho, dtype=l.dtype).view(1, Ho, 1)
    j = torch.arange(Wo, dtype=l.dtype).view(1, 1, Wo)
    flat = l.reshape(N, C, H * W)

    def at(yy, xx):
        idx = (yy * W + xx).reshape(N, 1, Ho * Wo).expand(N, C, Ho * Wo)
        return flat.gather(2, idx).reshape(N, C, Ho, Wo)

    out = []
    for k, (by, bx) in enumerate(TAP_BASE):
        y = torch.clamp((2 * i - 1 + by) + off[:, 2 * k], 0, H - 1)
        x = torch.clamp((2 * j - 1 + bx) + off[:, 2 * k + 1], 0, W - 1)
        y0, x0 = torch.floor(y), torch.floor(x)
        y1, x1 = torch.ceil(y).long(), torch.ceil(x).long()
        fy, fx = (y - y0)[:, None], (x - x0)[:, None]
        y0, x0 = y0.long(), x0.long()
        v00, v10, v01, v11 = at(y0, x0), at(y1, x0), at(y0, x1), at(y1, x1)
        t = v00 + (v10 - v00) * fy
        b = v01 + (v11 - v01) * fy
        out.append(t + (b - t) * fx)
    return torch.stack(out, 1)


def offsets(l, W, p):
    """conv2_offset (nn.py:474-476) read at the centres (2i, 2j): [N, 18, ceil(h / 2), ceil(w / 2)]."""
    off = frcnn._conv(l, W[p + "/conv2_offset/W"], pad=(1, 1, 1, 1), bias=W[p + "/conv2_offset/b"])
    return off[:, :, ::2, ::2]


def deform_conv(s, w_hwio):
    """The conv3d of deformable_conv2d on samples s [N, 9, C, Ho, Wo]: tap k times W[k // 3][k % 3]."""
    kh, kw, c, cout = w_hwio.shape
    wt = frcnn._t(w_hwio).reshape(kh * kw, c, cout)
    return torch.einsum("nkchw,kco->nohw", s, wt)


def bottleneck(x, W, p, use_gn, use_se):
    """resnet_bottleneck's deformable branch (nn.py:459-521) + shortcut (nn.py:551-566) + trailing relu: conv2 is the
    deformable conv, with no norm and no ReLU; conv3, squeeze-excite and the shortcut as in se_oracle.bottleneck."""
    conv = frcnn._conv
    norm = gn_oracle._norm
    sc = x
    l = torch.relu(norm(conv(x, W[p + "/conv1/W"]), W, p + "/conv1", use_gn))
    off = offsets(l, W, p)
    s = sample(l, off)
    LAST[p + "/conv2_offset"] = frcnn._np(off.permute(0, 2, 3, 1))
    LAST[p + "/conv2_sample"] = frcnn._np(s.permute(0, 3, 4, 1, 2))
    l = deform_conv(s, W[p + "/conv2/W"])
    l = norm(conv(l, W[p + "/conv3/W"]), W, p + "/conv3", use_gn)
    if use_se:
        l, _ = se_oracle.squeeze_excite(l, W, p)
    sc = conv(sc[:, :, :-1, :-1], W[p + "/convshortcut/W"], stride=2)          # nn.py:555-556
    sc = norm(sc, W, p + "/convshortcut", use_gn)
    return torch.relu(l + sc)


def backbone(x, W, cfg):
    """resnet_fpn_backbone (nn.py:843-944) with the deformable blocks of `cfg`; the others are se_oracle's bottleneck."""
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
            p = "group%d/block%d" % (g, i)
            stride = 2 if (g > 0 and i == 0) else 1
            dil = 2 if (g == 3 and cfg.use_dilations and i in range(count)[-3:]) else 1
            if is_deformable(cfg, g, i, count):
                if dil != 1:
                    raise ValueError("use_deformable with use_dilations: the [1, 0] pad after %s's deformable conv2 "
                                     "(nn.py:493-497) makes the branch larger than the shortcut" % p)
                l = bottleneck(l, W, p, use_gn, use_se)
            else:
                l = se_oracle.bottleneck(l, W, p, stride, dil, use_gn, use_se)
        feats.append(l)
    return feats


@contextlib.contextmanager
def graph(cfg):
    """Within the block, oracle.frcnn evaluates the graph `cfg` describes: GroupNorm, conv head, squeeze-excite, ResNeXt,
    the relation head and deformable blocks."""
    with relation_oracle.graph(cfg):             # restores every oracle.frcnn entry point on exit, backbone included
        if use_deformable(cfg):
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
