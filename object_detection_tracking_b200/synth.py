"""Seeded synthetic weights / frames for the detector, in the reference's variable naming.

No model weights ship with the reference (download links only, README.md:83,105) and
this environment has no network, so parity and the bench run on seeded random
weights.  Names follow the Tensorpack-npz convention the reference loads
(`obj_detect_tracking.py:417-443`; scopes from `nn.py:886-1005`,
`models.py:984-1101`) so a real `.npz` drops in unchanged:

  conv0/W, conv0/bn/{gamma,beta,mean/EMA,variance/EMA}
  group{0..3}/block{i}/{conv1,conv2,conv3,convshortcut}/W (+ bn/..)
  fpn/lateral_1x1_c{2..5}/{W,b}, fpn/posthoc_3x3_p{2..5}/{W,b}
  rpn/conv0/{W,b}, rpn/class/{W,b}, rpn/box/{W,b}
  fastrcnn/fc6/{W,b}, fastrcnn/fc7/{W,b}, fastrcnn/outputs/{class,box}/{W,b}
  use_gn: <conv scope>/gn/{gamma,beta} instead of bn/..., fpn/gn_c{2..5}/.., fpn/gn_p{2..5}/..
  use_conv_frcnn_head: fastrcnn/conv{0..3}/{W,b} (+ fastrcnn/gn{0..3}/.. with use_gn), fastrcnn/fc/{W,b}
  use_se: group{0..3}/block{i}/fc1/{W,b}, fc2/{W,b} (squeeze-excite dense layers)
  use_resnext: conv1 / conv2 at twice the width, conv2/W [3, 3, 2*ch/32, 2*ch] (32 groups), no fc1 / fc2
  add_relation_nn: fastrcnn/RM_r{1,2}/{geo_emb/{W,b}, geo_conv/{W,b}, query_linear/W, key_linear/W, output_linear/W}
  use_att_frcnn_head (class-specific head): fastrcnn/attention/{W,b} [3, 3, 256, 1], [1], fastrcnn/att_trans/{W,b} [256, dim]
  use_small_object_head: fastrcnn/small_objects/small_object_classification_c{1..C}/{W,b} [dim, 2], [2]; with
                         use_so_association fastrcnn/small_objects/person_object_relation/{geo_emb/{W,b}, geo_conv/{W,b},
                         query_linear/W, key_linear/W, output_linear/W}
  use_deformable: <deformable block>/conv2_offset/{W,b} [3, 3, C, 18], [18]; that block's conv2 has no bn / gn
  use_basic_block: conv1/W [3, 3, cin, ch], conv2/W [3, 3, ch, ch], no conv3; convshortcut [1, 1, cin, ch] where cin != ch;
                   laterals read 64 / 128 / 256 / 512 channels

Conv kernels are HWIO (`nn.py:350,367`), dense kernels [in,out] (`nn.py:753`).
The distributions are chosen so activations stay O(1) through 33 residual blocks
and the RPN / class logits have spread (otherwise every proposal collapses and
parity would be vacuous).
"""
from __future__ import annotations

import numpy as np


def _conv_w(rng, k, cin, cout, gain=2.0):
    std = np.sqrt(gain / (k * k * cin))
    return (rng.standard_normal((k, k, cin, cout)) * std).astype(np.float32)


def _bn(rng, w, name, c, gamma_lo=0.8, gamma_hi=1.2):
    w[name + "/bn/gamma"] = rng.uniform(gamma_lo, gamma_hi, c).astype(np.float32)
    w[name + "/bn/beta"] = (rng.standard_normal(c) * 0.05).astype(np.float32)
    w[name + "/bn/mean/EMA"] = (rng.standard_normal(c) * 0.05).astype(np.float32)
    w[name + "/bn/variance/EMA"] = rng.uniform(0.8, 1.2, c).astype(np.float32)


def synth_weights(cfg, seed: int = 1234) -> dict:
    rng = np.random.default_rng(seed)
    w = {}
    w["conv0/W"] = _conv_w(rng, 7, 3, 64)
    _bn(rng, w, "conv0", 64)
    cin = 64
    for g, (feat, count) in enumerate(zip((64, 128, 256, 512), cfg.resnet_num_block)):
        mid, cg = _block_widths(cfg, feat)
        for i in range(count):
            p = "group%d/block%d" % (g, i)
            if _use_basic(cfg):                      # resnet_basicblock (nn.py:439-456)
                w[p + "/conv1/W"] = _conv_w(rng, 3, cin, feat)
                _bn(rng, w, p + "/conv1", feat)
                w[p + "/conv2/W"] = _conv_w(rng, 3, feat, feat)
                _bn(rng, w, p + "/conv2", feat, 0.1, 0.3)              # residual-branch last BN, as conv3's below
                if cin != feat:
                    w[p + "/convshortcut/W"] = _conv_w(rng, 1, cin, feat, gain=1.0)
                    _bn(rng, w, p + "/convshortcut", feat)
                cin = feat
                continue
            w[p + "/conv1/W"] = _conv_w(rng, 1, cin, mid)
            _bn(rng, w, p + "/conv1", mid)
            w[p + "/conv2/W"] = _conv_w(rng, 3, cg, mid)            # fan-in 9 * cg: a grouped filter sees cg channels
            _bn(rng, w, p + "/conv2", mid)
            w[p + "/conv3/W"] = _conv_w(rng, 1, mid, feat * 4)
            # residual-branch last BN: small gamma keeps the running sum bounded
            _bn(rng, w, p + "/conv3", feat * 4, 0.1, 0.3)
            if cin != feat * 4:
                w[p + "/convshortcut/W"] = _conv_w(rng, 1, cin, feat * 4, gain=1.0)
                _bn(rng, w, p + "/convshortcut", feat * 4)
            cin = feat * 4
    nc = cfg.fpn_num_channel
    for i, c in enumerate(_c_channels(cfg)):
        w["fpn/lateral_1x1_c%d/W" % (i + 2)] = _conv_w(rng, 1, c, nc, gain=0.25)
        w["fpn/lateral_1x1_c%d/b" % (i + 2)] = (rng.standard_normal(nc) * 0.02).astype(np.float32)
        w["fpn/posthoc_3x3_p%d/W" % (i + 2)] = _conv_w(rng, 3, nc, nc, gain=(0.12, 0.3, 0.8, 2.5)[i])
        w["fpn/posthoc_3x3_p%d/b" % (i + 2)] = (rng.standard_normal(nc) * 0.02).astype(np.float32)
    na = len(cfg.anchor_ratios)
    w["rpn/conv0/W"] = _conv_w(rng, 3, nc, nc, gain=1.0)
    w["rpn/conv0/b"] = (rng.standard_normal(nc) * 0.02).astype(np.float32)
    w["rpn/class/W"] = (rng.standard_normal((1, 1, nc, na)) * 0.12).astype(np.float32)
    w["rpn/class/b"] = (rng.standard_normal(na) * 0.1).astype(np.float32)
    w["rpn/box/W"] = (rng.standard_normal((1, 1, nc, 4 * na)) * 0.03).astype(np.float32)
    w["rpn/box/b"] = (rng.standard_normal(4 * na) * 0.02).astype(np.float32)
    dim = cfg.fpn_frcnn_fc_head_dim
    fin = nc * 7 * 7
    w["fastrcnn/fc6/W"] = (rng.standard_normal((fin, dim)) * np.sqrt(2.0 / fin)).astype(np.float32)
    w["fastrcnn/fc6/b"] = (rng.standard_normal(dim) * 0.02).astype(np.float32)
    w["fastrcnn/fc7/W"] = (rng.standard_normal((dim, dim)) * np.sqrt(2.0 / dim)).astype(np.float32)
    w["fastrcnn/fc7/b"] = (rng.standard_normal(dim) * 0.02).astype(np.float32)
    ncls = cfg.num_class
    w["fastrcnn/outputs/class/W"] = (rng.standard_normal((dim, ncls)) * 0.15).astype(np.float32)
    w["fastrcnn/outputs/class/b"] = (rng.standard_normal(ncls) * 0.1).astype(np.float32)
    nbox = ncls if not cfg.use_frcnn_class_agnostic else 1
    w["fastrcnn/outputs/box/W"] = (rng.standard_normal((dim, nbox * 4)) * 0.03).astype(np.float32)
    w["fastrcnn/outputs/box/b"] = (rng.standard_normal(nbox * 4) * 0.02).astype(np.float32)
    if getattr(cfg, "add_mask", False):              # maskrcnn_up4conv_head (models.py:1173-1199); drawn last so that the
        md = getattr(cfg, "mrcnn_head_dim", 256)     # detector weights of a seed do not depend on add_mask
        for k in range(4):
            w["maskrcnn/fcn%d/W" % k] = _conv_w(rng, 3, nc if k == 0 else md, md)
            w["maskrcnn/fcn%d/b" % k] = (rng.standard_normal(md) * 0.02).astype(np.float32)
        w["maskrcnn/deconv/W"] = (rng.standard_normal((2, 2, md, md)) * np.sqrt(2.0 / md)).astype(np.float32)   # [kh,kw,out,in]
        w["maskrcnn/deconv/b"] = (rng.standard_normal(md) * 0.02).astype(np.float32)
        w["maskrcnn/conv/W"] = (rng.standard_normal((1, 1, md, ncls - 1)) * np.sqrt(4.0 / md)).astype(np.float32)
        w["maskrcnn/conv/b"] = (rng.standard_normal(ncls - 1) * 0.5).astype(np.float32)
    # The GroupNorm and conv-head variables are drawn after everything above, and the BatchNorm / fc6 / fc7 values they
    # replace are still drawn (then dropped): every weight a seed shares between the model families stays the same.
    if getattr(cfg, "use_gn", False):                # group_norm (nn.py:81-108) instead of every backbone BatchNorm
        for k in [k for k in w if "/bn/" in k]:
            del w[k]
        for scope, c, last in _backbone_norm_scopes(cfg):
            # residual-branch last GN: small gamma keeps the running sum bounded (as for BN above)
            _gn(rng, w, scope + "/gn", c, 0.1 if last else 0.8, 0.3 if last else 1.2)
        for i in range(4):
            _gn(rng, w, "fpn/gn_c%d" % (i + 2), nc)
            _gn(rng, w, "fpn/gn_p%d" % (i + 2), nc)
    if getattr(cfg, "use_conv_frcnn_head", False):   # conv_frcnn_head (models.py:1110-1125) instead of fc6 / fc7
        hd = int(getattr(cfg, "conv_frcnn_head_dim", 256))
        for k in ("fastrcnn/fc6/W", "fastrcnn/fc6/b", "fastrcnn/fc7/W", "fastrcnn/fc7/b"):
            del w[k]
        for k in range(4):
            w["fastrcnn/conv%d/W" % k] = _conv_w(rng, 3, nc if k == 0 else hd, hd)
            w["fastrcnn/conv%d/b" % k] = (rng.standard_normal(hd) * 0.02).astype(np.float32)
            if getattr(cfg, "use_gn", False):
                _gn(rng, w, "fastrcnn/gn%d" % k, hd)
        fin = hd * 7 * 7
        w["fastrcnn/fc/W"] = (rng.standard_normal((fin, dim)) * np.sqrt(2.0 / fin)).astype(np.float32)
        w["fastrcnn/fc/b"] = (rng.standard_normal(dim) * 0.02).astype(np.float32)
    # The squeeze-excite variables come last, so every other array of a seed is the same with and without use_se.
    if _use_se(cfg):                                 # resnet_bottleneck's fc1 / fc2 (nn.py:506-519)
        for p, c in _se_blocks(cfg):
            # channel means of conv3's BN output are O(0.1): fc1's gain and bias keep most hidden units live and
            # image-dependent; fc2's bias spread puts the gates around 0.2-0.8 (saturated gates would make parity vacuous)
            nr = c // 16
            w[p + "/fc1/W"] = (rng.standard_normal((c, nr)) * np.sqrt(8.0 / c)).astype(np.float32)
            w[p + "/fc1/b"] = rng.uniform(0.0, 0.1, nr).astype(np.float32)
            w[p + "/fc2/W"] = (rng.standard_normal((nr, c)) * np.sqrt(2.0 / nr)).astype(np.float32)
            w[p + "/fc2/b"] = (rng.standard_normal(c) * 0.4).astype(np.float32)
    # The relation modules come after everything else, so every other array of a seed is the same with and without them.
    if _use_relation(cfg):                           # relation_network (nn.py:115-190) of RM_r1 / RM_r2
        for name, shape in _relation_shapes(cfg).items():
            fan_in = int(np.prod(shape[:-1]))
            # geo_emb: the log-ratio features span ~[-7, 3], so a gain well under 1 keeps tanh off its rails; geo_conv
            # without a bias offset puts about half of the (i, g, j) weights under the 1e-6 clamp and the rest in
            # ~[1e-3, 2]; query / key give per-head logits of a few units (peaked, not one-hot rows); output_linear's
            # unit gain over the 16 averaged heads makes the module's output the size of h
            std = {"geo_emb/W": 0.3, "geo_emb/b": 0.1, "geo_conv/W": np.sqrt(1.0 / 64), "geo_conv/b": 0.05,
                   "query_linear/W": np.sqrt(2.0 / fan_in), "key_linear/W": np.sqrt(2.0 / fan_in),
                   "output_linear/W": np.sqrt(1.0 / fan_in)}[name.split("/", 2)[2]]
            w[name] = (rng.standard_normal(shape) * std).astype(np.float32)
    # The deformable blocks' conv2 norm is drawn above and dropped here, and their offset convs are drawn last: every array
    # a seed shares with the plain model is the same with and without use_deformable.
    for p, c in deformable_blocks(cfg):              # resnet_bottleneck's deformable branch (nn.py:470-486)
        for k in [k for k in w if k.startswith(p + "/conv2/bn/") or k.startswith(p + "/conv2/gn/")]:
            del w[k]
        # conv1's output is ReLU'd BN output: a fan-in gain of 2 and a bias spread of 0.5 give offsets of one to a few
        # pixels -- nearly every sample fractional, a fifth to two thirds of the offsets beyond one pixel, the border
        # taps clamped (test_deform_cpu states the thresholds)
        w[p + "/conv2_offset/W"] = _conv_w(rng, 3, c, 18)
        w[p + "/conv2_offset/b"] = (rng.standard_normal(18) * 0.5).astype(np.float32)
    # The attention branch draws from a stream of its own, so every other array of a seed is the same with and without it.
    if _use_att(cfg):                                # fastrcnn_2fc_head's attention branch (models.py:1064-1089)
        arng = np.random.default_rng([seed, 0x617474])
        nc = cfg.fpn_num_channel
        # the attention conv's values never change a finite result (its softmax runs over one channel); they only have to
        # pass the load check.  att_trans reads the sum of 49 cells: a fan-in gain of 1 over 49 * sqrt(256) makes its
        # output about the size of one mean cell, about half of hidden's norm, with about half of its units active
        w["fastrcnn/attention/W"] = (arng.standard_normal((3, 3, nc, 1)) * 0.05).astype(np.float32)
        w["fastrcnn/attention/b"] = (arng.standard_normal(1) * 0.1).astype(np.float32)
        w["fastrcnn/att_trans/W"] = (arng.standard_normal((nc, dim)) * (1.0 / (49.0 * np.sqrt(nc)))).astype(np.float32)
        w["fastrcnn/att_trans/b"] = (arng.standard_normal(dim) * 0.1).astype(np.float32)
    # The small-object branch draws from a stream of its own too.
    if getattr(cfg, "use_small_object_head", False):  # models.py:652-692
        srng = np.random.default_rng([seed, 0x736f])
        for name, shape in _so_shapes(cfg).items():
            fan_in = int(np.prod(shape[:-1]))
            # the classification layers: a unit fan-in gain gives logits of about one unit of either sign, so both the
            # score filter and negative final "probs" are exercised; the association follows the relation modules' choice
            rel = name.startswith(_SO_REL)
            std = ({"geo_emb/W": 0.3, "geo_emb/b": 0.1, "geo_conv/W": np.sqrt(1.0 / 64), "geo_conv/b": 0.05,
                    "query_linear/W": np.sqrt(2.0 / fan_in), "key_linear/W": np.sqrt(2.0 / fan_in),
                    "output_linear/W": np.sqrt(1.0 / fan_in)}[name[len(_SO_REL):]] if rel else
                   {"W": np.sqrt(1.0 / fan_in), "b": 0.5}[name.rsplit("/", 1)[1]])
            w[name] = (srng.standard_normal(shape) * std).astype(np.float32)
    return w


def _block_widths(cfg, feat):
    """(conv1 / conv2 width, input channels per conv2 filter) of a block with ch_out = feat: the ResNet bottleneck's
    (feat, feat) (nn.py:478-497), or ResNeXt 32x4d's (2 * feat, 2 * feat / 32) (nn.py:532-540)."""
    if getattr(cfg, "use_resnext", False):
        return 2 * feat, 2 * feat // 32
    return feat, feat


def _use_basic(cfg):
    """use_basic_block (--resnet34 / --resnet18) selects resnet_basicblock, unless use_resnext reassigns block_func after it
    (nn.py:864-868)."""
    return getattr(cfg, "use_basic_block", False) and not getattr(cfg, "use_resnext", False)


def _c_channels(cfg):
    """Channels of c2..c5: the blocks' output width, ch_out for the basic block and 4 * ch_out for the bottlenecks."""
    return (64, 128, 256, 512) if _use_basic(cfg) else (256, 512, 1024, 2048)


def _use_se(cfg):
    """use_se selects squeeze-excite in resnet_bottleneck only: the ResNeXt and basic blocks have no SE branch
    (nn.py:439-456, 524-549)."""
    return getattr(cfg, "use_se", False) and not getattr(cfg, "use_resnext", False) and not _use_basic(cfg)


def _use_relation(cfg):
    """add_relation_nn builds RM_r1 / RM_r2 in the 2fc head only: use_conv_frcnn_head takes precedence (models.py:1038-1041)."""
    return getattr(cfg, "add_relation_nn", False) and not getattr(cfg, "use_conv_frcnn_head", False)


def _relation_shapes(cfg):
    """Name -> shape of the relation modules' variables (nn.py:115-190, group 16, geo_feat_dim 64), in graph order."""
    dim = cfg.fpn_frcnn_fc_head_dim
    sh = {}
    for m in ("RM_r1", "RM_r2"):
        p = "fastrcnn/%s/" % m
        sh.update({p + "geo_emb/W": (4, 64), p + "geo_emb/b": (64,), p + "geo_conv/W": (1, 1, 64, 16),
                   p + "geo_conv/b": (16,), p + "query_linear/W": (dim, dim), p + "key_linear/W": (dim, dim),
                   p + "output_linear/W": (16 * dim, dim)})
    return sh


def _use_att(cfg):
    """use_att_frcnn_head adds the attention branch to the class-specific heads only: fastrcnn_2fc_head_class_agnostic has
    none (models.py:1126-1170)."""
    return getattr(cfg, "use_att_frcnn_head", False) and not cfg.use_frcnn_class_agnostic


def _att_shapes(cfg):
    """Name -> shape of the attention branch's variables (models.py:1075-1088): the 3x3 one-channel conv and the dense
    att_trans over the channel vector."""
    nc, dim = cfg.fpn_num_channel, cfg.fpn_frcnn_fc_head_dim
    return {"fastrcnn/attention/W": (3, 3, nc, 1), "fastrcnn/attention/b": (1,), "fastrcnn/att_trans/W": (nc, dim),
            "fastrcnn/att_trans/b": (dim,)}


_SO_REL = "fastrcnn/small_objects/person_object_relation/"


def _so_shapes(cfg):
    """Name -> shape of the small-object branch's own variables (models.py:652-692): one [D, 2] classification per class
    of small_objects and, with use_so_association, the shared person_object_relation (nn.py:194-270).  fc6 / fc7 are the
    box head's own (AUTO_REUSE)."""
    dim = cfg.fpn_frcnn_fc_head_dim
    sh = {}
    for i in range(len(cfg.small_objects)):
        p = "fastrcnn/small_objects/small_object_classification_c%d/" % (i + 1)
        sh.update({p + "W": (dim, 2), p + "b": (2,)})
    if cfg.use_so_association:
        p = _SO_REL
        sh.update({p + "geo_emb/W": (4, 64), p + "geo_emb/b": (64,), p + "geo_conv/W": (1, 1, 64, 16),
                   p + "geo_conv/b": (16,), p + "query_linear/W": (dim, dim), p + "key_linear/W": (dim, dim),
                   p + "output_linear/W": (16 * dim, dim)})
    return sh


def deformable_blocks(cfg):
    """(block scope, conv2 channels) of every deformable block, in graph order.  resnet_group passes deformable to the last
    3 blocks of a group (nn.py:577-581) and resnet_bottleneck uses it at stride 2 only (nn.py:470), so a group qualifies
    when its block 0 has stride 2 (groups 1-3) and the group has at most 3 blocks.  The ResNeXt and basic blocks have no
    deformable branch."""
    if not getattr(cfg, "use_deformable", False) or getattr(cfg, "use_resnext", False) or _use_basic(cfg):
        return []
    return [("group%d/block0" % g, feat) for g, (feat, count) in enumerate(zip((64, 128, 256, 512), cfg.resnet_num_block))
            if g > 0 and count <= 3]


def _se_blocks(cfg):
    """(block scope, gated channels 4 * ch_out) of every bottleneck, in graph order."""
    return [("group%d/block%d" % (g, i), feat * 4)
            for g, (feat, count) in enumerate(zip((64, 128, 256, 512), cfg.resnet_num_block)) for i in range(count)]


def _gn(rng, w, name, c, gamma_lo=0.8, gamma_hi=1.2):
    w[name + "/gamma"] = rng.uniform(gamma_lo, gamma_hi, c).astype(np.float32)
    w[name + "/beta"] = (rng.standard_normal(c) * 0.05).astype(np.float32)


def _backbone_norm_scopes(cfg):
    """(conv scope, channels, is the residual branch's last conv) of every normalised backbone conv, in graph order."""
    out = [("conv0", 64, False)]
    cin = 64
    for g, (feat, count) in enumerate(zip((64, 128, 256, 512), cfg.resnet_num_block)):
        mid = _block_widths(cfg, feat)[0]
        for i in range(count):
            p = "group%d/block%d" % (g, i)
            if _use_basic(cfg):
                out += [(p + "/conv1", feat, False), (p + "/conv2", feat, True)]
            else:
                out += [(p + "/conv1", mid, False), (p + "/conv2", mid, False), (p + "/conv3", feat * 4, True)]
            cout = _c_channels(cfg)[g]
            if cin != cout:
                out.append((p + "/convshortcut", cout, False))
            cin = cout
    return out


def frcnn_weight_shapes(cfg) -> dict:
    """Name -> shape of every variable the inference graph reads, in the reference's checkpoint naming (Tensorpack-style:
    conv2d `W`/`b` nn.py:367,376, BatchNorm `gamma`/`beta`/`mean/EMA`/`variance/EMA` nn.py:1739-1826, dense nn.py:762;
    scopes: nn.py:843-944 resnet, :947-1014 fpn, models.py:979-1009 rpn, :1030-1108 fastrcnn).  Used by the importer
    (backend.check_weights) to refuse incomplete or mis-shaped checkpoints before anything reaches the device."""
    sh = {}

    def conv(name, k, cin, cout, bias=False):
        sh[name + "/W"] = (k, k, cin, cout)
        if bias:
            sh[name + "/b"] = (cout,)

    gn = getattr(cfg, "use_gn", False)

    def bn(name, c):
        if gn:                                       # group_norm "<scope>/gn/{gamma,beta}" (nn.py:97-102, 591-603)
            for k in ("gamma", "beta"):
                sh["%s/gn/%s" % (name, k)] = (c,)
            return
        for k in ("gamma", "beta", "mean/EMA", "variance/EMA"):
            sh["%s/bn/%s" % (name, k)] = (c,)

    conv("conv0", 7, 3, 64)
    bn("conv0", 64)
    deform = dict(deformable_blocks(cfg))
    cin = 64
    for g, (feat, count) in enumerate(zip((64, 128, 256, 512), cfg.resnet_num_block)):
        mid, cg = _block_widths(cfg, feat)
        cout = _c_channels(cfg)[g]
        for i in range(count):
            p = "group%d/block%d" % (g, i)
            if _use_basic(cfg):                      # resnet_basicblock: two 3x3 convs (nn.py:443-450)
                convs = (("conv1", 3, cin, feat), ("conv2", 3, feat, feat))
            else:
                convs = (("conv1", 1, cin, mid), ("conv2", 3, cg, mid), ("conv3", 1, mid, feat * 4))
            for name, k, ci, co in convs:
                conv("%s/%s" % (p, name), k, ci, co)
                if not (name == "conv2" and p in deform):    # deformable_conv2d: no norm (nn.py:483-485)
                    bn("%s/%s" % (p, name), co)
            if p in deform:                          # conv2_offset: 3x3 SAME with bias (nn.py:474-476)
                conv(p + "/conv2_offset", 3, mid, 18, bias=True)
            if cin != cout:                          # resnet_shortcut (nn.py:551-566)
                conv(p + "/convshortcut", 1, cin, cout)
                bn(p + "/convshortcut", cout)
            cin = cout
    if _use_se(cfg):                                 # dense fc1 / fc2 of every bottleneck (nn.py:509-514, 762)
        for p, c in _se_blocks(cfg):
            sh[p + "/fc1/W"] = (c, c // 16)
            sh[p + "/fc1/b"] = (c // 16,)
            sh[p + "/fc2/W"] = (c // 16, c)
            sh[p + "/fc2/b"] = (c,)
    nc = cfg.fpn_num_channel
    for i, c in enumerate(_c_channels(cfg)):
        conv("fpn/lateral_1x1_c%d" % (i + 2), 1, c, nc, bias=True)
        conv("fpn/posthoc_3x3_p%d" % (i + 2), 3, nc, nc, bias=True)
        if gn:                                       # gn_c* / gn_p* (nn.py:987-990, 1007-1009)
            for s in ("gn_c%d" % (i + 2), "gn_p%d" % (i + 2)):
                sh["fpn/%s/gamma" % s] = (nc,)
                sh["fpn/%s/beta" % s] = (nc,)
    na = len(cfg.anchor_ratios)
    conv("rpn/conv0", 3, nc, nc, bias=True)
    conv("rpn/class", 1, nc, na, bias=True)
    conv("rpn/box", 1, nc, 4 * na, bias=True)
    dim = cfg.fpn_frcnn_fc_head_dim
    nbox = 1 if cfg.use_frcnn_class_agnostic else cfg.num_class
    if getattr(cfg, "use_conv_frcnn_head", False):   # conv_frcnn_head (models.py:1110-1125)
        hd = int(getattr(cfg, "conv_frcnn_head_dim", 256))
        for k in range(4):
            conv("fastrcnn/conv%d" % k, 3, nc if k == 0 else hd, hd, bias=True)
            if gn:
                sh["fastrcnn/gn%d/gamma" % k] = (hd,)
                sh["fastrcnn/gn%d/beta" % k] = (hd,)
        hidden = (("fastrcnn/fc", hd * 49, dim),)
    else:
        hidden = (("fastrcnn/fc6", nc * 49, dim), ("fastrcnn/fc7", dim, dim))
    for name, fin, fout in hidden + (("fastrcnn/outputs/class", dim, cfg.num_class), ("fastrcnn/outputs/box", dim, nbox * 4)):
        sh[name + "/W"] = (fin, fout)
        sh[name + "/b"] = (fout,)
    if _use_relation(cfg):                           # fastrcnn_2fc_head(_class_agnostic) (models.py:1044-1054, 1139-1148)
        sh.update(_relation_shapes(cfg))
    if _use_att(cfg):                                # fastrcnn_2fc_head (models.py:1064-1089), with either hidden variant
        sh.update(_att_shapes(cfg))
    if getattr(cfg, "use_small_object_head", False):  # models.py:652-692
        sh.update(_so_shapes(cfg))
    if getattr(cfg, "add_mask", False):              # models.py:1173-1199; Conv2DTranspose kernel is [kh, kw, out, in]
        md = getattr(cfg, "mrcnn_head_dim", 256)
        for k in range(4):
            conv("maskrcnn/fcn%d" % k, 3, nc if k == 0 else md, md, bias=True)
        sh["maskrcnn/deconv/W"] = (2, 2, md, md)
        sh["maskrcnn/deconv/b"] = (md,)
        conv("maskrcnn/conv", 1, md, cfg.num_class - 1, bias=True)
    return sh


def synth_frame(h: int, w: int, seed: int = 0, n_rects: int = 4) -> np.ndarray:
    """uint8 [h, w, 3] BGR frame: low-pass noise + a few flat rectangles + white noise
    (SURVEY.md section 8d), so RPN logits have spatial structure."""
    rng = np.random.default_rng(seed)
    gh, gw = max(2, h // 16), max(2, w // 16)
    coarse = rng.uniform(0, 255, (gh, gw, 3)).astype(np.float32)
    # separable bilinear up-sampling of the coarse grid (no cv2 dependency)
    ys = np.linspace(0, gh - 1, h, dtype=np.float32)
    xs = np.linspace(0, gw - 1, w, dtype=np.float32)
    y0 = np.floor(ys).astype(np.int64); y1 = np.minimum(y0 + 1, gh - 1); fy = (ys - y0)[:, None, None]
    x0 = np.floor(xs).astype(np.int64); x1 = np.minimum(x0 + 1, gw - 1); fx = (xs - x0)[None, :, None]
    rows = coarse[y0] * (1 - fy) + coarse[y1] * fy
    img = rows[:, x0] * (1 - fx) + rows[:, x1] * fx
    for _ in range(n_rects):
        rh, rw = int(rng.integers(h // 8, h // 2)), int(rng.integers(w // 10, w // 3))
        ry, rx = int(rng.integers(0, h - rh)), int(rng.integers(0, w - rw))
        img[ry:ry + rh, rx:rx + rw] = rng.uniform(0, 255, 3).astype(np.float32)
    img += rng.uniform(-10, 10, img.shape).astype(np.float32)
    return np.clip(img, 0, 255).astype(np.uint8)


def osnet_param_shapes() -> dict:
    """Parameter / buffer names and shapes of torchreid's osnet_x1_0 state_dict (osnet.py:282-438, :522-534),
    minus the unused classifier."""
    shapes = {}

    def bn(prefix, c):
        for k in ("weight", "bias", "running_mean", "running_var"):
            shapes[prefix + "." + k] = (c,)

    def light(prefix, c):
        shapes[prefix + ".conv1.weight"] = (c, c, 1, 1)
        shapes[prefix + ".conv2.weight"] = (c, 1, 3, 3)
        bn(prefix + ".bn", c)

    def osblock(prefix, cin, cout):
        mid = cout // 4
        shapes[prefix + ".conv1.conv.weight"] = (mid, cin, 1, 1)
        bn(prefix + ".conv1.bn", mid)
        light(prefix + ".conv2a", mid)
        for name, n in (("conv2b", 2), ("conv2c", 3), ("conv2d", 4)):
            for j in range(n):
                light("%s.%s.%d" % (prefix, name, j), mid)
        shapes[prefix + ".gate.fc1.weight"] = (mid // 16, mid, 1, 1)
        shapes[prefix + ".gate.fc1.bias"] = (mid // 16,)
        shapes[prefix + ".gate.fc2.weight"] = (mid, mid // 16, 1, 1)
        shapes[prefix + ".gate.fc2.bias"] = (mid,)
        shapes[prefix + ".conv3.conv.weight"] = (cout, mid, 1, 1)
        bn(prefix + ".conv3.bn", cout)
        if cin != cout:
            shapes[prefix + ".downsample.conv.weight"] = (cout, cin, 1, 1)
            bn(prefix + ".downsample.bn", cout)

    shapes["conv1.conv.weight"] = (64, 3, 7, 7)
    bn("conv1.bn", 64)
    chans = (64, 256, 384, 512)
    for s in range(3):
        name = "conv%d" % (s + 2)
        osblock(name + ".0", chans[s], chans[s + 1])
        osblock(name + ".1", chans[s + 1], chans[s + 1])
        if s < 2:
            shapes[name + ".2.0.conv.weight"] = (chans[s + 1], chans[s + 1], 1, 1)
            bn(name + ".2.0.bn", chans[s + 1])
    shapes["conv5.conv.weight"] = (512, 512, 1, 1)
    bn("conv5.bn", 512)
    shapes["fc.0.weight"] = (512, 512)
    shapes["fc.0.bias"] = (512,)
    bn("fc.1", 512)
    return shapes


def synth_osnet_state(seed: int = 4321) -> dict:
    """Seeded float32 state_dict for osnet_x1_0 with non-trivial BatchNorm statistics (a fresh torch model has
    mean 0 / var 1 / gamma 1, which would not exercise the BN folding)."""
    rng = np.random.default_rng(seed)
    out = {}
    for name, shp in osnet_param_shapes().items():
        if name.endswith("running_var"):
            v = rng.uniform(0.6, 1.4, shp)
        elif name.endswith("running_mean"):
            v = rng.standard_normal(shp) * 0.1
        elif name.endswith("conv3.bn.weight"):              # residual-branch BN: small gamma keeps the sum bounded
            v = rng.uniform(0.1, 0.3, shp)
        elif name.endswith("bn.weight") or name == "fc.1.weight":
            v = rng.uniform(0.7, 1.3, shp)
        elif name.endswith("bias"):
            v = rng.standard_normal(shp) * 0.05
        elif len(shp) == 4 and shp[1] == 1:                 # depthwise 3x3: fan_in 9
            v = rng.standard_normal(shp) * np.sqrt(1.0 / 9)
        elif len(shp) >= 2:
            fan_in = int(np.prod(shp[1:]))
            relu_follows = name.endswith("conv1.conv.weight") or name.endswith(".2.0.conv.weight") \
                or name in ("conv5.conv.weight", "fc.0.weight")
            v = rng.standard_normal(shp) * np.sqrt((2.0 if relu_follows else 1.0) / fan_in)
        else:
            v = rng.standard_normal(shp) * 0.05
        out[name] = v.astype(np.float32)
    return out


# torchreid's OSNet family (osnet.py:522-598, osnet_ain.py:524-541): channels, stem InstanceNorm, block kind of each
# stage's two blocks ("plain" OSBlock, "ibn" = OSBlock with IN after the residual, "inin" = OSBlockINin) and whether the
# module names are osnet_ain.py's (conv2.{t}.layers.{j} streams, poolN.0 transitions)
OSNET_FAMILY = {
    "osnet_x1_0": dict(ch=(64, 256, 384, 512), stem_in=False, kinds=(("plain",) * 2,) * 3, ain=False),
    "osnet_x0_75": dict(ch=(48, 192, 288, 384), stem_in=False, kinds=(("plain",) * 2,) * 3, ain=False),
    "osnet_x0_5": dict(ch=(32, 128, 192, 256), stem_in=False, kinds=(("plain",) * 2,) * 3, ain=False),
    "osnet_x0_25": dict(ch=(16, 64, 96, 128), stem_in=False, kinds=(("plain",) * 2,) * 3, ain=False),
    "osnet_ibn_x1_0": dict(ch=(64, 256, 384, 512), stem_in=True,
                           kinds=(("ibn", "ibn"), ("plain", "plain"), ("plain", "plain")), ain=False),
    "osnet_ain_x1_0": dict(ch=(64, 256, 384, 512), stem_in=True,
                           kinds=(("inin", "inin"), ("plain", "inin"), ("inin", "plain")), ain=True),
}


def osnet_family_param_shapes(name: str) -> dict:
    """Parameter / buffer names and shapes of torchreid's `name` state_dict (one of OSNET_FAMILY), minus the unused
    classifier.  InstanceNorm2d(affine=True) layers hold only .weight and .bias."""
    spec = OSNET_FAMILY[name]
    ch, ain = spec["ch"], spec["ain"]
    shapes = {}

    def bn(prefix, c):
        for k in ("weight", "bias", "running_mean", "running_var"):
            shapes[prefix + "." + k] = (c,)

    def inorm(prefix, c):
        shapes[prefix + ".weight"] = (c,)
        shapes[prefix + ".bias"] = (c,)

    def light(prefix, c):
        shapes[prefix + ".conv1.weight"] = (c, c, 1, 1)
        shapes[prefix + ".conv2.weight"] = (c, 1, 3, 3)
        bn(prefix + ".bn", c)

    def osblock(prefix, cin, cout, kind):
        mid = cout // 4
        shapes[prefix + ".conv1.conv.weight"] = (mid, cin, 1, 1)
        bn(prefix + ".conv1.bn", mid)
        for t in range(4):
            for j in range(t + 1):
                if ain:
                    light("%s.conv2.%d.layers.%d" % (prefix, t, j), mid)
                else:
                    light("%s.conv2%s" % (prefix, "abcd"[t]) + ("" if t == 0 else ".%d" % j), mid)
        shapes[prefix + ".gate.fc1.weight"] = (mid // 16, mid, 1, 1)
        shapes[prefix + ".gate.fc1.bias"] = (mid // 16,)
        shapes[prefix + ".gate.fc2.weight"] = (mid, mid // 16, 1, 1)
        shapes[prefix + ".gate.fc2.bias"] = (mid,)
        shapes[prefix + ".conv3.conv.weight"] = (cout, mid, 1, 1)
        if kind != "inin":
            bn(prefix + ".conv3.bn", cout)
        if cin != cout:
            shapes[prefix + ".downsample.conv.weight"] = (cout, cin, 1, 1)
            bn(prefix + ".downsample.bn", cout)
        if kind != "plain":
            inorm(prefix + ".IN", cout)

    shapes["conv1.conv.weight"] = (ch[0], 3, 7, 7)
    (inorm if spec["stem_in"] else bn)("conv1.bn", ch[0])
    for s in range(3):
        name_s = "conv%d" % (s + 2)
        osblock(name_s + ".0", ch[s], ch[s + 1], spec["kinds"][s][0])
        osblock(name_s + ".1", ch[s + 1], ch[s + 1], spec["kinds"][s][1])
        if s < 2:
            t = "pool%d.0" % (s + 2) if ain else name_s + ".2.0"
            shapes[t + ".conv.weight"] = (ch[s + 1], ch[s + 1], 1, 1)
            bn(t + ".bn", ch[s + 1])
    shapes["conv5.conv.weight"] = (ch[3], ch[3], 1, 1)
    bn("conv5.bn", ch[3])
    shapes["fc.0.weight"] = (512, ch[3])
    shapes["fc.0.bias"] = (512,)
    bn("fc.1", 512)
    return shapes


def osnet_family_in_layers(name: str) -> list:
    """The InstanceNorm2d scopes of `name`, in forward order: the norm layers without running statistics."""
    shapes = osnet_family_param_shapes(name)
    return [k[:-7] for k, s in shapes.items()
            if k.endswith(".weight") and len(s) == 1 and k[:-7] + ".running_mean" not in shapes]


def synth_osnet_family_state(name: str, seed: int = 4321) -> dict:
    """Seeded float32 state_dict for `name` (one of OSNET_FAMILY), drawn as synth_osnet_state draws osnet_x1_0's, with
    InstanceNorm gamma ~ U(0.8, 1.2) and beta ~ N(0, 0.05)."""
    rng = np.random.default_rng(seed)
    shapes = osnet_family_param_shapes(name)
    in_scopes = set(osnet_family_in_layers(name))
    out = {}
    for k, shp in shapes.items():
        scope = k.rsplit(".", 1)[0]
        if scope in in_scopes:
            v = rng.uniform(0.8, 1.2, shp) if k.endswith(".weight") else rng.standard_normal(shp) * 0.05
        elif k.endswith("running_var"):
            v = rng.uniform(0.6, 1.4, shp)
        elif k.endswith("running_mean"):
            v = rng.standard_normal(shp) * 0.1
        elif k.endswith("conv3.bn.weight"):              # residual-branch BN: small gamma keeps the sum bounded
            v = rng.uniform(0.1, 0.3, shp)
        elif k.endswith("bn.weight") or k == "fc.1.weight":
            v = rng.uniform(0.7, 1.3, shp)
        elif k.endswith("bias"):
            v = rng.standard_normal(shp) * 0.05
        elif len(shp) == 4 and shp[1] == 1:              # depthwise 3x3: fan_in 9
            v = rng.standard_normal(shp) * np.sqrt(1.0 / 9)
        elif len(shp) >= 2:
            fan_in = int(np.prod(shp[1:]))
            relu_follows = k.endswith("conv1.conv.weight") or k.endswith(".2.0.conv.weight") \
                or (k.startswith("pool") and k.endswith(".0.conv.weight")) or k in ("conv5.conv.weight", "fc.0.weight")
            v = rng.standard_normal(shp) * np.sqrt((2.0 if relu_follows else 1.0) / fan_in)
        else:
            v = rng.standard_normal(shp) * 0.05
        out[k] = v.astype(np.float32)
    return out


def resnet101_reid_param_shapes() -> dict:
    """Parameter / buffer names and shapes of torchreid's resnet101 state_dict (torchreid/models/resnet.py:157-290,
    441-455: Bottleneck [3, 4, 23, 3], last_stride 2), minus the unused classifier."""
    shapes = {"conv1.weight": (64, 3, 7, 7)}

    def bn(prefix, c):
        for k in ("weight", "bias", "running_mean", "running_var"):
            shapes[prefix + "." + k] = (c,)

    bn("bn1", 64)
    cin = 64
    for li, (n, planes) in enumerate(zip((3, 4, 23, 3), (64, 128, 256, 512))):
        for bi in range(n):
            p = "layer%d.%d" % (li + 1, bi)
            shapes[p + ".conv1.weight"] = (planes, cin, 1, 1)
            bn(p + ".bn1", planes)
            shapes[p + ".conv2.weight"] = (planes, planes, 3, 3)
            bn(p + ".bn2", planes)
            shapes[p + ".conv3.weight"] = (planes * 4, planes, 1, 1)
            bn(p + ".bn3", planes * 4)
            if bi == 0:
                shapes[p + ".downsample.0.weight"] = (planes * 4, cin, 1, 1)
                bn(p + ".downsample.1", planes * 4)
            cin = planes * 4
    return shapes


def synth_resnet101_reid_state(seed: int = 2468) -> dict:
    """Seeded float32 state_dict for torchreid's resnet101 with non-trivial BatchNorm statistics; the last BN of every
    residual branch gets a small gamma so that 33 stacked blocks keep activations O(1) (fp16-plane range, DESIGN 3)."""
    rng = np.random.default_rng(seed)
    out = {}
    for name, shp in resnet101_reid_param_shapes().items():
        if name.endswith("running_var"):
            v = rng.uniform(0.6, 1.4, shp)
        elif name.endswith("running_mean"):
            v = rng.standard_normal(shp) * 0.1
        elif name.endswith("bn3.weight"):
            v = rng.uniform(0.1, 0.3, shp)
        elif name.endswith(".weight") and len(shp) == 1:
            v = rng.uniform(0.7, 1.3, shp)
        elif name.endswith("bias"):
            v = rng.standard_normal(shp) * 0.05
        else:
            fan_in = int(np.prod(shp[1:]))
            gain = 1.0 if (name.endswith("conv3.weight") or "downsample" in name) else 2.0
            v = rng.standard_normal(shp) * np.sqrt(gain / fan_in)
        out[name] = v.astype(np.float32)
    return out


# torchreid's ResNet family (resnet.py:393-530, resnet_ibn_a.py:283-289, resnet_ibn_b.py:268-274): block ("basic" /
# "bottleneck"), blocks per layer, conv2 groups and width per group, layer4's stride, fc_dims[0] (0 = none) and the IBN
# kind ("a": bn1 of layer1-3 is IN of the first half beside BN of the rest; "b": IN stem, IN after the residual of the
# last block of layer1 and layer2)
RESNET_FAMILY = {
    "resnet18": dict(block="basic", layers=(2, 2, 2, 2), groups=1, width=64, last_stride=2, fc=0, ibn=None),
    "resnet34": dict(block="basic", layers=(3, 4, 6, 3), groups=1, width=64, last_stride=2, fc=0, ibn=None),
    "resnet50": dict(block="bottleneck", layers=(3, 4, 6, 3), groups=1, width=64, last_stride=2, fc=0, ibn=None),
    "resnet101": dict(block="bottleneck", layers=(3, 4, 23, 3), groups=1, width=64, last_stride=2, fc=0, ibn=None),
    "resnet152": dict(block="bottleneck", layers=(3, 8, 36, 3), groups=1, width=64, last_stride=2, fc=0, ibn=None),
    "resnext50_32x4d": dict(block="bottleneck", layers=(3, 4, 6, 3), groups=32, width=4, last_stride=2, fc=0, ibn=None),
    "resnext101_32x8d": dict(block="bottleneck", layers=(3, 4, 23, 3), groups=32, width=8, last_stride=2, fc=0,
                             ibn=None),
    "resnet50_fc512": dict(block="bottleneck", layers=(3, 4, 6, 3), groups=1, width=64, last_stride=1, fc=512, ibn=None),
    "resnet50_ibn_a": dict(block="bottleneck", layers=(3, 4, 6, 3), groups=1, width=64, last_stride=2, fc=0, ibn="a"),
    "resnet50_ibn_b": dict(block="bottleneck", layers=(3, 4, 6, 3), groups=1, width=64, last_stride=2, fc=0, ibn="b"),
}


def resnet_family_blocks(name: str):
    """[(prefix, stride, cin, width, cout, downsample)] of every residual block of `name`, in forward order
    (_make_layer, resnet.py:257-290)."""
    spec = RESNET_FAMILY[name]
    basic = spec["block"] == "basic"
    out, cin = [], 64
    for li, (n, planes) in enumerate(zip(spec["layers"], (64, 128, 256, 512))):
        cout = planes if basic else planes * 4
        width = planes if basic else planes * spec["width"] // 64 * spec["groups"]
        for bi in range(n):
            stride = 1 if bi > 0 or li == 0 else (spec["last_stride"] if li == 3 else 2)
            out.append(("layer%d.%d" % (li + 1, bi), stride, cin, width, cout, bi == 0 and (stride != 1 or cin != cout)))
            cin = cout
    return out


def resnet_family_param_shapes(name: str) -> dict:
    """Parameter / buffer names and shapes of torchreid's `name` state_dict (one of RESNET_FAMILY), minus the unused
    classifier.  InstanceNorm2d(affine=True) layers hold only .weight and .bias."""
    spec = RESNET_FAMILY[name]
    shapes = {"conv1.weight": (64, 3, 7, 7)}

    def bn(prefix, c):
        for k in ("weight", "bias", "running_mean", "running_var"):
            shapes[prefix + "." + k] = (c,)

    def inorm(prefix, c):
        shapes[prefix + ".weight"] = (c,)
        shapes[prefix + ".bias"] = (c,)

    (inorm if spec["ibn"] == "b" else bn)("bn1", 64)
    last = {"layer%d.%d" % (li + 1, n - 1) for li, n in enumerate(spec["layers"])}
    for p, _, cin, width, cout, down in resnet_family_blocks(name):
        li = int(p[5]) - 1
        if spec["block"] == "basic":
            shapes[p + ".conv1.weight"] = (width, cin, 3, 3)
            bn(p + ".bn1", width)
            shapes[p + ".conv2.weight"] = (cout, width, 3, 3)
            bn(p + ".bn2", cout)
        else:
            shapes[p + ".conv1.weight"] = (width, cin, 1, 1)
            if spec["ibn"] == "a" and li < 3:                  # IBN(planes): IN of planes // 2, BN of the rest
                inorm(p + ".bn1.IN", width // 2)
                bn(p + ".bn1.BN", width - width // 2)
            else:
                bn(p + ".bn1", width)
            shapes[p + ".conv2.weight"] = (width, width // spec["groups"], 3, 3)
            bn(p + ".bn2", width)
            shapes[p + ".conv3.weight"] = (cout, width, 1, 1)
            bn(p + ".bn3", cout)
        if spec["ibn"] == "b" and li < 2 and p in last:
            inorm(p + ".IN", cout)
        if down:
            shapes[p + ".downsample.0.weight"] = (cout, cin, 1, 1)
            bn(p + ".downsample.1", cout)
    if spec["fc"]:
        cin = resnet_family_blocks(name)[-1][4]
        shapes["fc.0.weight"] = (spec["fc"], cin)
        shapes["fc.0.bias"] = (spec["fc"],)
        bn("fc.1", spec["fc"])
    return shapes


def resnet_family_in_layers(name: str) -> list:
    """The InstanceNorm2d scopes of `name`, in forward order: the norm layers without running statistics."""
    shapes = resnet_family_param_shapes(name)
    return [k[:-7] for k, s in shapes.items()
            if k.endswith(".weight") and len(s) == 1 and k[:-7] + ".running_mean" not in shapes]


def synth_resnet_family_state(name: str, seed: int = 2468) -> dict:
    """Seeded float32 state_dict for `name` (one of RESNET_FAMILY), drawn as synth_resnet101_reid_state draws: the last BN
    of every residual branch (bn3, a BasicBlock's bn2) gets a small gamma so that 36 stacked blocks keep activations O(1)
    (fp16-plane range); InstanceNorm gamma ~ U(0.8, 1.2), beta ~ N(0, 0.05)."""
    rng = np.random.default_rng(seed)
    shapes = resnet_family_param_shapes(name)
    in_scopes = set(resnet_family_in_layers(name))
    last_bn = "bn2.weight" if RESNET_FAMILY[name]["block"] == "basic" else "bn3.weight"
    out = {}
    for k, shp in shapes.items():
        if k.rsplit(".", 1)[0] in in_scopes:
            v = rng.uniform(0.8, 1.2, shp) if k.endswith(".weight") else rng.standard_normal(shp) * 0.05
        elif k.endswith("running_var"):
            v = rng.uniform(0.6, 1.4, shp)
        elif k.endswith("running_mean"):
            v = rng.standard_normal(shp) * 0.1
        elif k.endswith(last_bn):
            v = rng.uniform(0.1, 0.3, shp)
        elif k.endswith(".weight") and len(shp) == 1:
            v = rng.uniform(0.7, 1.3, shp)
        elif k.endswith("bias"):
            v = rng.standard_normal(shp) * 0.05
        else:
            fan_in = int(np.prod(shp[1:]))
            residual = k.endswith("conv3.weight") or "downsample" in k or (last_bn == "bn2.weight"
                                                                           and k.endswith("conv2.weight"))
            v = rng.standard_normal(shp) * np.sqrt((1.0 if residual else 2.0) / fan_in)
        out[k] = v.astype(np.float32)
    return out


def synth_effdet_weights(cfg, seed: int = 99) -> dict:
    """Seeded weights of the EfficientDet feature network + class/box nets in the TF variable naming of
    efficientdet_arch.py (kernels HWIO, depthwise [3,3,C,1]); BN statistics non-trivial; predict biases spread
    so that the top-k / NMS path sees a non-degenerate score distribution."""
    from .effdet_config import BIFPN_NODES
    rng = np.random.default_rng(seed)
    W = {}
    F_ = cfg.fpn_num_filters

    def bn(name, c):
        W[name + "/gamma"] = rng.uniform(0.7, 1.3, c).astype(np.float32)
        W[name + "/beta"] = (rng.standard_normal(c) * 0.1).astype(np.float32)
        W[name + "/moving_mean"] = (rng.standard_normal(c) * 0.1).astype(np.float32)
        W[name + "/moving_variance"] = rng.uniform(0.6, 1.4, c).astype(np.float32)

    def conv(name, cin, cout):
        W[name + "/kernel"] = (rng.standard_normal((1, 1, cin, cout)) * np.sqrt(1.0 / cin)).astype(np.float32)
        W[name + "/bias"] = (rng.standard_normal(cout) * 0.05).astype(np.float32)

    def sep(name, c, cout, gain=1.6, bias_std=0.05):
        W[name + "/depthwise_kernel"] = (rng.standard_normal((3, 3, c, 1)) * np.sqrt(1.0 / 9)).astype(np.float32)
        W[name + "/pointwise_kernel"] = (rng.standard_normal((1, 1, c, cout)) * np.sqrt(gain / c)).astype(np.float32)
        W[name + "/bias"] = (rng.standard_normal(cout) * bias_std).astype(np.float32)

    node_gain_sum = 0.55     # un-normalised "sum" nodes add 2-3 maps: smaller pointwise gain keeps 8 cells O(1)
    c5 = cfg.backbone_channels[2]
    if c5 != F_:
        conv("resample_p6/conv2d", c5, F_)
        bn("resample_p6/bn", F_)
    chans = list(cfg.backbone_channels) + [F_, F_]
    for rep in range(cfg.fpn_cell_repeats):
        cur = list(chans) if rep == 0 else [F_] * 5
        for i, (lvl, offsets) in enumerate(BIFPN_NODES):
            pre = "fpn_cells/cell_%d/fnode%d" % (rep, i)
            for idx, o in enumerate(offsets):
                if cur[o] != F_:
                    nm = "%s/resample_%d_%d_%d" % (pre, idx, o, len(cur))
                    conv(nm + "/conv2d", cur[o], F_)
                    bn(nm + "/bn", F_)
                if cfg.fpn_weight_method == "fastattn":
                    W["%s/WSM%s" % (pre, "" if idx == 0 else "_%d" % idx)] = np.float32(rng.uniform(0.5, 1.5))
            op = "%s/op_after_combine%d" % (pre, len(cur))
            sep(op + "/conv", F_, F_, gain=3.0 if cfg.fpn_weight_method == "fastattn" else node_gain_sum)
            bn(op + "/bn", F_)
            cur.append(F_)
    na = cfg.num_scales * len(cfg.aspect_ratios)
    for kind, nout in (("class", cfg.num_classes * na), ("box", 4 * na)):
        for i in range(cfg.box_class_repeats):
            sep("%s_net/%s-%d" % (kind, kind, i), F_, F_, gain=3.0)
            for level in range(cfg.min_level, cfg.max_level + 1):
                bn("%s_net/%s-%d-bn-%d" % (kind, kind, i, level), F_)
        sep("%s_net/%s-predict" % (kind, kind), F_, nout, gain=6.0 if kind == "class" else 0.05,
            bias_std=0.5 if kind == "class" else 0.02)
    if "class_net/class-predict/bias" in W:
        W["class_net/class-predict/bias"] -= np.float32(3.0)     # mostly-negative logits, like a trained detector
    return W



def synth_efficientnet_weights(name: str, seed: int = 77) -> dict:
    """Seeded EfficientNet backbone weights in the keras variable naming of the reference graph
    (efficientnet_model.py:162-392, 504-704); gains chosen so that activations stay O(1) through all blocks."""
    from .effdet_config import efficientnet_blocks
    rng = np.random.default_rng(seed)
    stem_c, blocks = efficientnet_blocks(name)
    W = {}

    def bn(pre, c, g_lo=0.8, g_hi=1.2):
        W[pre + "/gamma"] = rng.uniform(g_lo, g_hi, c).astype(np.float32)
        W[pre + "/beta"] = (rng.standard_normal(c) * 0.1).astype(np.float32)
        W[pre + "/moving_mean"] = (rng.standard_normal(c) * 0.1).astype(np.float32)
        W[pre + "/moving_variance"] = rng.uniform(0.6, 1.4, c).astype(np.float32)

    def conv(pre, k, cin, cout, gain, bias=None):
        W[pre + "/kernel"] = (rng.standard_normal((k, k, cin, cout)) * np.sqrt(gain / (k * k * cin))).astype(np.float32)
        if bias is not None:
            W[pre + "/bias"] = (rng.standard_normal(cout) * 0.1 + bias).astype(np.float32)

    conv(name + "/stem/conv2d", 3, 3, stem_c, 1.0)
    bn(name + "/stem/tpu_batch_normalization", stem_c)
    for i, b in enumerate(blocks):
        pre = "%s/blocks_%d" % (name, i)
        mid = b.cin * b.expand
        proj = "conv2d"
        if b.expand != 1:
            conv(pre + "/conv2d", 1, b.cin, mid, 2.5)
            bn(pre + "/tpu_batch_normalization", mid)
            proj = "conv2d_1"
        W[pre + "/depthwise_conv2d/depthwise_kernel"] = (
            rng.standard_normal((b.kernel, b.kernel, mid, 1)) * np.sqrt(2.5 / (b.kernel ** 2))).astype(np.float32)
        bn(pre + "/tpu_batch_normalization_1", mid)
        nr = max(1, int(b.cin * b.se))
        conv(pre + "/se/conv2d", 1, mid, nr, 1.0, bias=0.0)
        conv(pre + "/se/conv2d_1", 1, nr, mid, 1.0, bias=0.5)
        conv(pre + "/" + proj, 1, mid, b.cout, 2.0)
        bn(pre + "/tpu_batch_normalization_2", b.cout, 0.45, 0.75)
    return W
