"""GroupNorm model family on the host: the oracle's group_norm, the conv box head's ReLU-then-GN order, the weight manifest
of the four (use_gn, use_conv_frcnn_head) combinations, the importer's refusal of a BatchNorm checkpoint for a GroupNorm
graph, and the synthetic weights of existing seeds."""
import hashlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from object_detection_tracking_b200.config import make_config
from object_detection_tracking_b200.synth import frcnn_weight_shapes, synth_weights
import gn_oracle
from oracle import frcnn


def moments_gn(x, gamma, beta, groups=32, eps=1e-5):
    """numpy restatement of group_norm (nn.py:81-108): tf.nn.moments over (C/G, H, W) -- the mean, then the mean of the
    squared deviations from it -- and tf.nn.batch_normalization (inv = rsqrt(var + eps) * gamma)."""
    n, c, h, w = x.shape
    xg = x.reshape(n, groups, c // groups, h, w)
    mean = xg.mean(axis=(2, 3, 4), keepdims=True)
    var = np.square(xg - mean).mean(axis=(2, 3, 4), keepdims=True)
    g = gamma.reshape(1, groups, c // groups, 1, 1)
    b = beta.reshape(1, groups, c // groups, 1, 1)
    inv = g / np.sqrt(var + eps)
    return (xg * inv + (b - mean * inv)).reshape(n, c, h, w)


@pytest.mark.parametrize("c,h,w", [(64, 5, 7), (256, 7, 7), (2048, 3, 4)])
def test_oracle_gn_matches_moments_and_torch(c, h, w):
    rng = np.random.default_rng(c)
    x = (rng.standard_normal((3, c, h, w)) * 2.0 + 0.5).astype(np.float64)
    gamma = rng.uniform(0.5, 1.5, c)
    beta = rng.standard_normal(c) * 0.1
    W = {"s/gamma": gamma.astype(np.float32), "s/beta": beta.astype(np.float32)}
    with frcnn.exact():
        got = gn_oracle.gn(torch.from_numpy(x), W, "s").numpy()
    ref = moments_gn(x, W["s/gamma"].astype(np.float64), W["s/beta"].astype(np.float64))
    assert np.abs(got - ref).max() < 1e-10
    tg = F.group_norm(torch.from_numpy(x), 32, torch.from_numpy(W["s/gamma"]).double(),
                      torch.from_numpy(W["s/beta"]).double(), eps=1e-5).numpy()
    assert np.abs(got - tg).max() < 1e-10
    # float32 oracle: statistics per image (an image's result does not depend on the others)
    got32 = gn_oracle.gn(torch.from_numpy(x.astype(np.float32)), W, "s").numpy()
    one32 = gn_oracle.gn(torch.from_numpy(x[1:2].astype(np.float32)), W, "s").numpy()
    assert np.abs(got32 - ref).max() < 1e-4
    np.testing.assert_array_equal(got32[1:2], one32)


def test_conv_head_is_relu_then_gn():
    """conv_frcnn_head (models.py:1110-1125): conv + bias, ReLU, THEN GroupNorm per ROI, no ReLU after it."""
    cfg = make_config(resnet_num_block=(1, 1, 1, 1), use_gn=True, use_conv_frcnn_head=True, conv_frcnn_head_dim=64,
                      fpn_frcnn_fc_head_dim=64)
    Wt = synth_weights(cfg, 3)
    rng = np.random.default_rng(0)
    feat = rng.standard_normal((2, 256, 7, 7)).astype(np.float32)
    with frcnn.exact():
        got = gn_oracle.conv_frcnn_head(feat, Wt, use_gn=True).numpy()
    x = feat.astype(np.float64)
    x_other = x
    for k in range(4):
        wk = torch.from_numpy(Wt["fastrcnn/conv%d/W" % k].astype(np.float64)).permute(3, 2, 0, 1)
        bk = torch.from_numpy(Wt["fastrcnn/conv%d/b" % k].astype(np.float64))
        g, b = Wt["fastrcnn/gn%d/gamma" % k].astype(np.float64), Wt["fastrcnn/gn%d/beta" % k].astype(np.float64)
        conv = F.conv2d(torch.from_numpy(x), wk, bk, padding=1).numpy()
        x = moments_gn(np.maximum(conv, 0.0), g, b)                       # reference: ReLU, then GN
        conv_o = F.conv2d(torch.from_numpy(x_other), wk, bk, padding=1).numpy()
        x_other = np.maximum(moments_gn(conv_o, g, b), 0.0)               # Tensorpack's GN head: GN, then ReLU
    fw, fb = Wt["fastrcnn/fc/W"].astype(np.float64), Wt["fastrcnn/fc/b"].astype(np.float64)
    ref = np.maximum(x.reshape(2, -1) @ fw + fb, 0.0)
    other = np.maximum(x_other.reshape(2, -1) @ fw + fb, 0.0)
    assert np.abs(got - ref).max() < 1e-9 * max(1.0, np.abs(ref).max())
    assert np.abs(got - other).max() > 1e-2                               # the order is observable
    assert (x < 0).any()                                                  # GN output keeps negatives: no ReLU after


@pytest.mark.parametrize("use_gn", [False, True])
@pytest.mark.parametrize("conv_head", [False, True])
def test_weight_manifest_four_combinations(use_gn, conv_head):
    cfg = make_config(resnet_num_block=(2, 1, 2, 1), num_class=81, use_gn=use_gn, use_conv_frcnn_head=conv_head)
    sh = frcnn_weight_shapes(cfg)
    w = synth_weights(cfg, 11)
    assert sorted(sh) == sorted(w)
    for k, v in w.items():
        assert tuple(v.shape) == tuple(sh[k]), k
    has = lambda n: n in sh
    assert has("conv0/gn/gamma") == use_gn and has("conv0/bn/mean/EMA") == (not use_gn)
    assert has("group1/block0/convshortcut/gn/beta") == use_gn
    assert has("group3/block0/conv3/gn/gamma") == use_gn
    assert not any("/bn/" in k for k in sh) if use_gn else not any("/gn/" in k for k in sh)
    for i in range(2, 6):
        assert has("fpn/gn_c%d/gamma" % i) == use_gn and has("fpn/gn_p%d/beta" % i) == use_gn
    assert has("fastrcnn/fc6/W") == (not conv_head) and has("fastrcnn/fc7/b") == (not conv_head)
    if conv_head:
        assert sh["fastrcnn/conv0/W"] == (3, 3, 256, 256) and sh["fastrcnn/conv3/b"] == (256,)
        assert sh["fastrcnn/fc/W"] == (256 * 49, 1024)
        assert has("fastrcnn/gn3/gamma") == use_gn and not has("fastrcnn/gn4/gamma")
    assert sh["fastrcnn/outputs/class/W"] == (1024, 81)


def test_check_weights_rejects_bn_checkpoint_for_gn_config():
    from object_detection_tracking_b200.backend import check_weights
    bn_cfg = make_config(resnet_num_block=(3, 4, 6, 3), num_class=81, use_dilations=False, version=2)
    gn_cfg = make_config(resnet_num_block=(3, 4, 6, 3), num_class=81, use_dilations=False, version=2, use_gn=True,
                         use_conv_frcnn_head=True)
    bn_ckpt = synth_weights(bn_cfg, 5)
    with pytest.raises(ValueError) as e:
        check_weights(gn_cfg, bn_ckpt)
    msg = str(e.value)
    assert "conv0/gn/beta" in msg and "conv0/gn/gamma" in msg and "missing" in msg
    check_weights(gn_cfg, synth_weights(gn_cfg, 5))                       # the GN checkpoint itself is accepted


# sha256 over sorted (name, bytes) of synth_weights as the BatchNorm-only code drew them
PARENT_DIGESTS = [
    (dict(), 1234, "db0c69c79a4e1bee6bcf9411f417b405f14ce05b5b101afb806f9754533878e8"),
    (dict(resnet_num_block=(3, 4, 6, 3), num_class=81, use_dilations=False, version=2), 4321,
     "ecbe73552e7762fa41f857a0e8abb2c91d0b4bb917a398acfd15ccbfef7b26e9"),
    (dict(resnet_num_block=(1, 1, 2, 1), add_mask=True, num_class=81), 7,
     "80bd9b5e6b65d753dc15f5446903f4b215381e9ef3d5b2f78fe25a07cf2e14ce"),
]


def _digest(w):
    h = hashlib.sha256()
    for k in sorted(w):
        h.update(k.encode())
        h.update(w[k].tobytes())
    return h.hexdigest()


@pytest.mark.parametrize("over,seed,digest", PARENT_DIGESTS)
def test_existing_seed_weights_unchanged(over, seed, digest):
    assert _digest(synth_weights(make_config(**over), seed)) == digest


def test_gn_family_shares_the_other_weights_of_a_seed():
    over = dict(resnet_num_block=(3, 4, 6, 3), num_class=81, use_dilations=False, version=2)
    bn = synth_weights(make_config(**over), 4321)
    gn = synth_weights(make_config(use_gn=True, use_conv_frcnn_head=True, **over), 4321)
    shared = [k for k in bn if k in gn]
    assert len(shared) > 50 and "group2/block5/conv2/W" in shared and "rpn/class/W" in shared
    for k in shared:
        np.testing.assert_array_equal(bn[k], gn[k])


def test_gn_oracle_is_frcnn_for_the_batchnorm_graph():
    """With both flags off the GroupNorm oracle is oracle.frcnn itself, and graph() puts frcnn's functions back."""
    from object_detection_tracking_b200.synth import synth_frame
    cfg = make_config(resnet_num_block=(1, 1, 1, 1), max_size=128, short_edge_size=96)
    Wt = synth_weights(cfg, 2)
    frame = synth_frame(96, 128, 1).astype(np.float32)
    before = (frcnn.backbone, frcnn.fpn, frcnn.fastrcnn_head)
    a = frcnn.forward(cfg, Wt, frame, stages=False)
    b = gn_oracle.forward(cfg, Wt, frame, stages=False)
    assert (frcnn.backbone, frcnn.fpn, frcnn.fastrcnn_head) == before
    for k in ("final_boxes", "final_probs", "final_labels", "fpn_box_feat"):
        np.testing.assert_array_equal(a[k], b[k])
    gcfg = make_config(resnet_num_block=(1, 1, 1, 1), max_size=128, short_edge_size=96, use_gn=True,
                       use_conv_frcnn_head=True)
    gw = synth_weights(gcfg, 2)
    o = gn_oracle.forward(gcfg, gw, frame)
    assert o["hidden"].shape[1] == gcfg.fpn_frcnn_fc_head_dim and len(o["final_boxes"]) > 0
    with pytest.raises(KeyError):                                          # frcnn alone has no GroupNorm branch
        frcnn.forward(gcfg, gw, frame, stages=False)
