"""ResNeXt detector (`use_resnext`) on the host: the oracle's grouped conv against an independent float64 numpy loop over
the groups, TF's SAME pads, the oracle with the flag off, the weight manifest and the importer's refusals, the synthetic
weights of existing seeds, and the config / ABI plumbing."""
import hashlib

import numpy as np
import pytest
import torch

from object_detection_tracking_b200.config import make_config
from object_detection_tracking_b200.synth import frcnn_weight_shapes, synth_frame, synth_weights
import resnext_oracle
from oracle import frcnn

RX = dict(use_resnext=True)


def np_group_conv(x, w, groups, stride, dil, pad):
    """float64 numpy grouped conv on NCHW x with the HWIO kernel w [R, S, C / groups, Cout]: one loop over the groups and
    one over the taps, each tap a strided window of the zero-padded input times that group's filter slice."""
    x = x.astype(np.float64)
    w = w.astype(np.float64)
    n, c, h, wd = x.shape
    R, S, cg, cout = w.shape
    cgo = cout // groups
    pt, pb, pl, pr = pad
    xp = np.zeros((n, c, h + pt + pb, wd + pl + pr))
    xp[:, :, pt:pt + h, pl:pl + wd] = x
    ho = (h + pt + pb - (R - 1) * dil - 1) // stride + 1
    wo = (wd + pl + pr - (S - 1) * dil - 1) // stride + 1
    out = np.zeros((n, cout, ho, wo))
    for g in range(groups):
        xg = xp[:, g * cg:(g + 1) * cg]
        for r in range(R):
            for s in range(S):
                win = xg[:, :, r * dil:r * dil + (ho - 1) * stride + 1:stride, s * dil:s * dil + (wo - 1) * stride + 1:stride]
                out[:, g * cgo:(g + 1) * cgo] += np.einsum("nchw,co->nohw", win, w[r, s, :, g * cgo:(g + 1) * cgo])
    return out


@pytest.mark.parametrize("cg", [4, 32])
@pytest.mark.parametrize("h,w", [(12, 10), (11, 13)])
@pytest.mark.parametrize("stride,dil", [(1, 1), (2, 1), (1, 2), (2, 2)])
def test_oracle_group_conv_matches_numpy_loop(cg, h, w, stride, dil):
    rng = np.random.default_rng(cg * 100 + h * 10 + stride + 3 * dil)
    c = 32 * cg
    x = rng.standard_normal((2, c, h, w))
    k = rng.standard_normal((3, 3, cg, c)) / np.sqrt(9 * cg)
    pad = resnext_oracle.same_pads(h, 3, stride, dil) + resnext_oracle.same_pads(w, 3, stride, dil)
    with frcnn.exact():
        got = resnext_oracle.group_conv(torch.from_numpy(x), k, 32, stride=stride, dilation=dil, pad=pad).numpy()
    ref = np_group_conv(x, k, 32, stride, dil, pad)
    assert got.shape == ref.shape == (2, c, -(-h // stride), -(-w // stride))
    assert np.abs(got - ref).max() < 1e-12 * np.abs(ref).max()
    # a dense conv of the same kernel shape would mix groups: the grouping is observable
    dense = np_group_conv(x[:, :cg], k[:, :, :, :c], 1, stride, dil, pad)
    assert np.abs(dense[:, cg:2 * cg] - ref[:, cg:2 * cg]).max() > 1e-3


@pytest.mark.parametrize("n,stride,dil,pads", [
    (184, 1, 1, (1, 1)), (46, 1, 2, (2, 2)),                 # stride 1: symmetric
    (184, 2, 1, (0, 1)), (46, 2, 2, (1, 2)),                 # stride 2 on the even sizes of the backbone: odd pad after
    (45, 2, 1, (1, 1)), (45, 2, 2, (2, 2)),                  # odd sizes
])
def test_same_pads_follow_tf(n, stride, dil, pads):
    assert resnext_oracle.same_pads(n, 3, stride, dil) == pads
    keff = 2 * dil + 1
    out = -(-n // stride)
    assert (n + sum(pads) - keff) // stride + 1 == out
    if stride == 2 and n % 2 == 0:
        # the ResNet bottleneck pads [1, 0] and runs VALID (nn.py:487-492): another window, same output size
        assert pads != (1, 0) and (n + 1 - keff) // 2 + 1 == out - (dil - 1)


def test_resnext_block_differs_from_the_bottleneck_padding():
    """The ResNeXt stride-2 conv2 with the bottleneck's [1, 0] pad gives other numbers: the pad is observable."""
    rng = np.random.default_rng(5)
    x = torch.from_numpy(rng.standard_normal((1, 128, 12, 16)))
    k = rng.standard_normal((3, 3, 4, 128)) / 6.0
    with frcnn.exact():
        same = resnext_oracle.group_conv(x, k, 32, stride=2, pad=(0, 1, 0, 1))
        tfpad = resnext_oracle.group_conv(x, k, 32, stride=2, pad=(1, 0, 1, 0))
    assert same.shape == tfpad.shape and (same - tfpad).abs().max() > 0.1


def test_resnext_oracle_is_frcnn_without_the_flag():
    cfg = make_config(resnet_num_block=(1, 1, 1, 1), max_size=128, short_edge_size=96)
    Wt = synth_weights(cfg, 2)
    frame = synth_frame(96, 128, 1).astype(np.float32)
    before = (frcnn.backbone, frcnn.fpn, frcnn.fastrcnn_head)
    a = frcnn.forward(cfg, Wt, frame, stages=False)
    b = resnext_oracle.forward(cfg, Wt, frame, stages=False)
    for k in ("final_boxes", "final_probs", "final_labels", "fpn_box_feat"):
        np.testing.assert_array_equal(a[k], b[k])
    rcfg = make_config(resnet_num_block=(1, 1, 1, 1), max_size=128, short_edge_size=96, **RX)
    rx = resnext_oracle.forward(rcfg, synth_weights(rcfg, 2), frame)
    assert (frcnn.backbone, frcnn.fpn, frcnn.fastrcnn_head) == before
    assert [c.shape[-3] for c in rx["c2345"]] == [256, 512, 1024, 2048] and len(rx["final_boxes"]) > 0


@pytest.mark.parametrize("extra", [dict(), dict(use_gn=True), dict(use_se=True, use_frcnn_class_agnostic=True)])
def test_manifest_lists_the_resnext_shapes(extra):
    cfg = make_config(resnet_num_block=(2, 1, 3, 1), **RX, **extra)
    sh = frcnn_weight_shapes(cfg)
    w = synth_weights(cfg, 11)
    assert sorted(sh) == sorted(w)
    for k, v in w.items():
        assert tuple(v.shape) == tuple(sh[k]), k
    norm = ("gn/gamma",) if extra.get("use_gn") else ("bn/gamma", "bn/mean/EMA")
    cin = 64
    for g, (feat, count) in enumerate(zip((64, 128, 256, 512), cfg.resnet_num_block)):
        for i in range(count):
            p = "group%d/block%d" % (g, i)
            assert sh[p + "/conv1/W"] == (1, 1, cin, 2 * feat)
            assert sh[p + "/conv2/W"] == (3, 3, 2 * feat // 32, 2 * feat)       # Cg = 4, 8, 16, 32
            assert sh[p + "/conv3/W"] == (1, 1, 2 * feat, 4 * feat)
            for n in norm:
                assert sh["%s/conv2/%s" % (p, n)] == (2 * feat,)
            cin = 4 * feat
    # the ResNeXt block has no squeeze-excite branch, with or without use_se
    assert not any("/fc1/" in k or "/fc2/" in k for k in sh)


def test_check_weights_refuses_the_other_backbone():
    from object_detection_tracking_b200.backend import check_weights
    base = dict(resnet_num_block=(1, 1, 2, 1))
    rcfg, pcfg = make_config(**base, **RX), make_config(**base)
    check_weights(rcfg, synth_weights(rcfg, 5))
    check_weights(pcfg, synth_weights(pcfg, 5))
    for cfg, other in ((rcfg, pcfg), (pcfg, rcfg)):
        with pytest.raises(ValueError) as e:
            check_weights(cfg, synth_weights(other, 5))
        assert "mis-shaped" in str(e.value) and "group0/block0/conv2/W" in str(e.value)


# sha256 (first 16 hex digits) over the sorted names and bytes of synth_weights(cfg, 1234), as before use_resnext existed
SEED_DIGESTS = {
    "default": (dict(), "db0c69c79a4e1bee"),
    "gn_convhead": (dict(use_gn=True, use_conv_frcnn_head=True), "2934f7bc85fbfc2f"),
    "se": (dict(use_se=True, use_frcnn_class_agnostic=True, use_dilations=False), "35169c6700bc40d4"),
    "mask": (dict(add_mask=True), "95eb188a019875a2"),
    "r50": (dict(resnet_num_block=(3, 4, 6, 3), num_class=81), "d46a6e37cf6d8a28"),
}


@pytest.mark.parametrize("name", sorted(SEED_DIGESTS))
def test_existing_seeds_are_unchanged(name):
    kw, digest = SEED_DIGESTS[name]
    w = synth_weights(make_config(**kw), 1234)
    h = hashlib.sha256()
    for k in sorted(w):
        h.update(k.encode())
        h.update(w[k].tobytes())
    assert h.hexdigest()[:16] == digest


def test_config_and_abi_carry_use_resnext():
    from object_detection_tracking_b200 import _lib
    assert make_config().use_resnext is False
    assert _lib.make_config(make_config(), 1, 192, 256).use_resnext == 0
    assert _lib.make_config(make_config(**RX), 1, 192, 256).use_resnext == 1
    c = _lib.make_config(make_config(use_se=True, **RX), 1, 192, 256)
    assert c.use_se == 1 and c.use_resnext == 1                            # the engine ignores use_se with use_resnext


def test_synthetic_resnext_activations_stay_bounded():
    """33 ResNeXt blocks on the synthetic weights keep c2..c5 O(1): well inside the fp16 planes' range, and not dead."""
    cfg = make_config(resnet_num_block=(3, 4, 23, 3), max_size=256, short_edge_size=192, **RX)
    Wt = synth_weights(cfg, 1234)
    x = frcnn.preprocess(synth_frame(192, 256, 3).astype(np.float32))
    feats = resnext_oracle.backbone(x, Wt, cfg)
    for f in feats:
        a = float(f.abs().max())
        assert 0.1 < a < 100.0, a
        assert float((f > 0).float().mean()) > 0.05
