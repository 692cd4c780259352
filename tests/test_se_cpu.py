"""SE-ResNet detector (`use_se`, `--version 6`) on the host: the weight manifest and the importer's refusal of incomplete
checkpoints, the synthetic weights of a seed, the oracle's squeeze-excite against an independent float64 restatement of
nn.py:506-519, the spread of the synthetic network's gates, and the config / ABI plumbing."""
import numpy as np
import pytest
import torch

from object_detection_tracking_b200.config import make_config
from object_detection_tracking_b200.synth import frcnn_weight_shapes, synth_frame, synth_weights
import se_oracle
from oracle import frcnn

V6 = dict(use_se=True, use_frcnn_class_agnostic=True, use_dilations=False, version=6)
SE_SUFFIXES = ("/fc1/W", "/fc1/b", "/fc2/W", "/fc2/b")


def np_se_block(l, sc, W, p):
    """numpy float64 restatement of nn.py:506-521 + 586-587 on NCHW l (conv3 after its norm) and the shortcut sc:
    GlobalAvgPooling, dense fc1 + relu, dense fc2 + sigmoid (dense: x @ W + b, W [in, out]), gate, + shortcut, relu."""
    w = lambda k: W[p + k].astype(np.float64)
    s = l.mean(axis=(2, 3))
    s = np.maximum(s @ w("/fc1/W") + w("/fc1/b"), 0.0)
    s = 1.0 / (1.0 + np.exp(-(s @ w("/fc2/W") + w("/fc2/b"))))
    return np.maximum(l * s[:, :, None, None] + sc, 0.0), s


@pytest.mark.parametrize("use_gn", [False, True])
def test_manifest_lists_the_se_variables(use_gn):
    cfg = make_config(resnet_num_block=(2, 1, 3, 1), use_gn=use_gn, **V6)
    sh = frcnn_weight_shapes(cfg)
    w = synth_weights(cfg, 11)
    assert sorted(sh) == sorted(w)
    for k, v in w.items():
        assert tuple(v.shape) == tuple(sh[k]), k
    for g, (feat, count) in enumerate(zip((64, 128, 256, 512), cfg.resnet_num_block)):
        c, nr = 4 * feat, feat // 4
        for i in range(count):
            p = "group%d/block%d" % (g, i)
            assert sh[p + "/fc1/W"] == (c, nr) and sh[p + "/fc1/b"] == (nr,)
            assert sh[p + "/fc2/W"] == (nr, c) and sh[p + "/fc2/b"] == (c,)
    assert sum(1 for k in sh if "/fc1/" in k or "/fc2/" in k) == 4 * sum(cfg.resnet_num_block)
    assert not any("/fc1/" in k for k in frcnn_weight_shapes(make_config(resnet_num_block=(2, 1, 3, 1))))


@pytest.mark.parametrize("missing", ["group0/block0/fc1/W", "group2/block1/fc2/b", "group3/block0/fc2/W"])
def test_check_weights_refuses_a_v6_set_without_one_se_array(missing):
    from object_detection_tracking_b200.backend import check_weights
    cfg = make_config(resnet_num_block=(1, 1, 2, 1), **V6)
    w = synth_weights(cfg, 5)
    check_weights(cfg, w)                                                 # the full set is accepted
    del w[missing]
    with pytest.raises(ValueError) as e:
        check_weights(cfg, w)
    assert missing in str(e.value) and "1 missing" in str(e.value)


def test_check_weights_refuses_a_transposed_se_array():
    from object_detection_tracking_b200.backend import check_weights
    cfg = make_config(resnet_num_block=(1, 1, 2, 1), **V6)
    w = synth_weights(cfg, 5)
    w["group1/block0/fc1/W"] = np.ascontiguousarray(w["group1/block0/fc1/W"].T)
    with pytest.raises(ValueError) as e:
        check_weights(cfg, w)
    assert "group1/block0/fc1/W" in str(e.value) and "mis-shaped" in str(e.value)


def test_se_arrays_are_ignored_without_use_se():
    """A v6 checkpoint loaded into a plain ResNet graph: the SE arrays are names the graph has no variable for."""
    from object_detection_tracking_b200.backend import check_weights
    v6 = make_config(resnet_num_block=(1, 1, 2, 1), **V6)
    plain = make_config(resnet_num_block=(1, 1, 2, 1), use_frcnn_class_agnostic=True, use_dilations=False)
    got = check_weights(plain, synth_weights(v6, 5))
    assert not any("/fc1/" in k or "/fc2/" in k for k in got)
    assert sorted(got) == sorted(frcnn_weight_shapes(plain))


def test_se_weights_leave_every_other_array_of_a_seed_unchanged():
    over = dict(resnet_num_block=(3, 4, 23, 3), use_frcnn_class_agnostic=True, use_dilations=False)
    plain = synth_weights(make_config(**over), 1234)
    se = synth_weights(make_config(use_se=True, **over), 1234)
    extra = sorted(set(se) - set(plain))
    assert set(plain) <= set(se) and len(extra) == 4 * 33
    assert all(k.endswith(SE_SUFFIXES) for k in extra)
    for k in plain:
        assert plain[k].tobytes() == se[k].tobytes(), k


def test_config_and_abi_carry_use_se():
    from object_detection_tracking_b200 import _lib
    assert make_config().use_se is False
    assert _lib.make_config(make_config(), 1, 192, 256).use_se == 0
    assert _lib.make_config(make_config(**V6), 1, 192, 256).use_se == 1
    assert make_config(version=6).use_se is False                         # the drivers map --version to flags


@pytest.mark.parametrize("g,i,stride", [(0, 1, 1), (1, 0, 2), (2, 0, 2)])
def test_oracle_se_bottleneck_matches_fp64_restatement(g, i, stride):
    """se_oracle.bottleneck (exact()) against nn.py:506-521 restated in numpy on the same conv3 / shortcut tensors.  The
    blocks gate 256, 512 and 1024 channels through 16, 32 and 64 hidden units: fc1 and fc2 are not square, so a
    transposed weight cannot pass."""
    cfg = make_config(resnet_num_block=(2, 1, 1, 1), **V6)
    Wt = synth_weights(cfg, 21)
    p = "group%d/block%d" % (g, i)
    cin = (64, 256, 512, 1024)[g] if i == 0 else 256 << g
    rng = np.random.default_rng(g)
    x = np.abs(rng.standard_normal((2, cin, 12, 10)))
    with frcnn.exact():
        xt = torch.from_numpy(x)
        got = se_oracle.bottleneck(xt, Wt, p, stride, 1, False, True).numpy()
        plain = se_oracle.bottleneck(xt, Wt, p, stride, 1, False, False).numpy()
        np.testing.assert_array_equal(plain, frcnn.bottleneck(xt, Wt, p, 64 << g, stride, 1).numpy())
        # the same block's conv3 output and shortcut, taken apart: relu(l + sc) is frcnn.bottleneck
        conv = frcnn._conv
        l = torch.relu(frcnn._bn(conv(xt, Wt[p + "/conv1/W"]), Wt, p + "/conv1"))
        if stride == 2:
            l = torch.relu(frcnn._bn(conv(l, Wt[p + "/conv2/W"], stride=2, pad=(1, 0, 1, 0)), Wt, p + "/conv2"))
        else:
            l = torch.relu(frcnn._bn(conv(l, Wt[p + "/conv2/W"], pad=(1, 1, 1, 1)), Wt, p + "/conv2"))
        l = frcnn._bn(conv(l, Wt[p + "/conv3/W"]), Wt, p + "/conv3").numpy()
        sc = xt
        if (p + "/convshortcut/W") in Wt:
            sc = sc[:, :, :-1, :-1] if stride == 2 else sc
            sc = frcnn._bn(conv(sc, Wt[p + "/convshortcut/W"], stride=stride), Wt, p + "/convshortcut")
        sc = sc.numpy()
    np.testing.assert_allclose(np.maximum(l + sc, 0.0), plain, rtol=0, atol=1e-12)
    ref, gate = np_se_block(l, sc, Wt, p)
    assert np.abs(got - ref).max() < 1e-12 * max(1.0, np.abs(ref).max())
    assert np.abs(got - plain).max() > 1e-2                               # the gate is observable
    assert gate.shape == (2, Wt[p + "/fc2/b"].shape[0]) and Wt[p + "/fc1/W"].shape[0] != Wt[p + "/fc1/W"].shape[1]


def test_oracle_gates_are_per_image():
    cfg = make_config(resnet_num_block=(1, 1, 1, 1), **V6)
    Wt = synth_weights(cfg, 21)
    x = np.random.default_rng(0).standard_normal((3, 256, 9, 11)).astype(np.float32)
    l = torch.from_numpy(x)
    _, g3 = se_oracle.squeeze_excite(l, Wt, "group0/block0")
    _, g1 = se_oracle.squeeze_excite(l[1:2], Wt, "group0/block0")
    np.testing.assert_allclose(g3[1:2].numpy(), g1.numpy(), rtol=0, atol=1e-6)   # BLAS may block a batch differently
    assert (g3[0] - g3[2]).abs().max() > 1e-3


def test_synthetic_v6_gates_neither_saturated_nor_constant():
    cfg = make_config(resnet_num_block=(3, 4, 23, 3), max_size=256, short_edge_size=192, **V6)
    Wt = synth_weights(cfg, 1234)
    x = frcnn.preprocess(synth_frame(192, 256, 3).astype(np.float32))
    gates = []
    se_oracle.backbone(x, Wt, cfg, gates)
    assert len(gates) == 33
    g = torch.cat([v.flatten() for _, v in gates]).numpy()
    lo, hi, std = float(g.min()), float(g.max()), float(g.std())
    print("synthetic v6 gates: min %.3f max %.3f std %.3f" % (lo, hi, std))
    assert lo > 0.02 and hi < 0.995 and std > 0.08
    mid = np.mean((g > 0.2) & (g < 0.8))
    assert mid > 0.85, mid
    # gates follow the image, not only the bias
    other = []
    se_oracle.backbone(frcnn.preprocess(synth_frame(192, 256, 9).astype(np.float32)), Wt, cfg, other)
    assert max(float((a - b).abs().max()) for (_, a), (_, b) in zip(gates, other)) > 0.05


def test_se_oracle_is_frcnn_without_use_se():
    cfg = make_config(resnet_num_block=(1, 1, 1, 1), max_size=128, short_edge_size=96)
    Wt = synth_weights(cfg, 2)
    frame = synth_frame(96, 128, 1).astype(np.float32)
    before = (frcnn.backbone, frcnn.fpn, frcnn.fastrcnn_head)
    a = frcnn.forward(cfg, Wt, frame, stages=False)
    b = se_oracle.forward(cfg, Wt, frame, stages=False)
    for k in ("final_boxes", "final_probs", "final_labels", "fpn_box_feat"):
        np.testing.assert_array_equal(a[k], b[k])
    scfg = make_config(resnet_num_block=(1, 1, 1, 1), max_size=128, short_edge_size=96, **V6)
    sw = synth_weights(scfg, 2)
    with_se = se_oracle.forward(scfg, sw, frame)
    assert (frcnn.backbone, frcnn.fpn, frcnn.fastrcnn_head) == before
    no_se = frcnn.forward(scfg, sw, frame)                                # the SE names present do not select the branch
    assert np.abs(with_se["c2345"][3] - no_se["c2345"][3]).max() > 1e-2
