"""Attention box head (`use_att_frcnn_head`) on the CPU: the oracle's bin sum against a literal float64 restatement of
models.py:1064-1089 (the 3x3 SAME conv and its length-1 softmax), finite and non-finite inputs; the weight manifest and
the importer's refusals; the synthetic weights of existing seeds; the ABI struct; and that the synthetic branch is not
degenerate on a real forward pass."""
import ctypes

import numpy as np
import pytest

from object_detection_tracking_b200.config import make_config
from object_detection_tracking_b200.synth import frcnn_weight_shapes, synth_frame, synth_weights
import att_oracle
from oracle import frcnn
from test_relation_cpu import SEED_DIGESTS, _digest

ATT = dict(use_att_frcnn_head=True)
NAMES = ("fastrcnn/attention/W", "fastrcnn/attention/b", "fastrcnn/att_trans/W", "fastrcnn/att_trans/b")
SMALL = dict(resnet_num_block=(1, 1, 2, 2), max_size=256, short_edge_size=192)


def np_attended(roi_nchw, w, b):
    """models.py:1064-1081 in float64 numpy: NHWC transpose, conv2d(1, 3x3, SAME, bias) with tf.nn.softmax over the last
    (length-1) axis, then reduce_sum(feature * attention) over the 49 cells."""
    x = np.transpose(roi_nchw.astype(np.float64), (0, 2, 3, 1))              # [K, 7, 7, C]
    K, H, W_, C = x.shape
    xp = np.pad(x, ((0, 0), (1, 1), (1, 1), (0, 0)))                          # SAME for a 3x3 stride-1 kernel
    logit = np.zeros((K, H, W_, 1))
    with np.errstate(invalid="ignore", over="ignore"):
        for dy in range(3):
            for dx in range(3):
                logit[..., 0] += np.einsum("khwc,c->khw", xp[:, dy:dy + H, dx:dx + W_, :], w[dy, dx, :, 0].astype(np.float64))
        logit += float(b[0])
        e = np.exp(logit - logit.max(axis=-1, keepdims=True))
        att = e / e.sum(axis=-1, keepdims=True)                              # softmax over the channel axis of length 1
        return (x.reshape(K, 49, C) * att.reshape(K, 49, 1)).sum(axis=1)


def _roi(rng, K, C=256):
    return (np.maximum(rng.standard_normal((K, C, 7, 7)), 0) * rng.uniform(0.1, 3.0, (K, 1, 1, 1))).astype(np.float32)


def _att_weights(seed):
    w = synth_weights(make_config(resnet_num_block=(1, 1, 1, 1), **ATT), seed)
    return w["fastrcnn/attention/W"], w["fastrcnn/attention/b"]


@pytest.mark.parametrize("K", [1, 7, 64])
def test_bin_sum_is_the_literal_head_on_finite_inputs(K):
    rng = np.random.default_rng(K)
    roi = _roi(rng, K)
    w, b = _att_weights(K)
    ref = np_attended(roi, w, b)
    assert np.isfinite(ref).all()
    with frcnn.exact():
        got = att_oracle.attended(roi).numpy()
    np.testing.assert_allclose(got, ref, rtol=1e-12, atol=1e-12)
    # the attention weights do not matter: other weights (larger, negative bias) give the same sum
    ref2 = np_attended(roi, -7.0 * w, -np.abs(b) - 30.0)
    np.testing.assert_allclose(ref2, ref, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("bad", [np.inf, -np.inf, np.nan])
@pytest.mark.parametrize("where", [(0, 0, 0), (37, 3, 6)])
def test_a_non_finite_feature_makes_its_roi_row_nan(bad, where):
    """One non-finite value in an ROI's 7x7x256 block: that ROI's whole row is NaN, in the literal head and in the oracle;
    every other row is unchanged."""
    rng = np.random.default_rng(5)
    roi = _roi(rng, 5)
    w, b = _att_weights(3)
    clean = np_attended(roi, w, b)
    roi[2, where[0], where[1], where[2]] = bad
    ref = np_attended(roi, w, b)
    with frcnn.exact():
        got = att_oracle.attended(roi).numpy()
    for r in (ref, got):
        assert np.isnan(r[2]).all()
        keep = [0, 1, 3, 4]
        np.testing.assert_allclose(r[keep], clean[keep], rtol=1e-12, atol=1e-12)


HEADS = {
    "2fc": dict(),
    "conv_head": dict(use_conv_frcnn_head=True),
    "gn_conv_head": dict(use_gn=True, use_conv_frcnn_head=True),
    "relation": dict(add_relation_nn=True),
    "coco_partial": dict(num_class=81, use_partial_classes=True),
}


@pytest.mark.parametrize("head", sorted(HEADS))
def test_manifest_lists_the_attention_variables(head):
    kw = HEADS[head]
    cfg = make_config(**dict(kw, **ATT))
    sh = frcnn_weight_shapes(cfg)
    base = frcnn_weight_shapes(make_config(**kw))
    extra = {k: v for k, v in sh.items() if k not in base}
    dim = cfg.fpn_frcnn_fc_head_dim
    assert extra == {"fastrcnn/attention/W": (3, 3, 256, 1), "fastrcnn/attention/b": (1,),
                     "fastrcnn/att_trans/W": (256, dim), "fastrcnn/att_trans/b": (dim,)}
    w = synth_weights(cfg, 7)
    assert set(w) == set(sh)
    for k, v in w.items():
        assert tuple(v.shape) == tuple(sh[k]), k


def test_no_attention_variables_without_the_flag_or_with_the_class_agnostic_head():
    for cfg in (make_config(), make_config(use_frcnn_class_agnostic=True, **ATT),
                make_config(use_frcnn_class_agnostic=True, add_relation_nn=True, **ATT)):
        assert not [k for k in frcnn_weight_shapes(cfg) if k in NAMES]
        assert not [k for k in synth_weights(cfg, 3) if k in NAMES]
    assert frcnn_weight_shapes(make_config(use_frcnn_class_agnostic=True, **ATT)) == \
        frcnn_weight_shapes(make_config(use_frcnn_class_agnostic=True))


@pytest.mark.parametrize("missing", NAMES)
def test_check_weights_refuses_an_attention_set_without_one_array(missing):
    from object_detection_tracking_b200.backend import check_weights
    cfg = make_config(**ATT)
    w = synth_weights(cfg, 2)
    del w[missing]
    with pytest.raises(ValueError) as e:
        check_weights(cfg, w)
    assert "1 missing" in str(e.value) and missing in str(e.value)
    got = check_weights(make_config(), w)                                    # ignored without the flag
    assert len(got) == len(frcnn_weight_shapes(make_config())) and not set(got) & set(NAMES)


@pytest.mark.parametrize("name", sorted(SEED_DIGESTS))
def test_existing_seeds_are_unchanged(name):
    kw, digest = SEED_DIGESTS[name]
    assert _digest(synth_weights(make_config(**kw), 1234)) == digest
    # with the attention head every other array is the seed's own
    w = synth_weights(make_config(**dict(kw, **ATT)), 1234)
    assert _digest({k: v for k, v in w.items() if k not in NAMES}) == digest


def test_config_and_abi_carry_use_att_frcnn_head():
    from object_detection_tracking_b200 import _lib
    from test_abi import _header_struct_words
    assert ctypes.sizeof(_lib.B2ConfigExt3) == 4 * _header_struct_words("b2_config_ext3")
    assert make_config().use_att_frcnn_head is False
    assert _lib.make_config_ext3(make_config()).use_att_frcnn_head == 0
    assert _lib.make_config_ext3(make_config(**ATT)).use_att_frcnn_head == 1
    names = [s[0] for s in _lib.SYMBOLS]
    assert "b2_create_ex3" in names and "b2_op_att_pool" in names


def test_synthetic_attention_branch_is_not_degenerate():
    """On the ROI features and hidden rows of a real (small) forward pass: between a fifth and four fifths of the
    att_trans units are active, and the branch moves hidden by between a fifth and all of its norm."""
    for kw in (dict(), dict(use_gn=True, use_conv_frcnn_head=True), dict(add_relation_nn=True)):
        cfg = make_config(**dict(SMALL, **dict(kw, **ATT)))
        W = synth_weights(cfg, 99)
        frame = synth_frame(192, 256, seed=3).astype(np.float32)
        o = att_oracle.forward(cfg, W, frame, stages=True)
        assert len(o["proposal_boxes"]) > 50 and len(o["final_boxes"]) > 0
        att, total = att_oracle.LAST["att_trans"], att_oracle.LAST["att_sum"]
        hidden = total - att
        active = float((att > 0).mean())
        assert 0.2 < active < 0.8, (kw, active)
        ratio = np.linalg.norm(att) / np.linalg.norm(hidden)
        assert 0.2 < ratio < 1.0, (kw, ratio)


def test_att_oracle_is_the_enclosing_head_without_the_flag_or_class_agnostic():
    frame = synth_frame(192, 256, seed=4).astype(np.float32)
    for kw in (dict(SMALL), dict(SMALL, use_frcnn_class_agnostic=True, **ATT)):
        cfg = make_config(**kw)
        W = synth_weights(cfg, 99)
        a = frcnn.forward(cfg, W, frame, stages=False)
        b = att_oracle.forward(cfg, W, frame, stages=False)
        for k in ("final_boxes", "final_labels", "final_probs"):
            np.testing.assert_array_equal(a[k], b[k])
    # the flag changes the logits; the attention conv's weights do not
    cfg = make_config(**dict(SMALL, **ATT))
    W = synth_weights(cfg, 99)
    c = att_oracle.forward(cfg, W, frame, stages=True)
    d = frcnn.forward(cfg, W, frame, stages=True)
    np.testing.assert_array_equal(c["proposal_boxes"], d["proposal_boxes"])
    assert np.abs(c["cls_logits"] - d["cls_logits"]).max() > 1e-2
    W2 = dict(W, **{"fastrcnn/attention/W": W["fastrcnn/attention/W"] * -3.0, "fastrcnn/attention/b": np.ones(1, np.float32)})
    e = att_oracle.forward(cfg, W2, frame, stages=True)
    np.testing.assert_array_equal(c["cls_logits"], e["cls_logits"])
    m = att_oracle.forward_multi(cfg, W, [frame, frame[::-1].copy()], stages=True)
    assert m["final_valid_indices"].min() > 0
