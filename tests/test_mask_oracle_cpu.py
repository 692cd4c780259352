"""Pins tests/mask_oracle.py on the CPU: its restatements of the engine's two index conventions (load_layer's kDeconv
tap packing and mask_select's un-shuffle), the crop-28 sample grid and the composed float64 chain against oracle.frcnn;
and b2_op_mask_head's refusals, which come before any device work."""
import numpy as np
import pytest

import mask_oracle as mo

F32 = np.float32


@pytest.fixture
def frcnn64(monkeypatch):
    """oracle.frcnn's torch stack in float64, its outputs kept in float64."""
    from oracle import frcnn
    monkeypatch.setattr(frcnn, "_np", lambda t: t.detach().numpy())
    with frcnn.exact():
        yield frcnn


def identity_fcn(C):
    w = np.zeros((3, 3, C, C), F32)
    w[1, 1] = np.eye(C, dtype=F32)
    return w


def head_weights(rng, C, Co, ncls):
    W = {}
    for k in range(4):
        W["maskrcnn/fcn%d/W" % k] = (rng.standard_normal((3, 3, C, C)) / np.sqrt(9 * C)).astype(F32)
        W["maskrcnn/fcn%d/b" % k] = (rng.standard_normal(C) * 0.1).astype(F32)
    W["maskrcnn/deconv/W"] = (rng.standard_normal((2, 2, Co, C)) / np.sqrt(C)).astype(F32)
    W["maskrcnn/deconv/b"] = (rng.standard_normal(Co) * 0.1).astype(F32)
    W["maskrcnn/conv/W"] = (rng.standard_normal((1, 1, Co, ncls - 1)) / np.sqrt(Co)).astype(F32)
    W["maskrcnn/conv/b"] = (rng.standard_normal(ncls - 1) * 0.1).astype(F32)
    return W


def test_deconv_tap_packing_then_unshuffle_is_the_transposed_conv(frcnn64):
    """A 1x1 conv with kDeconv's packed weights, ReLU, then the un-shuffle, equals the reference's Conv2DTranspose (through
    maskrcnn_head with identity fcn layers and an identity class conv) within 1e-12; a tap-transposed or out / in-swapped
    packing does not."""
    rng = np.random.default_rng(0)
    C = 12
    W = {"maskrcnn/fcn%d/W" % k: identity_fcn(C) for k in range(4)}
    W.update({"maskrcnn/fcn%d/b" % k: np.zeros(C, F32) for k in range(4)})
    W["maskrcnn/deconv/W"] = rng.standard_normal((2, 2, C, C)).astype(F32)
    W["maskrcnn/deconv/b"] = rng.standard_normal(C).astype(F32)
    W["maskrcnn/conv/W"] = np.eye(C, dtype=F32).reshape(1, 1, C, C)
    W["maskrcnn/conv/b"] = np.zeros(C, F32)
    x = np.abs(rng.standard_normal((3, C, 14, 14))).astype(F32)          # >= 0: the identity fcn layers keep it
    ref = frcnn64.maskrcnn_head(x, W, C + 1).transpose(0, 2, 3, 1)       # [M, 28, 28, C]
    xh = x.transpose(0, 2, 3, 1).astype(np.float64)

    def restated(packed):
        up = np.maximum(xh @ packed.astype(np.float64).T + np.tile(W["maskrcnn/deconv/b"], 4), 0.0)
        return mo.unshuffle(up)
    got = restated(mo.pack_deconv(W["maskrcnn/deconv/W"]))
    assert np.abs(got - ref).max() <= 1e-12 * np.abs(ref).max()
    tf28, _ = mo.deconv28(x.transpose(0, 2, 3, 1), W["maskrcnn/deconv/W"], W["maskrcnn/deconv/b"], split=None)
    assert np.abs(tf28 - ref).max() <= 1e-12 * np.abs(ref).max()
    for wrong in (W["maskrcnn/deconv/W"].transpose(1, 0, 2, 3), W["maskrcnn/deconv/W"].transpose(0, 1, 3, 2)):
        assert np.abs(restated(mo.pack_deconv(wrong)) - ref).max() > 0.1


def test_class_conv_on_tap_rows_commutes_with_the_unshuffle():
    """The 1x1 class conv over the (pixel, tap) rows, read back through mask_select's row formula, equals the conv of the
    un-shuffled 28 x 28 map."""
    rng = np.random.default_rng(1)
    M, C, K = 3, 16, 5
    up = rng.standard_normal((M, 14, 14, 4 * C))
    w = rng.standard_normal((C, K))
    b = rng.standard_normal(K)
    rows = up.reshape(-1, C) @ w + b                                     # [M * 784, K]
    got = mo.mask_rows(rows, M)
    exp = mo.unshuffle(up) @ w + b
    assert got.shape == (M, 28, 28, K)
    assert np.abs(got - exp).max() <= 1e-12 * np.abs(exp).max()


def test_crop28_samples_are_crop_and_resize_coordinates(monkeypatch):
    """mask_oracle.samples(.., crop=28) is the sample grid oracle.frcnn.roi_align(.., 14) hands crop_and_resize: a ramp
    image (channel 0 = x, channel 1 = y) crops to exactly those coordinates inside the level and 0 outside."""
    from oracle import frcnn, tf_ops
    crops = []
    real = tf_ops.crop_and_resize

    def capture(img, boxes, crop):
        r = real(img, boxes, crop)
        crops.append(r)
        return r
    monkeypatch.setattr(frcnn.tf_ops, "crop_and_resize", capture)
    H, W = 37, 53
    y, x = np.meshgrid(np.arange(H, dtype=F32), np.arange(W, dtype=F32), indexing="ij")
    feat = np.stack([x, y])
    rng = np.random.default_rng(2)
    boxes = [[-5, -3, 20, 12], [3.25, 4.5, 50.75, 36], [10, 10, 10, 30], [0, 0, 1, 1], [40, 30, 70, 50], [0, 0, W, H]]
    for _ in range(30):
        x0, y0 = rng.uniform(-10, W), rng.uniform(-10, H)
        boxes.append([x0, y0, x0 + rng.uniform(0, 40), y0 + rng.uniform(0, 40)])
    boxes = (np.round(np.asarray(boxes) * 8) / 8).astype(F32)
    frcnn.roi_align(feat, boxes, 14)
    c = crops[-1]
    assert c.shape == (len(boxes), 28, 28, 2)
    for i, (x0, y0, x1, y1) in enumerate(boxes):
        sx, sy = mo.samples(x0, x1, W, 28), mo.samples(y0, y1, H, 28)
        inx, iny = (sx >= 0) & (sx <= W - 1), (sy >= 0) & (sy <= H - 1)
        ex = np.where(iny[:, None] & inx[None, :], sx[None, :], 0)
        ey = np.where(iny[:, None] & inx[None, :], sy[:, None], 0)
        np.testing.assert_array_equal(c[i, ..., 0], ex)
        np.testing.assert_array_equal(c[i, ..., 1], ey)
    assert not np.array_equal(mo.samples(boxes[1, 0], boxes[1, 2], W, 28)[::2], mo.samples(boxes[1, 0], boxes[1, 2], W, 14))


def test_composed_chain_is_final_masks(frcnn64):
    """ROIAlign 14, fcn0..3, the TF-layout deconv, the class conv on tap rows and mask_select's read, composed in float64,
    equal oracle.frcnn.final_masks' logits (within 1e-12) and masks (its float32 sigmoid, within 2^-22)."""
    from object_detection_tracking_b200.config import make_config
    rng = np.random.default_rng(3)
    C, ncls = 16, 6
    cfg = make_config(num_class=ncls, add_mask=True)
    W = head_weights(rng, C, C, ncls)
    feats = [rng.standard_normal((C, h, w)).astype(F32) for h, w in ((24, 32), (12, 16), (6, 8), (3, 4))]
    boxes = np.array([[4, 6, 60, 50], [10, 20, 120, 90], [0, 0, 127, 95], [30, 30, 34, 33]], F32)
    labels = np.array([1, 5, 3, 2])
    masks, logits = frcnn64.final_masks(cfg, W, feats, boxes, labels)
    x = mo.roi14(feats, boxes, cfg.anchor_strides)
    for k in range(4):
        x = mo.fcn64(x, W["maskrcnn/fcn%d/W" % k], W["maskrcnn/fcn%d/b" % k])
    d28, _ = mo.deconv28(x, W["maskrcnn/deconv/W"], W["maskrcnn/deconv/b"], split=None)
    up = d28.reshape(4, 14, 2, 14, 2, C).transpose(0, 1, 3, 2, 4, 5).reshape(4, 14, 14, 4 * C)   # the engine's layout
    np.testing.assert_array_equal(mo.unshuffle(up), d28)
    rows = up.reshape(-1, C) @ W["maskrcnn/conv/W"][0, 0].astype(np.float64) + W["maskrcnn/conv/b"]
    lg = mo.mask_rows(rows, 4)                                           # [4, 28, 28, ncls - 1]
    ref = logits.transpose(0, 2, 3, 1)
    assert np.abs(lg - ref).max() <= 1e-12 * np.abs(ref).max()
    sel = lg[np.arange(4), :, :, labels - 1]
    assert np.abs(mo.sigmoid64(sel) - masks).max() <= 2.0 ** -22


def test_sigmoid_bound_covers_fp32_rounding():
    """The bound is wider than a float32 evaluation of 1 / (1 + exp(-z)) with numpy's exp (within 1 ulp) over the whole
    logit range, including expf's overflow."""
    z = np.concatenate([np.linspace(-120, 40, 20001), [-88.7, -88.8, 0.0, 1e-30]]).astype(F32)
    with np.errstate(over="ignore"):
        v = (F32(1) / (F32(1) + np.exp(-z))).astype(F32)
    s = mo.sigmoid64(z)
    assert np.all(np.abs(v - s) <= mo.sigmoid_bound(s))


# ---- b2_op_mask_head refuses before any device work ------------------------------------------------------------------
def _op_args(B=2, R=3, ncls=6):
    boxes = np.tile(np.array([10, 10, 60, 50], F32), (B, R, 1))
    return boxes, np.full(B, R, np.int32), np.ones((B, R), np.int32), ncls


@pytest.mark.parametrize("case,match", [
    ("label0", "labels\\[0\\]\\[1\\] = 0"), ("label_high", "labels\\[1\\]\\[2\\] = 6"), ("count_neg", "count\\[1\\]"),
    ("count_high", "count\\[0\\]"), ("ncls1", "num_class")])
def test_op_mask_head_refuses_on_the_host(case, match):
    from object_detection_tracking_b200.engine import op_mask_head
    boxes, count, labels, ncls = _op_args()
    if case == "label0":
        labels[0, 1] = 0
    elif case == "label_high":
        labels[1, 2] = ncls
    elif case == "count_neg":
        count[1] = -1
    elif case == "count_high":
        count[0] = 4
    else:
        ncls = 1
    ld = (ncls - 1 + 15) // 16 * 16
    logits = np.zeros((boxes.shape[0] * boxes.shape[1] * 784, ld), F32)
    with pytest.raises(RuntimeError, match=match):
        op_mask_head(boxes, count, labels, ncls, logits=logits)

