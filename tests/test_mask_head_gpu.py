"""The mask head (models.py:934-961, 1173-1199) one layer at a time, through b2_op_mask_head (the engine's builder,
add_mask_head, every layer in its own buffer), in split and fp16 precision:

  ROIAlign 14    bit for bit: its raw planes are the planes of oracle.frcnn.multilevel_roi_align(.., 14, ..)'s float32
  fcn0..fcn3     within conv_oracle.bound of the float64 conv of the engine's own held input; ReLU zeros exact
  deconv         the same against the transposed conv written from the TF layout, after the un-shuffle; its taps are
                 scaled by distinct powers of two, so a transposed tap or swapped out / in is an error of order 1
  class conv     within the bound, at num_class 2, 6 and 81; the padded columns exactly 0
  mask select    within mask_oracle.sigmoid_bound of the float64 sigmoid of the engine's logit; alone (logits_in) on
                 logits that identify their (row, channel), so every pixel is traced to its source

and the engine's phase 7 (set_stage + run_phases(128)) bit-identical to the op on the same inputs."""
import numpy as np
import pytest

import conv_oracle as co
import mask_oracle as mo
import selection_inputs as si

pytestmark = pytest.mark.gpu

F32 = np.float32
PRECISIONS = ("split", "fp16")
STRIDES = (4, 8, 16, 32)


def weights(rng, ncls, C=256):
    """maskrcnn/* weights; the deconv's four taps scaled by 1, 2, 4, 8."""
    W = {}
    for k in range(4):
        W["maskrcnn/fcn%d/W" % k] = (rng.standard_normal((3, 3, C, C)) * np.sqrt(2.0 / (9 * C))).astype(F32)
        W["maskrcnn/fcn%d/b" % k] = (rng.standard_normal(C) * 0.2).astype(F32)
    wd = rng.standard_normal((2, 2, C, C)) * np.sqrt(2.0 / C)
    W["maskrcnn/deconv/W"] = (wd * (2.0 ** np.arange(4)).reshape(2, 2, 1, 1) / 4).astype(F32)
    W["maskrcnn/deconv/b"] = (rng.standard_normal(C) * 0.2).astype(F32)
    W["maskrcnn/conv/W"] = (rng.standard_normal((1, 1, C, ncls - 1)) / np.sqrt(C)).astype(F32)
    W["maskrcnn/conv/b"] = (rng.standard_normal(ncls - 1) * 0.2).astype(F32)
    return W


def levels(B, crops, pad=(0, 0), salt=0, C=256):
    """p2..p5 [B, h + pad, w + pad, C]: selection_inputs' fp16-exact values over the crop, large distinct values (1000 +
    k / 8, never a feature value) in the padding.  Returns (levels, per-image oracle levels [C, h, w])."""
    fs, per = [], [[] for _ in range(B)]
    for l, (h, w) in enumerate(crops):
        ph, pw = h + pad[0], w + pad[1]
        s = si.feature_stage(B, (ph, pw), (h, w), C, salt + l)
        tail = np.ones(s.shape, bool)
        tail[:, :h, :w] = False
        s[tail] = F32(1000) + (np.arange(tail.sum()) % 4096).astype(F32) / F32(8)
        fs.append(s)
        for b in range(B):
            per[b].append(np.ascontiguousarray(s[b, :h, :w].transpose(2, 0, 1)))
    return fs, per


def run(feats, crops, boxes, count, labels, ncls, W, precision, outputs=("roi", "fcn", "up", "logits")):
    from object_detection_tracking_b200.engine import op_mask_head
    return op_mask_head(boxes, count, labels, ncls, feats=feats, level_hw=crops, strides=STRIDES, weights=W,
                        split=precision == "split", outputs=outputs)


def held(out, name, precision):
    """The value the engine's planes of output `name` hold, float64."""
    return co.join(out[name + "_hi"].view(np.float16), out[name + "_lo"].view(np.float16) if precision == "split" else None)


def assert_planes_bits(out, name, exp, precision, what):
    """The raw planes of out[name] are those of the float32 values exp."""
    hi, lo = co.split_planes(exp)
    assert np.array_equal(out[name + "_hi"], hi.view(np.uint16)), what + ": hi plane"
    if precision == "split":
        assert np.array_equal(out[name + "_lo"], lo.view(np.uint16)), what + ": lo plane"


# ---- ROIAlign 14 -----------------------------------------------------------------------------------------------------
def check_roi(feats, per, crops, boxes, count, precision):
    B, R = boxes.shape[:2]
    labels = np.ones((B, R), np.int32)
    out = run(feats, crops, boxes, count, labels, 2, weights(np.random.default_rng(0), 2), precision, outputs=("roi",))
    roi = out["roi"].reshape(B, R, 14, 14, 256)
    for b in range(B):
        n = int(count[b])
        exp = np.zeros((R, 14, 14, 256), F32)
        if n:
            exp[:n] = mo.roi14(per[b], boxes[b, :n], STRIDES)
        view = {k: out[k].reshape(B, R, 14, 14, 256)[b] for k in ("roi_hi", "roi_lo") if out[k] is not None}
        view.update(roi=roi[b])
        assert_planes_bits(view, "roi", exp, precision, "roi b%d" % b)
        assert np.all(roi[b, n:] == 0) and not np.any(np.signbit(roi[b, n:]))
    return out


def level_boundary_boxes():
    from test_selection_kernels_gpu import level_boundary_boxes as lbb
    return lbb()


@pytest.mark.parametrize("precision", PRECISIONS)
def test_roialign14_level_boundaries(precision):
    """Boxes with sqrt(area) on both sides of every level boundary, on a 512 x 768 frame; B = 3 with counts (R, 0, a
    partial count)."""
    crops = [(128, 192), (64, 96), (32, 48), (16, 24)]
    sides = level_boundary_boxes()
    R = len(sides)
    boxes = np.zeros((3, R, 4), F32)
    for i, (w, h) in enumerate(sides):
        x, y = 7 + (i * 37) % max(1, 768 - w - 14), 3 + (i * 23) % max(1, 512 - min(h, 506) - 6)
        boxes[:, i] = (x, y, x + w, y + h)
    boxes[2] = boxes[2, ::-1]
    feats, per = levels(3, crops, salt=1)
    count = np.array([R, 0, R // 3], np.int32)
    check_roi(feats, per, crops, boxes, count, precision)
    from oracle import frcnn
    assert set(frcnn.fpn_map_rois_to_levels(boxes[0]).tolist()) == {2, 3, 4, 5}


def edge_boxes(H, W, dim, rng, need_hit):
    """Boxes partly and wholly outside the frame, zero-width / zero-height / 1-px boxes, p2 right edges whose last crop-28
    sample lands exactly on dim - 1, and random ones."""
    bx = [[-30, -20, 40, 50], [W - 40, H - 30, W + 60, H + 20], [-80, 10, -10, 60], [W + 10, 5, W + 90, 70],
          [10, -90, 70, -5], [20, 30, 20, 80], [20, 30, 90, 30], [50, 60, 51, 61], [0, 0, 1, 1], [W - 1, H - 1, W, H],
          [0, 0, W, H], [-W, -H, 2 * W, 2 * H]]
    hits = 0
    for c1 in np.arange(dim - 2, dim + 2, 0.125, dtype=F32):
        c0 = F32(c1 - 28)
        if mo.samples(c0, c1, dim, 28)[-1] == F32(dim - 1):
            bx.append([c0 * 4, 40, c1 * 4, 80])
            hits += 1
    assert hits >= need_hit
    for _ in range(30):
        x0, y0 = rng.uniform(-40, W), rng.uniform(-40, H)
        bx.append([x0, y0, x0 + rng.uniform(0, 160), y0 + rng.uniform(0, 160)])
    return (np.round(np.asarray(bx, np.float64) * 8) / 8).astype(F32)


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("frame", ["192x256", "200x300", "32x256", "256x32"])
def test_roialign14_edges_and_odd_geometry(frame, precision):
    """Edge and degenerate boxes on: 192 x 256; 200 x 300 with every level's pitch past its crop, the padding holding
    large distinct values; 32 x 256 and 256 x 32, where p5 is 1 pixel high / wide."""
    from object_detection_tracking_b200.config import backbone_geometry, make_config
    H, W = map(int, frame.split("x"))
    crops = backbone_geometry(H, W, make_config(max_size=max(H, W), short_edge_size=min(H, W)))["p"][:4]
    rng = np.random.default_rng(H + W)
    bx = edge_boxes(H, W, crops[0][1], rng, frame == "192x256")
    R = len(bx)
    boxes = np.stack([bx, bx[rng.permutation(R)], bx[::-1]])
    feats, per = levels(3, crops, pad=(3, 5) if frame == "200x300" else (0, 0), salt=2)
    out = check_roi(feats, per, crops, boxes, np.array([R, 0, R - 7], np.int32), precision)
    assert np.abs(out["roi"]).max() < 8                      # no padding value reached an output
    if frame in ("32x256", "256x32"):
        assert 1 in crops[3]


# ---- the conv layers and the sigmoid select ----------------------------------------------------------------------------
def chain_inputs(rng, B=2, R=3, ncls=81):
    """A 192 x 256 frame's levels, R boxes per image (one wholly outside the frame: an all-zero ROI), counts (R, R - 1),
    labels including 1 and num_class - 1."""
    crops = [(48, 64), (24, 32), (12, 16), (6, 8)]
    feats, per = levels(B, crops, salt=5)
    boxes = np.zeros((B, R, 4), F32)
    for b in range(B):
        xy = rng.uniform(0, 150, (R, 2))
        boxes[b] = np.round(np.concatenate([xy, xy + rng.uniform(20, 100, (R, 2))], 1) * 4) / 4
    boxes[0, 1] = (300, 10, 340, 60)                         # outside the frame: ROIAlign gives exactly 0
    count = np.array([R, R - 1] + [R] * (B - 2), np.int32)
    labels = rng.integers(1, ncls, (B, R)).astype(np.int32)
    labels[0, 0], labels[1, 0] = 1, ncls - 1
    return feats, per, crops, boxes, count, labels


def check_bound(got, ref, e, what):
    err = np.abs(np.asarray(got, np.float64) - ref)
    i = np.unravel_index(np.argmax(err - e), err.shape)
    assert np.all(err <= e), "%s: |err| %.3g > bound %.3g at %s" % (what, err[i], e[i], i)


def check_chain(out, W, ncls, precision, count, labels, layers=True):
    split = precision == "split"
    B, R = labels.shape
    M = B * R
    if layers:
        x = held(out, "roi", precision).reshape(M, 14, 14, 256)
        for k in range(4):
            r = mo.fcn(x, W["maskrcnn/fcn%d/W" % k], W["maskrcnn/fcn%d/b" % k], split)
            got = out["fcn"][k]
            e = mo.bound(r, precision)[..., :256]
            check_bound(got, r["ref"][..., :256], e, "fcn%d" % k)
            assert np.all(got >= 0) and np.all(got[r["pre"][..., :256] < -e] == 0), "fcn%d: ReLU zeros" % k
            if k == 0:                                        # all-zero ROIs: exactly relu(bias) through the planes
                zero = ~np.any(x.reshape(M, -1), axis=1)
                assert zero.sum() >= 2
                rb = co.represent(np.maximum(W["maskrcnn/fcn0/b"], 0), split).astype(F32)
                assert np.all(got[zero] == rb)
            x = held({"h_hi": out["fcn_hi"][k], "h_lo": None if out["fcn_lo"] is None else out["fcn_lo"][k]}, "h",
                     precision)
        ref, S = mo.deconv28(x, W["maskrcnn/deconv/W"], W["maskrcnn/deconv/b"], split)
        b = np.broadcast_to(np.abs(W["maskrcnn/deconv/b"].astype(np.float64)), ref.shape)
        e = co.bound(256, S, b, 0.0, ref, precision)
        check_bound(mo.unshuffle(out["up"]), ref, e, "deconv")
        assert np.abs(ref).max() > 1000 * e.max()
    up = held(out, "up", precision).reshape(M, 14, 14, 1024)
    r = mo.class_conv(up, W["maskrcnn/conv/W"], W["maskrcnn/conv/b"], split)
    ld = (ncls - 1 + 15) // 16 * 16
    lg = out["logits"]
    assert lg.shape == (M * 784, ld) and r["Cp"] == ld
    check_bound(lg[:, :ncls - 1], r["ref"][0, 0, :, :ncls - 1], mo.bound(r, precision, out="f32")[0, 0, :, :ncls - 1],
                "class conv")
    assert np.all(lg[:, ncls - 1:] == 0)
    check_masks(out["masks"], lg, count, labels)


def check_masks(masks, logits, count, labels):
    B, R = labels.shape
    z = mo.mask_rows(logits, B * R).reshape(B, R, 28, 28, -1)
    for b in range(B):
        n = int(count[b])
        s = mo.sigmoid64(z[b, np.arange(n), :, :, labels[b, :n] - 1])
        check_bound(masks[b, :n], s, mo.sigmoid_bound(s), "masks b%d" % b)
        assert np.all(masks[b, n:] == 0) and not np.any(np.signbit(masks[b, n:]))


@pytest.mark.parametrize("precision", PRECISIONS)
def test_layers_against_float64(precision):
    """fcn0..3, the deconv, the class conv (num_class 81: Cout 80, ld 80) and the select, each from the engine's own
    held previous layer."""
    rng = np.random.default_rng(11)
    feats, per, crops, boxes, count, labels = chain_inputs(rng)
    W = weights(rng, 81)
    out = run(feats, crops, boxes, count, labels, 81, W, precision)
    check_chain(out, W, 81, precision, count, labels)


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("ncls", [2, 6])
def test_class_conv_narrow(ncls, precision):
    """num_class 2 (Cout 1, ld 16) and 6 (Cout 5, ld 16): the class conv and the select."""
    rng = np.random.default_rng(12 + ncls)
    feats, per, crops, boxes, count, labels = chain_inputs(rng, ncls=ncls)
    W = weights(rng, ncls)
    out = run(feats, crops, boxes, count, labels, ncls, W, precision, outputs=("up", "logits"))
    check_chain(out, W, ncls, precision, count, labels, layers=False)


@pytest.mark.parametrize("precision", PRECISIONS)
def test_mask_select_alone_traces_every_pixel(precision):
    """logits_in: image 0's boxes hold a permutation of a grid over [-4, 4] spaced far beyond the sigmoid's error, one
    value per (pixel row, channel), so each output pixel's logit is recovered and must be row (roi * 196 + (Y >> 1) * 14 +
    (X >> 1)) * 4 + (Y & 1) * 2 + (X & 1), channel label - 1; image 1's span [-100, 40] (saturation, expf overflow).
    Rows at or past the count hold NaN logits and must give exactly 0."""
    from object_detection_tracking_b200.engine import op_mask_head
    rng = np.random.default_rng(21)
    B, R, ncls = 2, 5, 6
    ld, n = 16, 784 * 16
    step = 8.0 / n
    logits = np.empty((B * R * 784, ld), F32)
    for m in range(R):
        logits[m * 784:(m + 1) * 784] = (-4 + step * rng.permutation(n)).reshape(784, ld)
    logits[R * 784:] = rng.uniform(-100, 40, (R * 784, ld))
    count = np.array([R, 3], np.int32)
    labels = np.array([[1, 5, 2, 3, 4], [5, 1, 4, 1, 1]], np.int32)
    logits[(R + 3) * 784:] = np.nan
    masks = op_mask_head(np.zeros((B, R, 4), F32), count, labels, ncls, logits=logits, split=precision == "split")["masks"]
    check_masks(masks, logits, count, labels)
    # trace image 0's pixels back to their grid value
    v = masks[0].astype(np.float64)
    k = np.round((np.log(v / (1 - v)) + 4) / step).astype(np.int64)
    for m in range(R):
        grid = np.round((logits[m * 784:(m + 1) * 784].astype(np.float64) + 4) / step).astype(np.int64)
        where = np.empty(n, np.int64)
        where[grid.ravel()] = np.arange(n)
        src = where[k[m]]
        Y, X = np.meshgrid(np.arange(28), np.arange(28), indexing="ij")
        np.testing.assert_array_equal(src // ld, ((Y >> 1) * 14 + (X >> 1)) * 4 + (Y & 1) * 2 + (X & 1))
        assert np.all(src % ld == labels[0, m] - 1)
    assert masks[1, :3].min() == 0 and masks[1, :3].max() == 1       # saturated both ways


@pytest.mark.parametrize("precision", PRECISIONS)
def test_images_are_independent(precision):
    """Each image run alone through the op equals its slice of the batch, bit for bit, at every layer."""
    rng = np.random.default_rng(31)
    feats, per, crops, boxes, count, labels = chain_inputs(rng, B=3, R=2, ncls=6)
    count[2] = 0
    W = weights(rng, 6)
    full = run(feats, crops, boxes, count, labels, 6, W, precision)
    M = 2
    for b in range(3):
        one = run([f[b:b + 1] for f in feats], crops, boxes[b:b + 1], count[b:b + 1], labels[b:b + 1], 6, W, precision)
        for k in ("roi", "up"):
            assert si.same_bits(one[k], full[k][b * M:(b + 1) * M]), (b, k)
        assert si.same_bits(one["fcn"], full["fcn"][:, b * M:(b + 1) * M]), (b, "fcn")
        assert si.same_bits(one["logits"], full["logits"][b * M * 784:(b + 1) * M * 784]), (b, "logits")
        assert si.same_bits(one["masks"], full["masks"][b:b + 1]), (b, "masks")


# ---- the engine's phase 7 is the op -------------------------------------------------------------------------------------
ENGINES = {
    "b2": (dict(), 2, False),
    "b2_multi": (dict(), 2, True),
    "partial": (dict(num_class=81, use_dilations=False, version=2, use_partial_classes=True,
                     partial_classes=["person", "car", "bus", "truck", "bicycle"]), 1, False),
}


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("name", list(ENGINES))
def test_engine_phase7_is_the_op(name, precision):
    """A Detector with add_mask: p2..p5 and final_boxes / labels / count set, run_phases(128); mask_logits and final_masks
    are bit-identical to op_mask_head on the same inputs."""
    from object_detection_tracking_b200.config import backbone_geometry, make_config
    from object_detection_tracking_b200.engine import Detector, op_mask_head
    from object_detection_tracking_b200.synth import synth_weights
    over, B, multi = ENGINES[name]
    H, W = 192, 256
    cfg = make_config(resnet_num_block=(1, 1, 1, 1), max_size=W, short_edge_size=H, add_mask=True, **over)
    Wt = synth_weights(cfg, 41)
    det = Detector(cfg, B, H, W, precision=precision, use_cuda_graph=False, multi_semantics=multi)
    try:
        det.load_weights(Wt)
        R, ncls = det.R, int(cfg.num_class)
        nlab = len(cfg.partial_class_ids) if getattr(cfg, "partial_class_ids", ()) else ncls - 1
        crops = backbone_geometry(H, W, det.cfg)["p"][:4]
        feats = []
        for l in range(4):
            shape = det.stage_shape("p%d" % (l + 2))[0]
            s = si.feature_stage(B, shape[1:3], crops[l], shape[3], 50 + l) / F32(4)
            det.set_stage("p%d" % (l + 2), s)
            feats.append(s)
        rng = np.random.default_rng(42)
        xy = rng.uniform(-20, 220, (B, R, 2))
        boxes = (np.round(np.concatenate([xy, xy + rng.uniform(1, 120, (B, R, 2))], -1) * 4) / 4).astype(F32)
        count = np.array([R, 37][:B], np.int32)
        labels = rng.integers(1, nlab + 1, (B, R)).astype(np.int32)
        labels[:, 0], labels[:, 1] = 1, nlab
        det.set_stage("final_boxes", boxes[..., None])
        det.set_stage("final_labels", labels.reshape(B, R, 1, 1))
        det.set_stage("final_count", count.reshape(B, 1, 1, 1))
        det.run_phases(128)
        eng_logits = det.get_stage("mask_logits")
        eng_masks = det.get_stage("final_masks")
        mw = {k: v for k, v in Wt.items() if k.startswith("maskrcnn/")}
        op = op_mask_head(boxes, count, labels, ncls, feats=feats, level_hw=crops, strides=STRIDES, weights=mw,
                          split=precision == "split", outputs=("logits",))
        ld = (ncls - 1 + 15) // 16 * 16
        assert eng_logits.shape == (B * R, 784, ld, 1)
        assert si.same_bits(eng_logits.reshape(-1, ld), op["logits"]), "mask_logits"
        assert si.same_bits(eng_masks, op["masks"]), "final_masks"
        assert np.any(eng_masks[0, :count[0]] > 0.5) and np.any(eng_masks[0, :count[0]] < 0.5)
    finally:
        det.close()
