"""Mask paste and RLE on the GPU (csrc/mask_rle.cu, object_detection_tracking_b200/masks.py): full-frame masks byte for
byte against the NumPy oracle (tests/mask_rle_oracle.py) and the cv2 golden (tests/golden/mask_paste_cv2.npz), RLE strings
against the oracle's encoder applied to the oracle's masks (the drivers' composition), and the engine's in-place encode of
final_masks."""
import os

import numpy as np
import pytest

import mask_rle_oracle as oracle

pytestmark = pytest.mark.gpu


def seeded_boxes(rng, n, H, W):
    """n boxes whose patches fit the frame, sizes from 1 pixel to most of it."""
    out = []
    while len(out) < n:
        w = float(rng.uniform(0.5, W * rng.choice([0.05, 0.2, 0.6])))
        h = float(rng.uniform(0.5, H * rng.choice([0.05, 0.2, 0.6])))
        x, y = float(rng.uniform(0, W - w)), float(rng.uniform(0, H - h))
        box = np.array([x, y, x + w, y + h], np.float32)
        try:
            x0, y0, x1, y1, bw, bh = oracle.geometry(box)
            np.zeros((H, W), np.uint8)[y0:y1 + 1, x0:x1 + 1] = np.ones((bh, bw), np.uint8)
        except ValueError:
            continue
        out.append(box)
    return np.array(out, np.float32).reshape(-1, 4)


def seeded_masks(rng, n):
    yy, xx = np.mgrid[0:28, 0:28].astype(np.float32)
    out = []
    for i in range(n):
        if i % 3 == 2:
            out.append(np.float32(0.5) + rng.integers(-3, 4, (28, 28)).astype(np.float32) * np.float32(2.0 ** -24))
        else:
            cx, cy, r = rng.uniform(4, 24, 2).tolist() + [rng.uniform(8, 120)]
            blob = 1.0 / (1.0 + np.exp(((xx - cx) ** 2 + (yy - cy) ** 2) / r - 1.0 + rng.normal(0, 0.5, (28, 28))))
            out.append(blob.astype(np.float32))
    return np.array(out, np.float32).reshape(-1, 28, 28)


def check_against_oracle(boxes, masks, H, W, device_masks=False):
    from object_detection_tracking_b200 import masks as gm
    m_in = masks
    if device_masks:
        import torch
        m_in = torch.from_numpy(masks).cuda()
    full = gm.fill_full_masks(boxes, m_in, (H, W))
    rles = gm.encode_masks(boxes, m_in, (H, W))
    assert full.shape == (len(boxes), H, W) and full.dtype == np.uint8 and len(rles) == len(boxes)
    for i in range(len(boxes)):
        ref = oracle.fill_full_mask(boxes[i], masks[i], (H, W))
        np.testing.assert_array_equal(full[i], ref, err_msg="box %d %s" % (i, boxes[i]))
        assert rles[i] == oracle.encode(ref), (i, boxes[i])
    return full, rles


@pytest.mark.parametrize("H,W,n", [(720, 1280, 100), (1080, 1920, 100), (1281, 2989, 20), (2160, 3840, 10)])
def test_seeded_frames_match_oracle(H, W, n):
    rng = np.random.default_rng(H + n)
    boxes, masks = seeded_boxes(rng, n, H, W), seeded_masks(rng, n)
    check_against_oracle(boxes, masks, H, W)


def test_device_masks_match_host_masks():
    rng = np.random.default_rng(9)
    H, W = 480, 640
    boxes, masks = seeded_boxes(rng, 30, H, W), seeded_masks(rng, 30)
    a = check_against_oracle(boxes, masks, H, W, device_masks=False)
    b = check_against_oracle(boxes, masks, H, W, device_masks=True)
    np.testing.assert_array_equal(a[0], b[0])
    assert a[1] == b[1]


def test_edge_boxes():
    H, W = 48, 64
    boxes = np.array([
        [0, 0, 1, 1], [63, 47, 64, 48], [0, 0, 64, 48],              # first pixel, last pixel, the full frame
        [0, 0, 1, 48], [63, 0, 64, 48], [0, 0, 64, 1], [0, 47, 64, 48],   # first / last column and row
        [5, 0, 9, 48], [5, 0, 64, 48], [0, 0, 33, 48],               # full-height patches: columns abut
        [3, 10, 40, 42.3], [10.2, 3.7, 11.9, 40.1], [0, 0, 64, 33],  # a patch 33 rows tall straddles two words
        [70, 10, 70.2, 20], [10, 50, 20, 50.1],                       # size-1 patch broadcast into an empty slice
        [5, 5, 5.2, 5.3], [3, 3, 0.4, 0.2], [-0.9, -0.6, 3, 4],       # clamped and truncated corners
    ], np.float32)
    rng = np.random.default_rng(21)
    masks = seeded_masks(rng, len(boxes))
    masks[2] = 1.0                                                    # all-ones full frame: counts [0, H * W]
    masks[5] = 0.0
    full, rles = check_against_oracle(boxes, masks, H, W)
    assert rles[2]["counts"] == oracle.rle_string([0, H * W]) and full[2].all()
    assert not full[13].any() and not full[14].any() and rles[13]["counts"] == oracle.rle_string([H * W])
    # checkerboard-like patches: the longest strings
    cb = (np.indices((28, 28)).sum(0) % 2).astype(np.float32)
    check_against_oracle(np.array([[0, 0, 28, 28], [0, 0, 64, 48], [1, 0, 29, 48]], np.float32), np.stack([cb] * 3),
                         H, W)


def test_zero_and_one_box():
    from object_detection_tracking_b200 import masks as gm
    assert gm.encode_masks(np.zeros((0, 4), np.float32), np.zeros((0, 28, 28), np.float32), (10, 10)) == []
    assert gm.fill_full_masks(np.zeros((0, 4), np.float32), np.zeros((0, 28, 28), np.float32), (10, 10)).shape == (0, 10,
                                                                                                                      10)
    rng = np.random.default_rng(2)
    box, mask = np.array([2.3, 4.1, 30.7, 19.9], np.float32), seeded_masks(rng, 1)[0]
    np.testing.assert_array_equal(gm.fill_full_mask(box, mask, (40, 50)), oracle.fill_full_mask(box, mask, (40, 50)))
    check_against_oracle(box[None], mask[None], 40, 50)


def test_golden_patches():
    from object_detection_tracking_b200 import masks as gm
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "mask_paste_cv2.npz"))
    masks = z["masks"]
    for i, (w, h) in enumerate(z["sizes"]):
        w, h = int(w), int(h)
        H, W = h + 3, w + 2
        boxes = np.tile(np.array([1, 2, 1 + w, 2 + h], np.float32), (len(masks), 1))
        full = gm.fill_full_masks(boxes, masks, (H, W))
        rles = gm.encode_masks(boxes, masks, (H, W))
        for k in range(len(masks)):
            bits = np.unpackbits(z["bits_%d_%d" % (i, k)], count=w * h).reshape(h, w)
            exp = np.zeros((H, W), np.uint8)
            exp[2:2 + h, 1:1 + w] = bits
            np.testing.assert_array_equal(full[k], exp, err_msg="%dx%d mask %d" % (w, h, k))
            assert rles[k] == oracle.encode(exp)


def test_refusals_raise_before_any_launch():
    from object_detection_tracking_b200 import masks as gm
    m = np.full((1, 28, 28), 0.9, np.float32)
    for box in ([0, 0, 10, 49], [60, 0, 66, 10], [70, 10, 75, 20], [-2, 0, 5, 5], [0, -1.6, 5, 5], [np.nan, 0, 3, 3]):
        with pytest.raises(ValueError):
            gm.fill_full_masks(np.array([box], np.float32), m, (48, 64))
        with pytest.raises(ValueError):
            gm.encode_masks(np.array([box], np.float32), m, (48, 64))
    with pytest.raises(ValueError):
        gm.encode_masks(np.array([[0, 0, 5, 5]], np.float32), np.zeros((1, 14, 14), np.float32), (48, 64))
    with pytest.raises(ValueError):
        gm.encode_masks(np.array([[0, 0, 5, 5]], np.float32), np.zeros((2, 28, 28), np.float32), (48, 64))
    # a good call after the refusals still works
    check_against_oracle(np.array([[0, 0, 5, 5]], np.float32), m, 48, 64)


def _mask_model(is_multi):
    from object_detection_tracking_b200.backend import get_model
    from object_detection_tracking_b200.config import make_config
    from object_detection_tracking_b200.synth import synth_weights
    H, W = 192, 256
    cfg = make_config(resnet_num_block=(1, 1, 2, 1), max_size=W, short_edge_size=H, add_mask=True)
    model = get_model(cfg, gpuid=0, is_multi=is_multi)
    model.set_weights(synth_weights(cfg, 1234))
    return model, H, W


def test_engine_encode_single_image():
    import torch
    from object_detection_tracking_b200 import masks as gm
    from object_detection_tracking_b200.backend import Session
    from object_detection_tracking_b200.synth import synth_frame
    model, H, W = _mask_model(False)
    frame = synth_frame(H, W, 5).astype(np.float32)
    boxes, masks = Session().run([model.final_boxes, model.final_masks], feed_dict=model.get_feed_dict_forward(frame))
    assert len(boxes) > 0
    scale = 0.5                                                   # the source frame was 2x the resized one
    boxes_scaled = boxes / scale
    assert boxes_scaled.dtype == np.float32
    im_shape = (2 * H, 2 * W)
    got = model.encode_masks(boxes_scaled, im_shape)
    assert got == gm.encode_masks(boxes_scaled, masks, im_shape)
    assert got == gm.encode_masks(boxes_scaled, torch.from_numpy(masks).cuda(), im_shape)
    assert got == [oracle.encode(oracle.fill_full_mask(b, m, im_shape)) for b, m in zip(boxes_scaled, masks)]
    assert model.encode_masks(boxes_scaled[:0], im_shape) == []


def test_engine_encode_batch():
    from object_detection_tracking_b200 import masks as gm
    from object_detection_tracking_b200.backend import Session
    from object_detection_tracking_b200.synth import synth_frame
    model, H, W = _mask_model(True)
    frames = [synth_frame(H, W, 5).astype(np.float32), synth_frame(H, W, 11).astype(np.float32)]
    boxes, valid, masks = Session().run([model.final_boxes, model.final_valid_indices, model.final_masks],
                                        feed_dict=model.get_feed_dict_forward_multi(frames))
    im_shape = (2 * H, 2 * W)
    at = 0
    for b in range(2):
        r = int(valid[b])
        bs = boxes[b, :r] / 0.5
        mb = masks[at:at + r]
        at += r
        got = model.encode_masks(bs, im_shape, image=b)
        assert got == gm.encode_masks(bs, mb, im_shape)
        assert got == [oracle.encode(oracle.fill_full_mask(x, m, im_shape)) for x, m in zip(bs, mb)]
