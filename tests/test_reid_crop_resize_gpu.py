"""ReID crops cut and resized on the GPU (b2_op_reid_crop_resize, b2_reid_embed_boxes[_dev]) against the Pillow golden
(tests/golden/reid_crops_pil.npz, tests/golden/make_golden_reid_crops.py): the kernel's crops byte for byte, and the
features of embed_boxes bit for bit against embed() on the golden's Pillow crops, for both models and both precisions."""
import os

import numpy as np
import pytest

import pil_resize_oracle

pytestmark = pytest.mark.gpu

SIZES = ((256, 128), (128, 256))   # (out_h, out_w): osnet_x1_0, resnet101
MODELS = {"osnet_x1_0": (256, 128), "resnet101": (128, 256)}


@pytest.fixture(scope="module")
def golden(golden_dir):
    return pil_resize_oracle.load_golden(os.path.join(golden_dir, "reid_crops_pil.npz"))


def op_crop_resize(frames, boxes, out_h, out_w):
    from object_detection_tracking_b200 import _lib
    frames = np.ascontiguousarray(frames, np.uint8)
    boxes = np.ascontiguousarray(boxes, np.int32)
    out = np.empty((len(boxes), out_h, out_w, 3), np.uint8)
    _lib.check(_lib.load().b2_op_reid_crop_resize(0, _lib.ptr(frames), frames.shape[0], frames.shape[1], frames.shape[2],
                                                  _lib.ptr(boxes), len(boxes), out_h, out_w, _lib.ptr(out)),
               "b2_op_reid_crop_resize")
    return out


def engine(model, batch, precision):
    from object_detection_tracking_b200.reid import ReidEngine
    from object_detection_tracking_b200.synth import synth_osnet_state, synth_resnet101_reid_state
    eng = ReidEngine(batch=batch, precision=precision, model=model)
    eng.load_state(synth_osnet_state(4321) if model == "osnet_x1_0" else synth_resnet101_reid_state(2468))
    return eng


def test_op_matches_pillow_golden(golden):
    for g in range(int(golden["num_groups"])):
        frames, boxes = golden["g%d_frames" % g], golden["g%d_boxes" % g]
        for out_h, out_w in SIZES:
            got = op_crop_resize(frames, boxes, out_h, out_w)
            ref = golden["g%d_crops_%dx%d" % (g, out_h, out_w)]
            for i in range(len(boxes)):
                np.testing.assert_array_equal(got[i], ref[i], err_msg="group %d box %s -> %dx%d" % (g, boxes[i], out_w,
                                                                                                   out_h))


def test_op_matches_oracle_on_noise_frames():
    """White-noise frames (every rounding case the golden's smooth textures may not reach) against the numpy oracle,
    which the CPU tests pin to live Pillow: the whole frame, its edges, 1x1, a vertical-first column and person boxes."""
    rng = np.random.default_rng(31)
    H, W = 540, 960
    frames = rng.integers(0, 256, (2, H, W, 3), dtype=np.uint8)
    boxes = [(0, 0, 0, W, H), (1, W - 1, H - 1, 1, 1), (0, W - 37, 0, 37, H), (1, 0, H - 41, W, 41), (0, 500, 0, 3, H),
             (1, 10, 20, 128, 256), (0, 300, 100, 256, 128)]
    for _ in range(9):
        w = int(rng.integers(8, 240))
        h = min(H, int(w * rng.uniform(1.5, 3.2)))
        boxes.append((int(rng.integers(0, 2)), int(rng.integers(0, W - w + 1)), int(rng.integers(0, H - h + 1)), w, h))
    boxes = np.asarray(boxes, np.int32)
    for out_h, out_w in SIZES:
        got = op_crop_resize(frames, boxes, out_h, out_w)
        for i, b in enumerate(boxes):
            np.testing.assert_array_equal(got[i], pil_resize_oracle.crop_resize(frames[b[0]], b[1:], out_w, out_h),
                                          err_msg="box %s -> %dx%d" % (b, out_w, out_h))


@pytest.mark.parametrize("precision", ["split", "fp16"])
@pytest.mark.parametrize("model", ["osnet_x1_0", "resnet101"])
def test_embed_boxes_bit_identical_to_embed_of_pillow_crops(golden, model, precision):
    out_h, out_w = MODELS[model]
    eng = engine(model, 8, precision)
    for g in range(int(golden["num_groups"])):
        frames, boxes = golden["g%d_frames" % g], golden["g%d_boxes" % g]
        crops = golden["g%d_crops_%dx%d" % (g, out_h, out_w)]
        for i in range(0, len(boxes), 8):
            ref = eng.embed(crops[i:i + 8])
            got = eng.embed_boxes(frames, boxes[i:i + 8])
            assert got.shape == ref.shape and np.isfinite(got).all()
            np.testing.assert_array_equal(got, ref, err_msg="group %d boxes %d.." % (g, i))
    eng.close()


def test_batch_fill_replay_and_device_output(golden):
    import torch
    eng = engine("osnet_x1_0", 8, "split")
    frames, boxes = golden["g0_frames"], golden["g0_boxes"]
    assert frames.shape[0] == 2 and len(set(boxes[:8, 0])) == 2                     # boxes from both frames
    full = eng.embed_boxes(frames, boxes[:8])                                         # n = B
    part = eng.embed_boxes(frames, boxes[:5])                                         # n < B, rows 5..7 zeroed
    np.testing.assert_array_equal(part, full[:5])
    np.testing.assert_array_equal(eng.embed_boxes(frames, boxes[:8]), full)          # graph replay
    single = eng.embed_boxes(frames[int(boxes[3, 0])], np.concatenate([[0], boxes[3, 1:]])[None])   # one [h, w, 3] frame
    np.testing.assert_array_equal(single[0], full[3])
    out = torch.full((5, 512), float("nan"), device="cuda")
    eng.embed_boxes_dev(frames, boxes[:5], out)
    np.testing.assert_array_equal(out.cpu().numpy(), part)
    eng.close()


def test_extract_boxes_chunks_like_the_drivers(golden):
    import torch
    from object_detection_tracking_b200.reid import FeatureExtractor
    from object_detection_tracking_b200.synth import synth_osnet_state
    ext = FeatureExtractor(model_name="osnet_x1_0", batch=3, state_dict=synth_osnet_state(4321))
    frames, boxes = golden["g0_frames"], golden["g0_boxes"]
    sel = boxes[boxes[:, 0] == 0]
    assert len(sel) > 6 and len(sel) % 3                                              # three chunks of 3, the last short
    tlwhs = [(x + 0.75, y + 0.25, w + 0.5, h + 0.99) for _, x, y, w, h in sel]        # int() truncates like the drivers
    feats = ext.extract_boxes(frames[0], tlwhs)
    assert isinstance(feats, torch.Tensor) and tuple(feats.shape) == (len(sel), 512)
    crops = golden["g0_crops_256x128"][boxes[:, 0] == 0]
    ref = np.concatenate([ext.engine.embed(crops[i:i + 3]) for i in range(0, len(crops), 3)])
    np.testing.assert_array_equal(feats.numpy(), ref)
    assert tuple(ext.extract_boxes(frames[0], []).shape) == (0, 512)
    ext.engine.close()


def test_bad_boxes_are_refused_before_any_launch(golden):
    eng = engine("osnet_x1_0", 4, "split")
    frames, boxes = golden["g0_frames"], golden["g0_boxes"][:4].copy()
    good = eng.embed_boxes(frames, boxes)
    conv1 = eng.get_activation("conv1")
    H, W = frames.shape[1:3]
    bad = {"leaves the frame": (0, W - 5, 0, 6, 10), "past the bottom": (0, 0, H - 2, 4, 3), "negative x": (1, -1, 0, 4, 4),
           "zero width": (0, 3, 3, 0, 5), "zero height": (1, 3, 3, 5, 0), "frame index": (2, 0, 0, 4, 4),
           "negative frame": (-1, 0, 0, 4, 4)}
    for b in bad.values():
        t = boxes.copy()
        t[2] = b
        with pytest.raises(RuntimeError, match="b2_reid_embed_boxes"):
            eng.embed_boxes(frames, t)
        with pytest.raises(RuntimeError, match="b2_op_reid_crop_resize"):
            op_crop_resize(frames, t, 256, 128)
    with pytest.raises(RuntimeError, match="batch"):
        eng.embed_boxes(frames, np.concatenate([boxes, boxes[:1]]))                   # n > B
    np.testing.assert_array_equal(eng.get_activation("conv1"), conv1)                # nothing ran in between
    np.testing.assert_array_equal(eng.embed_boxes(frames, boxes), good)
    eng.close()
