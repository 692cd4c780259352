"""ReID crop resize (csrc/reid_ingest.cu): the numpy restatement of Pillow's bilinear resize (tests/pil_resize_oracle.py)
against live Pillow and against the committed Pillow golden (tests/golden/reid_crops_pil.npz, written by
tests/golden/make_golden_reid_crops.py), and the kernel's arithmetic (csrc/pil_resize_math.h, compiled here into a host
harness) against the oracle."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import pil_resize_oracle as oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZES = ((256, 128), (128, 256))   # (out_h, out_w): osnet_x1_0, resnet101

# (w, h) crops: upscaling, identity, one-pixel rows and columns, whole 2160-row heights and 3840-wide rows, and both
# sides of Image.resize's 100x rule
EDGE_SHAPES = [(1, 1), (2, 3), (7, 5), (13, 29), (128, 256), (256, 128), (1, 200), (200, 1), (1, 420), (330, 1),
               (4, 400), (4, 410), (3, 420), (60, 150), (330, 420), (24, 2160), (7, 2160), (1, 2160), (4, 2160),
               (3840, 8), (3840, 1), (2840, 8), (1, 700), (3840, 16), (4, 604), (3, 500), (2, 260), (2, 300), (5, 501),
               (1, 101), (1, 100), (127, 255), (129, 257), (255, 129), (257, 127), (300, 120), (600, 250), (120, 50)]


def sweep_shapes():
    rng = np.random.default_rng(4242)
    shapes = list(EDGE_SHAPES)
    while len(shapes) < 110:
        w = int(rng.integers(1, 400))
        h = int(rng.integers(1, 800)) if rng.random() < 0.8 else int(rng.integers(101 * w, 101 * w + 300))
        shapes.append((w, h))
    return shapes                                     # x 2 output sizes = 220 cases


def test_sweep_covers_the_required_shapes():
    shapes = sweep_shapes()
    assert len(shapes) * len(SIZES) >= 200
    vfirst = [(w, h) for w, h in shapes if h > 100 * w]
    assert (4, 410) in vfirst and (4, 400) in shapes and (4, 400) not in vfirst
    assert (1, 1) in shapes and (24, 2160) in shapes and (3840, 1) in shapes and len(vfirst) >= 15


def test_oracle_matches_live_pillow():
    Image = pytest.importorskip("PIL.Image")
    rng = np.random.default_rng(99)
    for w, h in sweep_shapes():
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        for out_h, out_w in SIZES:
            ref = np.asarray(Image.fromarray(img).resize((out_w, out_h), Image.BILINEAR), np.uint8)
            np.testing.assert_array_equal(oracle.resize(img, out_w, out_h), ref, err_msg="%dx%d -> %dx%d" % (w, h, out_w,
                                                                                                               out_h))


@pytest.fixture(scope="module")
def golden(golden_dir):
    return oracle.load_golden(os.path.join(golden_dir, "reid_crops_pil.npz"))


def test_golden_covers_the_required_boxes(golden):
    seen = set()
    for g in range(int(golden["num_groups"])):
        H, W = golden["g%d_frames" % g].shape[1:3]
        for _, x, y, w, h in golden["g%d_boxes" % g]:
            seen.add((int(w), int(h)))
            seen.update(edge for edge, hit in (("left", x == 0), ("top", y == 0), ("right", x + w == W),
                                                ("bottom", y + h == H)) if hit)
    for need in ((1, 1), (128, 256), (256, 128), (1, 200), (200, 1), (4, 400), (4, 410), (24, 2160), (7, 2160),
                 (3840, 1), "left", "top", "right", "bottom"):
        assert need in seen, need


def test_oracle_matches_golden(golden):
    for g in range(int(golden["num_groups"])):
        frames, boxes = golden["g%d_frames" % g], golden["g%d_boxes" % g]
        for out_h, out_w in SIZES:
            ref = golden["g%d_crops_%dx%d" % (g, out_h, out_w)]
            for i, b in enumerate(boxes):
                np.testing.assert_array_equal(oracle.crop_resize(frames[b[0]], b[1:], out_w, out_h), ref[i],
                                              err_msg="group %d box %s -> %dx%d" % (g, b, out_w, out_h))


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("pil_resize") / "libpil_resize_harness.so")
    subprocess.run(["g++", "-O2", "-shared", "-fPIC", "-o", out, os.path.join(ROOT, "tests", "pil_resize_harness.cpp")],
                   check=True)
    lib = ctypes.CDLL(out)
    lib.pil_resize_harness.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int,
                                       ctypes.c_int]
    lib.pil_resize_harness.restype = None
    return lib


def test_kernel_arithmetic_matches_oracle(harness, golden):
    rng = np.random.default_rng(7)
    cases = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for w, h in sweep_shapes()]
    for g in range(int(golden["num_groups"])):
        frames = golden["g%d_frames" % g]
        cases += [frames[b[0], b[2]:b[2] + b[4], b[1]:b[1] + b[3], ::-1] for b in golden["g%d_boxes" % g]]
    for src in cases:
        src = np.ascontiguousarray(src)
        for out_h, out_w in SIZES:
            dst = np.empty((out_h, out_w, 3), np.uint8)
            harness.pil_resize_harness(src.ctypes.data, src.shape[0], src.shape[1], dst.ctypes.data, out_h, out_w)
            np.testing.assert_array_equal(dst, oracle.resize(src, out_w, out_h),
                                          err_msg="%dx%d -> %dx%d" % (src.shape[1], src.shape[0], out_w, out_h))


def test_extract_boxes_refuses_empty_or_outside_crops():
    """extract_boxes checks the int()-truncated crops before the engine is touched: no GPU needed for the refusals."""
    from object_detection_tracking_b200.reid import FeatureExtractor
    ext = FeatureExtractor.__new__(FeatureExtractor)        # the checks run before any engine call
    ext.batch, ext.engine = 4, None
    frame = np.zeros((50, 40, 3), np.uint8)
    for tlwh in ((0, 0, 0.9, 20), (0, 0, 10, 0.5), (35.5, 0, 6, 10), (0, 45, 10, 6), (-1, 0, 10, 10), (0, -1.5, 10, 10.0)):
        with pytest.raises(ValueError):
            ext.extract_boxes(frame, [(1, 1, 5, 5), tlwh])
    with pytest.raises(ValueError):
        ext.extract_boxes(frame.astype(np.float32), [(1, 1, 5, 5)])
