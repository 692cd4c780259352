"""Mask paste and RLE (csrc/mask_rle.cu): the NumPy restatement (tests/mask_rle_oracle.py) against live cv2 and the
committed cv2 golden (tests/golden/mask_paste_cv2.npz, written by tests/golden/make_golden_mask_paste.py), its RLE against
pycocotools' known answers, and the kernels' arithmetic (csrc/mask_rle_math.h, compiled here into a host harness) against
the oracle."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import mask_rle_oracle as oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def sweep_sizes():
    rng = np.random.default_rng(515)
    sizes = [(w, int(rng.integers(1, 200))) for w in range(1, 58)] + [(int(rng.integers(1, 200)), h) for h in range(1, 58)]
    sizes += [(14, 14), (28, 28), (1, 1), (3840, 4), (3840, 1), (2560, 7), (1920, 2), (5, 2160), (400, 399)]
    while len(sizes) < 300:
        sizes.append((int(rng.integers(1, 700)), int(rng.integers(1, 700))))
    return sizes


def sweep_masks(rng):
    near = np.float32(0.5) + rng.integers(-3, 4, (28, 28)).astype(np.float32) * np.float32(2.0 ** -24)
    return [rng.random((28, 28), dtype=np.float32), near]


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "mask_paste_cv2.npz"))


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("mask_rle") / "libmask_rle_harness.so")
    subprocess.run(["g++", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-o", out,
                    os.path.join(ROOT, "tests", "mask_rle_harness.cpp")], check=True)
    lib = ctypes.CDLL(out)
    lib.mask_geometry_harness.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    lib.mask_resize_harness.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
    lib.rle_string_harness.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
    lib.rle_string_harness.restype = ctypes.c_int64
    lib.fmaf_harness.argtypes = [ctypes.c_void_p] * 4 + [ctypes.c_int]
    return lib


# -- the oracle's fmaf -------------------------------------------------------------------------------------------------

def test_oracle_fmaf_rounds_once(harness):
    rng = np.random.default_rng(3)
    n = 200000
    a = rng.standard_normal(n).astype(np.float32)
    b = rng.random(n, dtype=np.float32)
    c = rng.standard_normal(n).astype(np.float32)
    # midpoint-adversarial: a * b = 2^-24 - 2^-70, half an ulp of c in [1, 2) less a term float64 drops, so c + a * b
    # rounds in float64 to the midpoint and then, by ties-to-even, the wrong way for every odd c
    c2 = np.float32(1.0) + np.arange(n, dtype=np.float32) * np.float32(2.0 ** -23)
    a2 = np.full(n, 1.0 + 2.0 ** -23, np.float32)
    b2 = np.full(n, 2.0 ** -24 - 2.0 ** -47, np.float32)
    for x, y, z in ((a, b, c), (a2, b2, c2), (-a2, b2, c2)):
        ref = np.empty(n, np.float32)
        harness.fmaf_harness(x.ctypes.data, y.ctypes.data, z.ctypes.data, ref.ctypes.data, n)
        np.testing.assert_array_equal(oracle.fmaf(x, y, z).view(np.uint32), ref.view(np.uint32))
    naive = (a2.astype(np.float64) * b2.astype(np.float64) + c2.astype(np.float64)).astype(np.float32)
    assert (naive != oracle.fmaf(a2, b2, c2)).any()     # the case double rounding gets wrong


# -- resize against cv2 -------------------------------------------------------------------------------------------------

def test_sweep_covers_the_required_sizes():
    s = set(sweep_sizes())
    assert len(s) >= 250 and (14, 14) in s and (28, 28) in s and (3840, 4) in s
    assert {w for w, _ in s} >= set(range(1, 58)) and {h for _, h in s} >= set(range(1, 58))


def test_oracle_matches_live_cv2():
    cv2 = pytest.importorskip("cv2")
    assert cv2.useOptimized()
    rng = np.random.default_rng(11)
    for w, h in sweep_sizes():
        for m in sweep_masks(rng):
            np.testing.assert_array_equal(oracle.resize(m, w, h).view(np.uint32), cv2.resize(m, (w, h)).view(np.uint32),
                                          err_msg="%dx%d" % (w, h))


def test_oracle_matches_golden(golden):
    masks, sizes = golden["masks"], golden["sizes"]
    assert len(sizes) >= 120 and masks.shape == (3, 28, 28)
    raw = 0
    for i, (w, h) in enumerate(sizes):
        for k, m in enumerate(masks):
            r = oracle.resize(m, int(w), int(h))
            bits = np.unpackbits(golden["bits_%d_%d" % (i, k)], count=int(w) * int(h))
            np.testing.assert_array_equal((r > 0.5).astype(np.uint8).ravel(), bits, err_msg="%dx%d mask %d" % (w, h, k))
            if "raw_%d_%d" % (i, k) in golden.files:
                raw += 1
                np.testing.assert_array_equal(r.view(np.uint32), golden["raw_%d_%d" % (i, k)].view(np.uint32))
    assert raw >= 100
    # the near-0.5 mask really straddles the threshold
    on = np.unpackbits(golden["bits_%d_2" % list(map(tuple, sizes)).index((28, 28))])
    assert 0 < on.sum() < on.size


def test_harness_resize_matches_oracle(harness, golden):
    rng = np.random.default_rng(12)
    cases = [(m, w, h) for w, h in sweep_sizes()[::3] for m in sweep_masks(rng)]
    cases += [(m, int(w), int(h)) for w, h in golden["sizes"] for m in golden["masks"]]
    for m, w, h in cases:
        m = np.ascontiguousarray(m, np.float32)
        out = np.empty((h, w), np.float32)
        on = np.empty((h, w), np.uint8)
        harness.mask_resize_harness(m.ctypes.data, w, h, out.ctypes.data, on.ctypes.data)
        ref = oracle.resize(m, w, h)
        np.testing.assert_array_equal(out.view(np.uint32), ref.view(np.uint32), err_msg="%dx%d" % (w, h))
        np.testing.assert_array_equal(on, (ref > 0.5).astype(np.uint8))


# -- geometry ----------------------------------------------------------------------------------------------------------

def _harness_geometry(harness, box, H, W):
    box = np.asarray(box, np.float32)
    out = np.zeros(6, np.int32)
    harness.mask_geometry_harness(box.ctypes.data, H, W, out.ctypes.data)
    return out


GEOMETRY_CASES = [
    ((10.2, 20.7, 30.4, 40.6), 100, 100),     # ordinary
    ((0.0, 0.0, 1.0, 1.0), 5, 5),             # 1x1 at the origin
    ((-0.9, -0.6, 3.0, 4.0), 50, 50),         # int() truncates -0.4 / -0.1 to 0, floor would not
    ((5.0, 5.0, 5.2, 5.3), 50, 50),           # x1 < x0 clamped: 1x1
    ((3.0, 3.0, 0.4, 0.2), 50, 50),           # box[2:] - 0.5 in (-1, 0): truncates to 0, then clamped
    ((0.0, 0.0, 64.0, 48.0), 48, 64),         # the full frame
    ((0.0, 0.0, 10.0, 48.3), 48, 64),         # y1 = int(47.8) = 47: fits
    ((0.0, 0.0, 10.0, 49.0), 48, 64),         # y1 = 48 = H: the slice is cut short -> ValueError
    ((60.0, 0.0, 66.0, 10.0), 48, 64),        # x1 = 65 >= W -> ValueError
    ((70.0, 10.0, 70.2, 20.0), 48, 64),       # x0 >= W with a 1-wide patch: broadcasts into the empty slice
    ((10.0, 50.0, 20.0, 50.1), 48, 64),       # y0 >= H with a 1-tall patch: the same
    ((70.0, 10.0, 75.0, 20.0), 48, 64),       # x0 >= W, 5 wide -> ValueError
    ((63.0, 47.0, 64.0, 48.0), 48, 64),       # the last pixel
    ((-2.0, 0.0, 5.0, 5.0), 48, 64),          # negative corner: refused
    ((0.0, -1.6, 5.0, 5.0), 48, 64),
]


def _oracle_status(box, H, W):
    x0, y0, x1, y1, w, h = oracle.geometry(box)
    if x0 < 0 or y0 < 0:
        return 1, None
    try:
        np.zeros((H, W), np.uint8)[y0:y1 + 1, x0:x1 + 1] = np.ones((h, w), np.uint8)
    except ValueError:
        return 2, None
    return 0, (x0, y0, w, h, int(x0 < W and y0 < H))


def test_geometry_matches_numpy(harness):
    statuses = set()
    rng = np.random.default_rng(5)
    cases = list(GEOMETRY_CASES)
    for _ in range(3000):
        H, W = int(rng.integers(1, 60)), int(rng.integers(1, 60))
        x0, y0 = rng.uniform(-2, W + 2), rng.uniform(-2, H + 2)
        cases.append(((x0, y0, x0 + rng.uniform(-2, W), y0 + rng.uniform(-2, H)), H, W))
    for box, H, W in cases:
        got = _harness_geometry(harness, box, H, W)
        st, place = _oracle_status(box, H, W)
        statuses.add(st)
        assert got[0] == st, (box, H, W, got)
        if st == 0:
            assert tuple(got[1:]) == place, (box, H, W, got, place)
    assert statuses == {0, 1, 2}
    assert _harness_geometry(harness, (np.nan, 0, 1, 1), 8, 8)[0] == 3
    assert _harness_geometry(harness, (0, 0, 2.0 ** 31, 1), 8, 8)[0] == 3


def test_issue_overhang_example():
    """A 1281x2989 frame resized to 720 / 1280 (scale 1280 / 2989, 549 rows): a box touching the resized frame's bottom
    edge gives y1 = int(549 / scale - 0.5) = H, and fill_full_mask raises."""
    H, W = 1281, 2989
    scale = min(720.0 / H, 1280.0 / W)
    box = np.array([100.0, 300.0, 600.0, int(H * scale + 0.5)], np.float32) / scale
    assert box.dtype == np.float32
    x0, y0, x1, y1, w, h = oracle.geometry(box)
    assert y1 == H
    with pytest.raises(ValueError):
        oracle.fill_full_mask(box, np.ones((28, 28), np.float32), (H, W))


# -- RLE ---------------------------------------------------------------------------------------------------------------

def test_rle_known_answers(harness):
    assert oracle.rle_counts(np.array([[0, 1], [1, 1]], np.uint8)) == [1, 3]
    assert oracle.rle_string([1, 3]) == "13"
    assert oracle.rle_counts(np.array([[1]], np.uint8)) == [0, 1]
    assert oracle.rle_string([0, 1]) == "01"
    assert oracle.rle_string([100]) == "T3"
    assert oracle.rle_string([0, 10, 0, 5])[-1] == "K"         # count 5 after count 10: a delta of -5
    for counts in ([1, 3], [0, 1], [100], [0, 10, 0, 5], [7, 1, 9, 300, 2, 70000, 1, 1, 5000000]):
        c = np.array(counts, np.int64)
        buf = ctypes.create_string_buffer(8 * len(counts) + 1)
        n = harness.rle_string_harness(c.ctypes.data, len(counts), buf)
        assert buf.raw[:n].decode("ascii") == oracle.rle_string(counts)


def _masks_for_rle():
    rng = np.random.default_rng(6)
    yield np.zeros((7, 5), np.uint8)
    yield np.ones((7, 5), np.uint8)
    yield (np.indices((9, 11)).sum(0) % 2).astype(np.uint8)       # checkerboard: the longest strings
    yield (np.indices((1, 13)).sum(0) % 2).astype(np.uint8)
    for _ in range(40):
        H, W = int(rng.integers(1, 40)), int(rng.integers(1, 40))
        yield (rng.random((H, W)) < rng.random()).astype(np.uint8)


def test_rle_round_trips(harness):
    for full in _masks_for_rle():
        H, W = full.shape
        counts = oracle.rle_counts(full)
        assert sum(counts) == H * W
        s = oracle.rle_string(counts)
        assert oracle.rle_parse(s) == counts
        np.testing.assert_array_equal(oracle.rle_decode(counts, H, W), full)
        c = np.array(counts, np.int64)
        buf = ctypes.create_string_buffer(8 * len(counts) + 1)
        n = harness.rle_string_harness(c.ctypes.data, len(counts), buf)
        assert buf.raw[:n].decode("ascii") == s
    assert oracle.rle_counts(np.zeros((3, 4), np.uint8)) == [12]
    assert oracle.rle_counts(np.ones((3, 4), np.uint8)) == [0, 12]


def test_rle_matches_pycocotools_when_importable():
    mask = pytest.importorskip("pycocotools.mask")
    for full in _masks_for_rle():
        rle = mask.encode(np.array(full[:, :, None], order="F"))[0]
        rle["counts"] = rle["counts"].decode("ascii")
        assert rle == oracle.encode(full)


def test_refusals_need_no_gpu():
    """Shape and dtype refusals happen in Python before the library is asked for anything."""
    from object_detection_tracking_b200 import masks
    enc = masks.MaskEncoder.__new__(masks.MaskEncoder)
    with pytest.raises(TypeError):
        masks._boxes(np.zeros((2, 4), np.float64))
    with pytest.raises(ValueError):
        masks._im_shape((10, 10, 3))
    with pytest.raises(ValueError):
        enc._mask_hw((2, 14, 14, 1), 2)
    with pytest.raises(ValueError):
        enc._mask_hw((3, 28, 28), 2)
