"""numpy restatement of Pillow's Image.resize(size, BILINEAR) on 8-bit RGB (libImaging/Resample.c and Image.resize in
PIL/Image.py), the resize step of torchreid's FeatureExtractor (feature_extractor.py:190-196).  The algorithm is spelled
out in object_detection_tracking_b200/csrc/pil_resize_math.h, which the crop-resize kernel compiles; this module is the
CPU oracle the CPU tests pin against live Pillow and the committed golden, and the kernel's host harness against."""
import math

import numpy as np

PRECISION_BITS = 22


def coeffs(in_size, out_size):
    """-> (xmin [out], k [out, ksize] int64): first source index and fixed-point weights of each output index (weights
    past an index's own tap count are 0)."""
    scale = float(in_size) / float(out_size)
    fs = max(scale, 1.0)
    support = fs * 1.0
    ksize = int(math.ceil(support)) * 2 + 1
    ss = 1.0 / fs
    xmin = np.zeros(out_size, np.int64)
    k = np.zeros((out_size, ksize), np.int64)
    for xx in range(out_size):
        centre = (xx + 0.5) * scale
        lo = max(int(centre - support + 0.5), 0)
        n = min(int(centre + support + 0.5), in_size) - lo
        w = [max(0.0, 1.0 - abs((x + lo - centre + 0.5) * ss)) for x in range(n)]
        ww = 0.0
        for v in w:
            ww += v
        for x in range(n):
            v = w[x] / ww if ww != 0.0 else w[x]
            k[xx, x] = int(-0.5 + v * (1 << PRECISION_BITS)) if v < 0 else int(0.5 + v * (1 << PRECISION_BITS))
        xmin[xx] = lo
    return xmin, k


def _pass(img, out_size, axis):
    """One 1-D pass of uint8 img [h, w, c] along `axis` (1 horizontal, 0 vertical) -> uint8; identity when the size does
    not change (Pillow skips that pass)."""
    in_size = img.shape[axis]
    if in_size == out_size:
        return img
    xmin, k = coeffs(in_size, out_size)
    src = np.moveaxis(img, axis, 0).astype(np.int64)
    acc = np.full((out_size,) + src.shape[1:], 1 << (PRECISION_BITS - 1), np.int64)
    for x in range(k.shape[1]):
        idx = np.minimum(xmin + x, in_size - 1)          # taps past the count carry weight 0
        acc += src[idx] * k[:, x].reshape((-1,) + (1,) * (src.ndim - 1))
    out = np.clip(acc >> PRECISION_BITS, 0, 255).astype(np.uint8)
    return np.moveaxis(out, 0, axis)


def resize(img, out_w, out_h):
    """uint8 [h, w, c] -> uint8 [out_h, out_w, c] as Image.fromarray(img).resize((out_w, out_h), Image.BILINEAR)."""
    img = np.asarray(img, dtype=np.uint8)
    h, w = img.shape[:2]
    if (h, w) == (out_h, out_w):
        return img.copy()
    if h > 100 * w and out_h < h:                        # Image.resize: vertical first for very tall inputs
        return _pass(_pass(img, out_h, 0), out_w, 1)
    return _pass(_pass(img, out_w, 1), out_h, 0)


def crop_resize(frame_bgr, box, out_w, out_h):
    """One track box (x, y, w, h) of a BGR frame -> its RGB crop resized, as the drivers prepare a ReID input."""
    x, y, w, h = (int(v) for v in box)
    return resize(frame_bgr[y:y + h, x:x + w, ::-1], out_w, out_h)


def load_golden(path):
    """tests/golden/reid_crops_pil.npz with its row-delta images restored: {name: array}."""
    g = dict(np.load(path))
    for k, v in g.items():
        if v.dtype == np.uint8 and v.ndim == 4:
            g[k] = np.cumsum(v, axis=-2, dtype=np.uint8)
    return g
