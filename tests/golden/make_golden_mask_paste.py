"""Writes tests/golden/mask_paste_cv2.npz: cv2.resize(mask, (w, h)) > 0.5 of 28x28 float32 masks, the patch
fill_full_mask (nn.py:1565-1584) pastes, as OpenCV computes it with its default settings.  Written with OpenCV 4.13.

Masks: seeded uniform noise, a smooth blob, and masks within a few ulps of 0.5, so that the threshold decides pixels where
a slip in the resize arithmetic would show.  Sizes: 1..57 on each axis, 14x14, 28x28, up to 3840 wide and 2160 tall.
The thresholded patches are stored bit-packed (np.packbits of the row-major patch); raw float32 outputs only for patches
of at most 1024 pixels, to keep the file small.

    python tests/golden/make_golden_mask_paste.py
"""
import os

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
RAW_MAX = 1024


def golden_masks():
    rng = np.random.default_rng(2028)
    noise = rng.random((28, 28), dtype=np.float32)
    yy, xx = np.mgrid[0:28, 0:28].astype(np.float32)
    blob = (1.0 / (1.0 + np.exp(((xx - 13.2) ** 2 + (yy - 15.7) ** 2) / 40.0 - 2.0))).astype(np.float32)
    near = np.float32(0.5) + rng.integers(-4, 5, (28, 28)).astype(np.float32) * np.float32(2.0 ** -24)   # exact
    return np.stack([noise, blob, near])


def golden_sizes():
    rng = np.random.default_rng(77)
    sizes = [(w, int(rng.integers(1, 120))) for w in range(1, 58)] + [(int(rng.integers(1, 120)), h) for h in range(1, 58)]
    sizes += [(14, 14), (28, 28), (1, 1), (3840, 2), (3840, 1), (2, 2160), (1, 2160), (1920, 3), (500, 400), (121, 377)]
    return sizes


def main():
    masks = golden_masks()
    sizes = golden_sizes()
    out = {"masks": masks, "sizes": np.array(sizes, np.int32), "cv2_version": np.array(cv2.__version__)}
    assert cv2.useOptimized()
    for i, (w, h) in enumerate(sizes):
        for k, m in enumerate(masks):
            r = cv2.resize(m, (w, h))
            out["bits_%d_%d" % (i, k)] = np.packbits((r > 0.5).astype(np.uint8).ravel())
            if w * h <= RAW_MAX:
                out["raw_%d_%d" % (i, k)] = r
    np.savez_compressed(os.path.join(HERE, "mask_paste_cv2.npz"), **out)


if __name__ == "__main__":
    main()
