"""Writes tests/golden/reid_crops_pil.npz: seeded uint8 BGR frames, track-box tables [n][5] (frame, x, y, w, h) and what
Pillow makes of each box as the drivers prepare a ReID input (single_video_reid.py:211-227 + torchreid's T.Resize):
Image.fromarray(frame[y:y+h, x:x+w, ::-1]).resize((out_w, out_h), Image.BILINEAR), for both ReID crop sizes (256x128
OSNet, 128x256 ResNet-101).  The Pillow version is recorded in the file, so the tests that read it do not depend on the
Pillow a machine has installed.

Three groups of one frame shape each (one b2_reid_embed_boxes call takes frames of one shape):
  g0: two 264x264 frames -- upscaling down to 1x1, identity (128x256 and 256x128 boxes), one-pixel rows and columns,
      boxes on every frame edge and seeded person-shaped boxes;
  g1: one 2160x24 frame -- the whole 2160-row height into 128 (and 256) rows, vertical-first and not, and both sides of
      Image.resize's 100x rule (w 4 with h 400 and 410);
  g2: one 8x3840 frame -- a whole 3840-wide row into 256 (and 128) columns.
The frames are smooth textures without noise, and every uint8 image array is stored as its differences along the row
(mod 256), so that deflate packs the file small; tests/pil_resize_oracle.py load_golden() undoes the differences.  The
GPU tests also check the kernel against the oracle on seeded noise frames, which need no file.
Run: python tests/golden/make_golden_reid_crops.py
"""
import os

import numpy as np
import PIL
from PIL import Image

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reid_crops_pil.npz")
SIZES = ((256, 128), (128, 256))   # (out_h, out_w): osnet_x1_0, resnet101


def frames(rng, nf, h, w):
    """Smooth gradients with a sine texture, wrapped mod 256: every level 0..255 occurs."""
    yy, xx = np.mgrid[0:h, 0:w]
    out = np.empty((nf, h, w, 3), np.uint8)
    for f in range(nf):
        for c in range(3):
            a, b, p = rng.uniform(-1.5, 1.5), rng.uniform(-1.5, 1.5), rng.uniform(0, 255)
            base = (a * xx + b * yy + p + 40 * np.sin(xx / rng.uniform(20, 60)) * np.cos(yy / rng.uniform(20, 60))) % 256
            out[f, ..., c] = base.astype(np.uint8)
    return out


def g0_boxes(rng, nf, H, W):
    b = [(0, 0, 0, 1, 1), (1, 200, 100, 1, 1), (0, 17, 33, 2, 3), (1, 5, 9, 7, 5), (0, 30, 40, 13, 29),
         (0, 4, 3, 128, 256), (1, 6, 7, 256, 128),                                   # identity for each model
         (0, 11, 0, 1, 200), (1, 0, 30, 200, 1), (0, W - 1, 0, 1, H), (1, 0, H - 1, W, 1),
         (0, 0, 0, 60, 150), (1, W - 90, H - 200, 90, 200)]
    for _ in range(2):                                                                # person-shaped
        w = int(rng.integers(16, 160))
        h = min(H, int(w * rng.uniform(1.6, 3.2)))
        b.append((int(rng.integers(0, nf)), int(rng.integers(0, W - w + 1)), int(rng.integers(0, H - h + 1)), w, h))
    return np.asarray(b, np.int32)


def pil_crop(frame_bgr, box, out_h, out_w):
    _, x, y, w, h = (int(v) for v in box)
    img = Image.fromarray(np.ascontiguousarray(frame_bgr[y:y + h, x:x + w, ::-1]))
    return np.asarray(img.resize((out_w, out_h), Image.BILINEAR), np.uint8)


def row_delta(a):
    """uint8 [..., w, 3] -> its differences along w, mod 256 (the first column kept)."""
    d = a.copy()
    d[..., 1:, :] = a[..., 1:, :] - a[..., :-1, :]
    return d


def main():
    rng = np.random.default_rng(20261017)
    groups = [
        (frames(rng, 2, 264, 264), None),
        (frames(rng, 1, 2160, 24), np.asarray([(0, 0, 0, 24, 2160), (0, 3, 0, 7, 2160), (0, 0, 0, 1, 2160),
                                               (0, 20, 0, 4, 2160), (0, 10, 1000, 2, 1160),
                                               (0, 5, 17, 4, 400), (0, 9, 1700, 4, 410), (0, 0, 0, 3, 420)], np.int32)),
        (frames(rng, 1, 8, 3840), np.asarray([(0, 0, 0, 3840, 8), (0, 0, 3, 3840, 1), (0, 0, 7, 3840, 1)],
                                             np.int32)),
    ]
    groups[0] = (groups[0][0], g0_boxes(rng, 2, 264, 264))
    data = {"pillow_version": np.asarray(PIL.__version__), "num_groups": np.asarray(len(groups))}
    for g, (fr, bx) in enumerate(groups):
        data["g%d_frames" % g] = row_delta(fr)
        data["g%d_boxes" % g] = bx
        for out_h, out_w in SIZES:
            data["g%d_crops_%dx%d" % (g, out_h, out_w)] = row_delta(np.stack([pil_crop(fr[b[0]], b, out_h, out_w)
                                                                             for b in bx]))
    np.savez_compressed(OUT, **data)
    print("wrote %s (Pillow %s, %d bytes)" % (OUT, PIL.__version__, os.path.getsize(OUT)))


if __name__ == "__main__":
    main()
