"""References for main.py --mode forward's scene feature (models.py:517-518): fpn_feature is p5 transposed to NHWC and
resized to 7 x 7 by tf.image.resize_images, TF1's legacy bilinear (align_corners=False, half_pixel_centers=False).
`fpn_feature` runs the oracle's float32 restatement of that resize (oracle/efficientnet.py resize_bilinear_legacy) on a p5;
`fpn_feature_exact` is an independent per-pixel evaluation of TF's formula: indices from the float32 scale and coordinate
as TF computes them, the interpolation in float64."""
import math

import numpy as np


def fpn_feature(p5_chw):
    """[1, 7, 7, C] float32 of one image's p5 [C, h, w]."""
    from oracle.efficientnet import resize_bilinear_legacy
    return resize_bilinear_legacy(np.ascontiguousarray(np.transpose(p5_chw, (1, 2, 0)), np.float32), 7, 7)[None]


def taps(in_size, out_size=7):
    """TF's LegacyScaler per output index: (lo, hi, lerp) with lerp as the float32 value TF uses."""
    scale = np.float32(in_size) / np.float32(out_size)
    out = []
    for d in range(out_size):
        x = np.float32(np.float32(d) * scale)
        lo = int(math.floor(x))
        out.append((lo, min(int(math.ceil(x)), in_size - 1), float(np.float32(x - np.float32(lo)))))
    return out


def fpn_feature_exact(p5_chw):
    """[1, 7, 7, C] float64."""
    p = np.asarray(p5_chw, np.float64)
    C, h, w = p.shape
    out = np.empty((1, 7, 7, C), np.float64)
    for oy, (y0, y1, ly) in enumerate(taps(h)):
        for ox, (x0, x1, lx) in enumerate(taps(w)):
            top = p[:, y0, x0] + (p[:, y0, x1] - p[:, y0, x0]) * lx
            bot = p[:, y1, x0] + (p[:, y1, x1] - p[:, y1, x0]) * lx
            out[0, oy, ox] = top + (bot - top) * ly
    return out
