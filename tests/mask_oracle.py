"""Float64 reference of the mask head one layer at a time (models.py:934-961, 1173-1199), with an element-wise error bound
per layer.

Each layer is computed from the engine's own previous layer as its planes hold it, so what is left between a layer's
output and its reference is that layer's arithmetic alone:
  ROIAlign 14   oracle.frcnn.multilevel_roi_align(..., 14, ...), exact float32: compared bit for bit through the planes
  fcn0..fcn3    conv 3x3 SAME + bias + ReLU, K = 2304 (conv_oracle.reference / bound)
  deconv        Conv2DTranspose 2x2 stride 2 + bias + ReLU, written from the TF kernel layout [kh, kw, out, in]:
                out[2y + dy, 2x + dx, o] = sum_i W[dy, dx, o, i] x[y, x, i] + b[o], K = 256
  class conv    1x1 + bias, K = 256, fp32 output
  mask select   sigmoid of the box's own class, within sigmoid_bound of the float64 sigmoid of the engine's logit

The engine holds the deconv output as (tap, channel) rows -- pixel (y, x) of a box, channel t * 256 + o with
t = dy * 2 + dx -- and mask_select_kernel un-shuffles the class conv's rows (roi * 196 + (Y >> 1) * 14 + (X >> 1)) * 4 +
(Y & 1) * 2 + (X & 1).  `pack_deconv`, `unshuffle` and `mask_rows` restate those two index conventions so that
test_mask_oracle_cpu.py can pin them against oracle.frcnn.maskrcnn_head.
"""
from __future__ import annotations

import numpy as np

import conv_oracle as co

F32 = np.float32
U = 2.0 ** -24


def samples(c0, c1, dim, crop=14):
    """The float32 sample coordinates of oracle.frcnn.roi_align / tf_ops.crop_and_resize along one axis of `dim` pixels
    for a box side [c0, c1] in level coordinates and a crop of `crop` samples (2 x the output bins)."""
    f = F32
    sp = f(f(c1 - c0) / f(crop))
    n0 = f(f(f(c0 + f(sp / f(2))) - f(0.5)) / f(dim - 1))
    nl = f(f(sp * f(crop - 1)) / f(dim - 1))
    n1 = f(n0 + nl)
    sc = f(f(f(n1 - n0) * f(dim - 1)) / f(crop - 1))
    return f(n0 * f(dim - 1)) + np.arange(crop, dtype=f) * sc


def roi14(feats, boxes, strides=(4, 8, 16, 32)):
    """ROIAlign 14 of one image's boxes [n, 4] on its cropped levels feats[l] [C, h, w]: [n, 14, 14, C] float32."""
    from oracle import frcnn
    r, _ = frcnn.multilevel_roi_align(feats, np.asarray(boxes, F32), 14, strides)
    return np.ascontiguousarray(r.transpose(0, 2, 3, 1))


def fcn(x, w, b, split=True):
    """conv 3x3 SAME + bias + ReLU of the held maps x [M, 14, 14, C]: conv_oracle.reference's dict (ref, S, b, K ...)."""
    return co.reference(np.asarray(x, F32), np.asarray(w, F32), bias=b, pad=(1, 1, 1, 1), relu=1, split=split)


def held(x, split):
    """x as the kernels hold it in `split` precision (True / False), or x itself in float64 with split None."""
    return np.asarray(x, np.float64) if split is None else co.represent(x, split)


def fcn64(x, w, b):
    """conv 3x3 SAME + bias + ReLU in plain float64 (no plane rounding): x [M, 14, 14, C], w HWIO."""
    return np.maximum(co._conv64(np.asarray(x, np.float64), np.asarray(w, np.float64), 1, 1, (1, 1, 1, 1)) +
                      np.asarray(b, np.float64), 0.0)


def deconv28(x, w, b, split=True):
    """The transposed conv from the TF layout: x [M, 14, 14, Ci], w [2, 2, Co, Ci], b [Co], both as held in `split`
    precision (held).  Returns (out, S) as [M, 28, 28, Co] float64: out = relu(sum_i W~[dy, dx, o, i] x~[y, x, i] + b[o])
    at (2y + dy, 2x + dx), S the sum of |products|."""
    xr = held(x, split)
    wr = held(w, split)
    M, H, W_, _ = xr.shape
    Co = wr.shape[2]
    t = np.einsum("myxi,deoi->mydxeo", xr, wr).reshape(M, 2 * H, 2 * W_, Co) + np.asarray(b, F32).astype(np.float64)
    S = np.einsum("myxi,deoi->mydxeo", np.abs(xr), np.abs(wr)).reshape(M, 2 * H, 2 * W_, Co)
    return np.maximum(t, 0.0), S


def pack_deconv(w):
    """load_layer's kDeconv packing (detplan.cu): the TF kernel [2, 2, Co, Ci] as the [4 Co][Ci] weights of a 1x1 conv,
    output row (dy * 2 + dx) * Co + o."""
    w = np.asarray(w)
    return w.reshape(4 * w.shape[2], w.shape[3])


def unshuffle(up):
    """The engine's (tap, channel) maps up [M, 14, 14, 4 Co] (channel (dy * 2 + dx) * Co + o at pixel (y, x)) as the
    [M, 28, 28, Co] map they stand for."""
    M, H, W_, C4 = up.shape
    return up.reshape(M, H, W_, 2, 2, C4 // 4).transpose(0, 1, 3, 2, 4, 5).reshape(M, 2 * H, 2 * W_, C4 // 4)


def mask_rows(logits, M):
    """mask_select_kernel's read of the class conv's rows: logits [M * 784, ld] as [M, 28, 28, ld], pixel (Y, X) of box m
    at row (m * 196 + (Y >> 1) * 14 + (X >> 1)) * 4 + (Y & 1) * 2 + (X & 1)."""
    Y, X = np.meshgrid(np.arange(28), np.arange(28), indexing="ij")
    rows = (np.arange(M)[:, None, None] * 196 + (Y >> 1) * 14 + (X >> 1)) * 4 + (Y & 1) * 2 + (X & 1)
    return np.asarray(logits)[rows]


def class_conv(up, w, b, split=True):
    """The 1x1 class conv over the held (pixel, tap) rows: up [M, 14, 14, 4 C] -> conv_oracle.reference's dict over
    [1, 1, M * 784, ld] (w [1, 1, C, Cout], fp32 output)."""
    C = w.shape[2]
    rows = np.asarray(up, F32).reshape(1, 1, -1, C)
    return co.reference(rows, np.asarray(w, F32), bias=b, split=split)


def bound(r, precision, out="planes"):
    """conv_oracle.bound of a reference dict r from fcn / class_conv (or a dict with K, S, b, ref)."""
    return co.bound(r["K"], r["S"], r["b"], 0.0, r["ref"], precision, out=out)


def sigmoid64(z):
    z = np.asarray(z, np.float64)
    with np.errstate(over="ignore"):
        return 1.0 / (1.0 + np.exp(-z))


def sigmoid_bound(s):
    """Bound on |1.f / (1.f + expf(-z)) - sigmoid(z)| for the fp32 logit z, s = sigmoid(z) in float64.
    * expf(-z) = e (1 + d1), |d1| <= 2 ulp of the result (CUDA's expf, full range), at most 2 * 2^-23 relative;
    * 1 + e rounds once: (1 + e)(1 + d1 e / (1 + e))(1 + d2), |d2| <= U, and e / (1 + e) < 1;
    * the division rounds once (IEEE, not fast-math): (1 + d3), |d3| <= U.
    So v = s (1 + d), |d| <= 2^-22 + 2 U + O(2^-44): 4 * 2^-23 relative covers it.  Where expf overflows (z < -88.7) or the
    quotient is subnormal (s < 2^-126), v is 0 or within 2^-150 of s, so an absolute 2^-126 is added."""
    return 4 * 2.0 ** -23 * np.abs(s) + 2.0 ** -126
