"""Input builders for the selection-kernel tests (RPN top-k + NMS, box-head post-processing, ROIAlign).

Every builder produces values on which the CUDA kernels and the float32 oracle compute the same bits, so that those tests
can compare index-aligned and bit for bit.  test_selection_inputs_cpu.py checks each exactness claim on the CPU.
"""
from __future__ import annotations

import numpy as np

F32 = np.float32
LO_SCALE = F32(2048.0)       # planes.cuh: x = hi + lo / 2048
SENTINEL = F32(1000.0)       # fp16-exact, far outside the k/256 feature range: marks the padded rows beyond the crop


# ---- RPN -----------------------------------------------------------------------------------------------------------
def rpn_deltas(rng, fh, fw, na=3, step=8, span=8):
    """Box regression [fh, fw, na, 4]: tx, ty in multiples of 1/step within [-span/step, span/step], tw = th = 0.
    The anchors are small half-integers with integer sides, so the decode is exact in float32."""
    t = np.zeros((fh, fw, na, 4), F32)
    t[..., :2] = rng.integers(-span, span + 1, (fh, fw, na, 2)).astype(F32) / F32(step)
    return t


def quantised_logits(rng, n, k):
    """n objectness logits from four values: about k/2 above the k-th value and a few thousand (or a third of the level)
    equal to it, so that the k-th value is tied many times over and the tie order decides the selected set."""
    p_top = min(0.3, 0.5 * (k - 1) / n)
    u = rng.random(n)
    return np.select([u < p_top, u < p_top + 0.35, u < 0.8], [F32(1.5), F32(0.75), F32(0.0)], F32(-0.5)).astype(F32)


def rpn_stage(cls, box):
    """The rpn_l* stage row of one image: [fh, fw, 16] = 3 logits, 3 x (tx, ty, tw, th), one unused column."""
    fh, fw, na = cls.shape
    s = np.zeros((fh, fw, 16), F32)
    s[..., :na] = cls
    s[..., 3:3 + 4 * na] = box.reshape(fh, fw, 4 * na)
    return s


# ---- box head --------------------------------------------------------------------------------------------------------
def head_logits_row(nc, cls, box, ld, class_agnostic=False):
    """One head_logits row: class logits [nc], then box logits ([4] class-agnostic, else [nc, 4] incl. background)."""
    r = np.zeros((ld,), F32)
    r[:nc] = cls
    nb = 4 if class_agnostic else 4 * nc
    r[nc:nc + nb] = np.asarray(box, F32).reshape(-1)
    return r


def iou_threshold_pairs():
    """Two box pairs (x1, y1, x2, y2) far apart: the first overlaps at IoU exactly f32(0.5), the second at the next
    float32 overlap above it (its short side one ulp longer)."""
    y_up = np.nextafter(F32(5.0), F32(10.0))
    return [(np.array([0, 0, 10, 10], F32), np.array([0, 0, 10, 5], F32)),
            (np.array([100, 0, 110, 10], F32), np.array([100, 0, 110, y_up], F32))]


# ---- features --------------------------------------------------------------------------------------------------------
def feature_values(B, H, W, C, salt=0):
    """[B, H, W, C] distinct-looking fp16-exact values k/256, |k| < 2048, that change with every (b, y, x, c)."""
    b, y, x, c = np.meshgrid(np.arange(B), np.arange(H), np.arange(W), np.arange(C), indexing="ij", sparse=True)
    h = (b * 7919 + y * 1031 + x * 131 + c * 37 + salt * 613) % 4093
    return ((h * 2477) % 4093 - 2046).astype(F32) / F32(256.0)


def feature_stage(B, pitch_hw, crop_hw, C, salt=0):
    """A p2..p5 stage [B, pitch_H, pitch_W, C]: feature_values over the cropped extent, SENTINEL in the padded tail."""
    ph, pw = pitch_hw
    h, w = crop_hw
    s = np.full((B, ph, pw, C), SENTINEL, F32)
    s[:, :h, :w] = feature_values(B, h, w, C, salt)
    return s


def planes_value(v):
    """The value an fp16 (hi, lo) plane pair stores for float32 v (planes.cuh split, read back as hi + lo/2048)."""
    v = np.asarray(v, F32)
    hi = v.astype(np.float16)
    lo = ((v - hi.astype(F32)) * LO_SCALE).astype(np.float16)
    return (hi.astype(F32) + lo.astype(F32) / LO_SCALE).astype(F32)


def same_bits(a, b):
    """Bitwise equality of two float32 arrays (distinguishes -0.0 from +0.0, and NaN payloads)."""
    a = np.ascontiguousarray(a, F32)
    b = np.ascontiguousarray(b, F32)
    return a.shape == b.shape and bool(np.array_equal(a.view(np.uint32), b.view(np.uint32)))
