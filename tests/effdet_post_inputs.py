"""Input builders for the EfficientDet post-processing tests (global top-k, sigmoid + decode, NMS: effdet.cu; own-level
box features: roialign.cu).

Every builder produces values on which the CUDA kernels and the float32 oracle (oracle.effdet) compute the same bits, so
that test_effdet_post_gpu.py can compare index-aligned and bit for bit.  test_effdet_post_inputs_cpu.py checks each
exactness claim on the CPU.
"""
from __future__ import annotations

import numpy as np

import selection_inputs as si

F32 = np.float32
SENTINEL = F32(1e30)          # in the padding columns of the head rows: above every real logit, so never selectable
rpn_deltas = si.rpn_deltas    # exact deltas: ty, tx multiples of 1/8, th = tw = 0
feature_values = si.feature_values
same_bits = si.same_bits


def pad16(c):
    return (c + 15) // 16 * 16


def pad64(c):
    return (c + 63) // 64 * 64


def num_anchors(cfg):
    return cfg.num_scales * len(cfg.aspect_ratios)


def level_sizes(cfg):
    """{level: (h, w)} for levels 3..7."""
    from object_detection_tracking_b200.effdet_config import feat_sizes
    fs = feat_sizes(cfg)
    return {l: fs[l] for l in range(3, 8)}


def level_offsets(cfg):
    """Flat logit index of the first logit of every level, and the total: {level: offset}, total."""
    na, nc = num_anchors(cfg), cfg.num_classes
    off, out = 0, {}
    for l, (h, w) in level_sizes(cfg).items():
        out[l] = off
        off += h * w * na * nc
    return out, off


def padded(x, ld, fill=SENTINEL):
    """A head output [h, w, c] as its stage row [h, w, ld]: the padding columns hold `fill`."""
    h, w, c = x.shape
    s = np.full((h, w, ld), fill, F32)
    s[..., :c] = x
    return s


def split_levels(cfg, flat, width):
    """A flat array over all levels (level-major, then y, x, column) -> {level: [h, w, width]}."""
    out, o = {}, 0
    for l, (h, w) in level_sizes(cfg).items():
        out[l] = np.asarray(flat[o:o + h * w * width], F32).reshape(h, w, width)
        o += h * w * width
    return out


def exact_deltas(cfg, rng):
    """{level: [h, w, A*4]} box regressions of rpn_deltas (ty, tx multiples of 1/8, th = tw = 0)."""
    na = num_anchors(cfg)
    return {l: rpn_deltas(rng, h, w, na).reshape(h, w, na * 4) for l, (h, w) in level_sizes(cfg).items()}


# ---- logits --------------------------------------------------------------------------------------------------------
def band_logits(rng, n, k, ties=3.0):
    """n logits from four values: about k/2 at 1.5, about ties*k at 0.75 (the k-th value, spread uniformly over the flat
    index range, so every radix block holds some when n / 1056 << n / (ties*k)), the rest at 0 or -0.5."""
    u = rng.random(n)
    p_top, p_tie = 0.5 * k / n, ties * k / n
    return np.select([u < p_top, u < p_top + p_tie, u < 0.5 + p_top + p_tie], [F32(1.5), F32(0.75), F32(0.0)],
                     F32(-0.5)).astype(F32)


def key_of(x):
    """effdet.cu float_key: the order-preserving uint32 key of float32 x (+0.0 and -0.0 share one key)."""
    u = np.ascontiguousarray(x, F32).view(np.uint32).copy()
    u[np.asarray(x, F32) == 0] = 0
    return np.where(u & 0x80000000, ~u, u | 0x80000000).astype(np.uint32)


def float_of_key(key):
    """The float32 whose key is `key` (the positive zero for the zero key)."""
    key = np.asarray(key, np.uint32)
    u = np.where(key & 0x80000000, key & 0x7FFFFFFF, ~key).astype(np.uint32)
    return u.view(F32)


def prefix_logits(rng, n, value, bits):
    """n distinct-ish logits whose keys agree with key_of(value) in their top `bits` bits (the radix passes before the
    last see one bucket): the low 32 - bits key bits are random.  NaN keys cannot occur for finite `value` of small
    magnitude."""
    base = int(key_of(np.array([value], F32))[0])
    low = (1 << (32 - bits)) - 1
    keys = (base & ~low & 0xFFFFFFFF) | rng.integers(0, low + 1, n, dtype=np.int64)
    return float_of_key(keys.astype(np.uint32))


def signed_zero_logits(rng, n, n_above):
    """n logits: n_above positive ones, the rest +0.0 and -0.0 interleaved at random (all tied at the k-th value)."""
    x = np.where(rng.random(n) < 0.5, F32(0.0), F32(-0.0)).astype(F32)
    x[rng.choice(n, n_above, replace=False)] = rng.integers(1, 64, n_above).astype(F32) / F32(8)
    return x


# ---- exact top-k for large inputs ------------------------------------------------------------------------------------
def fast_top_k(x, k):
    """tf_ops.top_k's result (values descending, ties -> lower index) by argpartition: the values above the k-th one,
    plus the lowest-index ties, then sorted.  Exact for every input without NaN (+0.0 and -0.0 compare equal in both)."""
    x = np.asarray(x, F32)
    n = x.shape[0]
    k = int(min(k, n))
    kth = np.partition(x, n - k)[n - k]
    gt = np.flatnonzero(x > kth)
    eq = np.flatnonzero(x == kth)[:k - len(gt)]
    idx = np.concatenate([gt, eq])
    idx = idx[np.lexsort((idx, -x[idx].astype(np.float64)))]
    return x[idx], idx.astype(np.int64)


# ---- NMS threshold pairs ---------------------------------------------------------------------------------------------
IOU_ABOVE = np.nextafter(F32(0.5), F32(1))   # one float32 ulp above the 0.5 NMS threshold


def iou_shift(anchor_a, anchor_b, target, span=48):
    """(ty, tx) for anchor_b (th = tw = 0; anchor_a undecoded) such that the float32 IoU of the two decoded boxes is
    exactly `target`, for same-size anchors side by side: (0, 0) when the anchors already overlap at `target`, else the
    first hit of a grid of small shifts around the analytic tx (fine steps in both axes, so that the rounded box corners
    reach every float32 IoU near it); None when no candidate lands on it."""
    from oracle import effdet as oe
    from oracle import tf_ops
    a = np.asarray(anchor_a, F32)
    b = np.asarray(anchor_b, F32)
    w = float(a[3] - a[1])
    t0 = ((1 - float(target)) / (1 + float(target)) * w - float(b[1] - a[1])) / w
    step = 2.0 ** -26
    ty, tx = np.meshgrid(np.arange(0, span + 1) * step, t0 + np.arange(-span, span + 1) * step, indexing="ij")
    rel = np.zeros((ty.size, 4), F32)
    rel[:, 0], rel[:, 1] = ty.ravel(), tx.ravel()
    rel = np.concatenate([np.zeros((1, 4), F32), rel])
    bb = oe.decode_boxes(rel, np.repeat(b[None], len(rel), 0))
    for r, box in zip(rel, bb):
        if tf_ops.iou_tf(a, box) == F32(target):
            return F32(r[0]), F32(r[1])
    return None


# ---- box features ----------------------------------------------------------------------------------------------------
def sample_coords(c0, c1, dim, crop=14):
    """roialign.cu make_axis / oracle.frcnn.roi_align + tf_ops.crop_and_resize along one axis: the crop sample
    coordinates of the feature-map box side [c0, c1] on an axis of `dim` pixels, float32 op by op."""
    if dim == 1:
        return np.zeros(crop, F32)
    c0, c1, dm1 = F32(c0), F32(c1), F32(dim - 1)
    with np.errstate(invalid="ignore", over="ignore"):
        sp = F32(F32(c1 - c0) / F32(crop))
        n0 = F32(F32(F32(c0 + F32(sp / F32(2))) - F32(0.5)) / dm1)
        nlen = F32(F32(sp * F32(crop - 1)) / dm1)
        n1 = F32(n0 + nlen)
        scale = F32(F32(F32(n1 - n0) * dm1) / F32(crop - 1))
        return (F32(n0 * dm1) + np.arange(crop, dtype=F32) * scale).astype(F32)


def quarter_exact(c0, c1, dim):
    """Every sample coordinate inside the axis is a multiple of 1/4: the bilinear weights are then 0, 1/4, 1/2, 3/4, so
    with feature_values (k/256, |k| < 2048) every sample, 2x2 average and the 49-bin sum is exact in float32."""
    s = sample_coords(c0, c1, dim)
    inside = (s >= 0) & (s <= dim - 1)
    return bool(np.all(np.asarray(s[inside] * 4, np.float64) == np.round(np.asarray(s[inside] * 4, np.float64))))


def exact_feature_boxes(rng, sizes, n, lo=-0.5, hi=1.5):
    """n boxes (x1, y1, x2, y2) in network pixels with their levels, whose sample coordinates are all quarter_exact on
    the box's level: corners multiples of 1/8 feature pixel, spanning from `lo` to `hi` times the level's extent (so some
    lie partly or wholly outside it).  sizes: {level: (h, w)}."""
    boxes, levels = [], []
    lv = sorted(sizes)
    while len(boxes) < n:
        l = lv[len(boxes) % len(lv)]
        h, w = sizes[l]
        cand = []
        for dim in (w, h):
            a, b = np.sort(rng.integers(int(lo * 8 * dim), int(hi * 8 * dim) + 1, 2)) / 8.0
            cand.append((a, b + 1.75))
        (x0, x1), (y0, y1) = cand
        if quarter_exact(x0, x1, w) and quarter_exact(y0, y1, h):
            boxes.append(np.array([x0, y0, x1, y1], F32) * F32(2.0 ** l))
            levels.append(l)
    return np.asarray(boxes, F32), np.asarray(levels, np.int32)
