"""ORACLE (test infrastructure only -- never imported by the product path).

CPU restatement of the TensorFlow-1.15 ops the reference's detector graph calls.
TensorFlow (`tensorflow-gpu==1.15`, prose pin README.md:63) is NOT in /root/reference
and NOT installable here, so these follow TF's published op semantics; the reference
pins none of them with tests (SURVEY.md section 4) => **parity unpinned** at this boundary.
Reference call sites are cited per function.  All arithmetic is float32.
"""
from __future__ import annotations

import numpy as np

F32 = np.float32


def top_k(scores: np.ndarray, k: int):
    """tf.nn.top_k(sorted=False) call sites: nn.py:1368, models.py:432,1295.
    TF leaves the order unspecified; the oracle fixes the canonical order
    (score descending, ties -> lower index first), which is what TF's CPU kernel
    produces for sorted=True."""
    scores = np.asarray(scores, dtype=F32)
    k = int(min(k, scores.shape[0]))
    order = np.lexsort((np.arange(scores.shape[0]), -scores.astype(np.float64)))
    idx = order[:k]
    return scores[idx], idx.astype(np.int64)


def iou_tf(a, b) -> F32:
    """IOU() of tensorflow/core/kernels/non_max_suppression_op.cc (TF 1.15), float32.
    Boxes are 4 corner coords; TF canonicalises with min/max so x/y order is free."""
    ymin_i = min(a[0], a[2]); xmin_i = min(a[1], a[3])
    ymax_i = max(a[0], a[2]); xmax_i = max(a[1], a[3])
    ymin_j = min(b[0], b[2]); xmin_j = min(b[1], b[3])
    ymax_j = max(b[0], b[2]); xmax_j = max(b[1], b[3])
    area_i = F32(F32(ymax_i - ymin_i) * F32(xmax_i - xmin_i))
    area_j = F32(F32(ymax_j - ymin_j) * F32(xmax_j - xmin_j))
    if area_i <= 0 or area_j <= 0:
        return F32(0.0)
    iy0 = max(ymin_i, ymin_j); ix0 = max(xmin_i, xmin_j)
    iy1 = min(ymax_i, ymax_j); ix1 = min(xmax_i, xmax_j)
    inter = F32(max(F32(iy1 - iy0), F32(0.0)) * max(F32(ix1 - ix0), F32(0.0)))
    return F32(inter / F32(F32(area_i + area_j) - inter))


def non_max_suppression(boxes, scores, max_output_size, iou_threshold,
                        score_threshold=-np.inf):
    """tf.image.non_max_suppression (V3) -- call sites nn.py:1390-1393, models.py:1211-1213.
    Greedy: candidates by score descending (ties -> lower index); keep a candidate iff its
    IoU with every kept box is <= iou_threshold (suppress on '>').  Returns kept indices in
    selection order."""
    boxes = np.asarray(boxes, dtype=F32).reshape(-1, 4)
    scores = np.asarray(scores, dtype=F32)
    n = boxes.shape[0]
    order = np.lexsort((np.arange(n), -scores.astype(np.float64)))
    thr = F32(iou_threshold)
    keep = []
    # vectorised IoU of one candidate against the kept set, all float32
    ymin = np.minimum(boxes[:, 0], boxes[:, 2]); ymax = np.maximum(boxes[:, 0], boxes[:, 2])
    xmin = np.minimum(boxes[:, 1], boxes[:, 3]); xmax = np.maximum(boxes[:, 1], boxes[:, 3])
    area = ((ymax - ymin).astype(F32) * (xmax - xmin).astype(F32)).astype(F32)
    for i in order:
        if len(keep) >= max_output_size:
            break
        if not (scores[i] > score_threshold):
            continue
        ok = True
        if keep and area[i] > 0:
            k = np.asarray(keep)
            iy = np.maximum((np.minimum(ymax[i], ymax[k]) - np.maximum(ymin[i], ymin[k])).astype(F32), F32(0))
            ix = np.maximum((np.minimum(xmax[i], xmax[k]) - np.maximum(xmin[i], xmin[k])).astype(F32), F32(0))
            inter = (iy * ix).astype(F32)
            union = ((area[i] + area[k]).astype(F32) - inter).astype(F32)
            with np.errstate(divide="ignore", invalid="ignore"):
                iou = np.where(area[k] > 0, (inter / union).astype(F32), F32(0))
            ok = not bool(np.any(iou > thr))
        if ok:
            keep.append(int(i))
    return np.asarray(keep, dtype=np.int64)


def crop_and_resize(image_hwc: np.ndarray, boxes_norm: np.ndarray, crop: int) -> np.ndarray:
    """tf.image.crop_and_resize(method=bilinear, extrapolation_value=0) for one image
    -- call site nn.py:1276-1278.  image [H,W,C], boxes normalised [y1,x1,y2,x2].
    Follows CropAndResize CPU kernel: in = y1*(H-1) + i*(y2-y1)*(H-1)/(crop-1);
    whole row/col is 0 when in < 0 or in > H-1."""
    image_hwc = np.asarray(image_hwc, dtype=F32)
    H, W, C = image_hwc.shape
    n = boxes_norm.shape[0]
    out = np.zeros((n, crop, crop, C), dtype=F32)
    for b in range(n):
        y1, x1, y2, x2 = [F32(v) for v in boxes_norm[b]]
        with np.errstate(invalid="ignore", over="ignore"):
            hs = F32((y2 - y1) * F32(H - 1) / F32(crop - 1)) if crop > 1 else F32(0)
            ws = F32((x2 - x1) * F32(W - 1) / F32(crop - 1)) if crop > 1 else F32(0)
            ys = (F32(y1 * F32(H - 1)) + np.arange(crop, dtype=F32) * hs).astype(F32)
            xs = (F32(x1 * F32(W - 1)) + np.arange(crop, dtype=F32) * ws).astype(F32)
        # A 1-pixel axis samples its only pixel.  Boxes normalised by (H - 1) = 0 give NaN coordinates there, which TF's
        # kernel casts to an index (undefined behaviour); the GPU kernels define the case this way.  A NaN coordinate on a
        # longer axis (an infinite box side) fails both range tests: extrapolation value, like any coordinate outside.
        if H == 1:
            ys = np.zeros(crop, F32)
        if W == 1:
            xs = np.zeros(crop, F32)
        yv = (ys >= 0) & (ys <= F32(H - 1))
        xv = (xs >= 0) & (xs <= F32(W - 1))
        yc = np.clip(np.where(yv, ys, F32(0)), 0, H - 1); xc = np.clip(np.where(xv, xs, F32(0)), 0, W - 1)
        t = np.floor(yc).astype(np.int64); bt = np.ceil(yc).astype(np.int64)
        l = np.floor(xc).astype(np.int64); r = np.ceil(xc).astype(np.int64)
        yl = (yc - t.astype(F32)).astype(F32)[:, None, None]
        xl = (xc - l.astype(F32)).astype(F32)[None, :, None]
        tl = image_hwc[t][:, l]; tr = image_hwc[t][:, r]
        bl = image_hwc[bt][:, l]; br = image_hwc[bt][:, r]
        top = (tl + (tr - tl) * xl).astype(F32)
        bot = (bl + (br - bl) * xl).astype(F32)
        val = (top + (bot - top) * yl).astype(F32)
        val[~yv] = 0
        val[:, ~xv] = 0
        out[b] = val
    return out
