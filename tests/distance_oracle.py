"""Float64 reference of the appearance-distance entry points, a float32 restatement of their epilogue kernels, and an
element-wise error bound for the tensor-core results.

References, each with the NaN and eps semantics of the code it restates:
  * nn_cosine / nn_euclidean: deep_sort/nn_matching.py _nn_cosine_distance and _nn_euclidean_distance (rows divided by
    their norm without an eps; np.min, np.clip and np.maximum keep NaN);
  * cosine_matrix(eps=1e-12) / sq_euclidean: torchreid/distance.py (F.normalize clamps the norm at 1e-12; the squared
    euclidean distance is not clamped);
  * feature_dist: multi_video_reid.py compute_feature_dist (min over two tracks' crops of sklearn's squared
    euclidean_distances, which clamps at 0), gated, with the kernel's `fill` for ungated pairs and empty tracks;
  * jde_cdist: tmot/matching.py embedding_distance, np.maximum(0, scipy cdist).
The *_f32 functions restate distance_finish, cosine_segmin and pair_segmin (csrc/cosine.cu) op for op in IEEE float32, so
a kernel result must equal them exactly (NaN where they are NaN).
"""
from __future__ import annotations

import numpy as np
from scipy.spatial.distance import cdist

import conv_oracle as co

U = 2.0 ** -24
EMPTY_SEGMENT = np.float32(3.4e38)   # cosine_segmin's value for a track without gallery rows
FP16_INF_FROM = 65520.0              # the smallest |x| that rounds to an fp16 inf
TORCHREID_EPS = 1e-12
PLANE = {"split": (2.0 ** -22, 2.0 ** -36), "fp16": (2.0 ** -11, 2.0 ** -25)}   # (relative, absolute) storage error


# ---- float64 references ------------------------------------------------------------------------------------------
def _f64(x):
    return np.asarray(x, np.float64)


def dot(a, b):
    """a @ b.T in float64 with IEEE semantics for non-finite inputs (inf * 0 = NaN, inf - inf = NaN)."""
    a, b = _f64(a), _f64(b)
    if np.isfinite(a).all() and np.isfinite(b).all():
        return a @ b.T
    with np.errstate(invalid="ignore", over="ignore"):
        return np.einsum("ik,jk->ij", a, b)


def normalize(x, eps=0.0):
    """x / max(|x|, eps) per row: eps 0 is nn_matching's division (0/0 = NaN), 1e-12 F.normalize's clamp."""
    x = _f64(x)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        n = np.sqrt((x * x).sum(axis=1, keepdims=True))
        n = np.where(n < eps, eps, n)    # a NaN norm stays NaN, as torch's clamp_min
        return x / n


def cosine_matrix(a, b, eps=0.0):
    with np.errstate(invalid="ignore"):
        return 1.0 - dot(normalize(a, eps), normalize(b, eps))


def sq_euclidean(a, b):
    a, b = _f64(a), _f64(b)
    with np.errstate(invalid="ignore", over="ignore"):
        return (a * a).sum(1)[:, None] + (b * b).sum(1)[None, :] - 2.0 * dot(a, b)


def seg_reduce(x, seg, axis, ufunc, empty):
    """ufunc.reduce of x over the segments [seg[i], seg[i+1]) along `axis`; `empty` for an empty segment.  NaN
    propagates through np.minimum / np.maximum."""
    x = np.moveaxis(np.asarray(x), axis, 0)
    seg = np.asarray(seg, np.int64)
    out = np.full((len(seg) - 1,) + x.shape[1:], empty, dtype=x.dtype)
    live = np.flatnonzero(seg[1:] > seg[:-1])
    if live.size:
        out[live] = ufunc.reduceat(x, seg[:-1][live], axis=0)
    return np.moveaxis(out, 0, axis)


def nn_cosine(gallery, seg, dets):
    """[T, N]: min over each track's gallery rows of the cosine distance (empty track: EMPTY_SEGMENT)."""
    return seg_reduce(cosine_matrix(gallery, dets, 0.0), seg, 0, np.minimum, float(EMPTY_SEGMENT))


def nn_euclidean(gallery, seg, dets):
    with np.errstate(invalid="ignore"):
        d = np.clip(sq_euclidean(gallery, dets), 0.0, np.inf)
    return np.maximum(0.0, seg_reduce(d, seg, 0, np.minimum, np.inf))


def feature_dist(a, seg_a, b, seg_b, gate=None, fill=999.0):
    """[N, M]: min over the two tracks' crops of max(0, squared distance) where gate != 0, else fill; fill for a track
    without crops."""
    with np.errstate(invalid="ignore"):
        d = np.maximum(sq_euclidean(a, b), 0.0)
    m = seg_reduce(seg_reduce(d, seg_a, 0, np.minimum, np.inf), seg_b, 1, np.minimum, np.inf)
    empty = (np.diff(seg_a) == 0)[:, None] | (np.diff(seg_b) == 0)[None, :]
    if gate is not None:
        empty |= np.asarray(gate) == 0
    return np.where(empty, fill, m)


def jde_cdist(a, b):
    with np.errstate(invalid="ignore"):
        return np.maximum(0.0, cdist(_f64(a), _f64(b)))


# ---- float32 restatements of the epilogue kernels -----------------------------------------------------------------
def finish_f32(dots, metric, na2=None, nb2=None):
    """distance_finish: 1 - d, or (na2[i] + nb2[j]) - 2 d, each op rounded to float32."""
    d = np.asarray(dots, np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        if metric == 0:
            return np.float32(1.0) - d
        s = np.asarray(na2, np.float32)[:, None] + np.asarray(nb2, np.float32)[None, :]
        return s - np.float32(2.0) * d


def cosine_segmin_f32(dots, seg):
    return seg_reduce(finish_f32(dots, 0), seg, 0, np.minimum, EMPTY_SEGMENT)


def pair_segmin_f32(dots, na2, nb2, seg_a, seg_b, gate=None, fill=0.0):
    d = np.maximum(finish_f32(dots, 1, na2, nb2), np.float32(0.0))
    m = seg_reduce(seg_reduce(d, seg_a, 0, np.minimum, np.float32(np.inf)), seg_b, 1, np.minimum, np.float32(np.inf))
    empty = (np.diff(seg_a) == 0)[:, None] | (np.diff(seg_b) == 0)[None, :]
    if gate is not None:
        empty |= np.asarray(gate) == 0
    return np.where(empty, np.float32(fill), m).astype(np.float32)


def planes_raw(x, ld=None):
    """rows_to_planes' planes of x [rows, D] as raw uint16 [rows, ld], columns >= D zero."""
    x = np.asarray(x, np.float32)
    ld = x.shape[1] if ld is None else ld
    pad = np.zeros((x.shape[0], ld), np.float32)
    pad[:, :x.shape[1]] = x
    hi, lo = co.split_planes(pad)
    return hi.view(np.uint16), lo.view(np.uint16)


def out_of_range(x):
    """rows_to_planes' range flag: a finite component that rounds to an fp16 inf."""
    x = np.abs(np.asarray(x, np.float32))
    return bool((np.isfinite(x) & (x >= FP16_INF_FROM)).any())


# ---- error bounds ---------------------------------------------------------------------------------------------
def sum_bound(n):
    """Relative bound of a per-warp sum of squares (csrc/cosine.cu): each lane an fmaf chain of ceil(n / 32) terms,
    then five shuffle adds -- one rounding of at most U of the running sum per step, second order included."""
    return (-(-n // 32) + 5) * U * 1.01


def norm_rel(D):
    """Relative error of a row divided by its fp32 norm: half the sum's error through sqrtf, sqrtf's and the division's
    own rounding."""
    return sum_bound(D) / 2 + 2 * U * 1.01


def _finite_rows(x):
    return np.isfinite(_f64(x)).all(axis=1)


def _dot_error(a, b, rel_a, rel_b, precision, Dp):
    """|GEMM(a~, b~) - a.b| where a~, b~ are a and b with a relative error rel_a, rel_b and then stored as planes of
    `precision`; the GEMM's own arithmetic is conv_oracle.bound over K = Dp.  Also returns S = sum_k |a_k b_k|."""
    prel, pabs = PLANE[precision]
    ra, rb = rel_a + prel * (1 + rel_a), rel_b + prel * (1 + rel_b)
    A, B = np.abs(np.nan_to_num(_f64(a), nan=0.0, posinf=0.0, neginf=0.0)), np.abs(
        np.nan_to_num(_f64(b), nan=0.0, posinf=0.0, neginf=0.0))
    S = A @ B.T
    D = A.shape[1]
    rep = (ra + rb + ra * rb) * S + pabs * (1 + max(ra, rb)) * (A.sum(1)[:, None] + B.sum(1)[None, :]) + D * pabs * pabs
    S_t = S * (1 + ra) * (1 + rb) + rep
    gemm = co.bound(Dp, S_t, 0.0, 0.0, S_t, precision=precision, out="f32")
    return rep + gemm, S


def cosine_bound(a, b, eps, precision):
    """Per-element bound on |kernel 1 - a^.b^ - float64 cosine distance| for finite rows."""
    D = _f64(a).shape[1]
    Dp = -(-D // 64) * 64
    e, _ = _dot_error(normalize(a, eps), normalize(b, eps), norm_rel(D), norm_rel(D), precision, Dp)
    with np.errstate(invalid="ignore"):
        ref = np.abs(cosine_matrix(a, b, eps))
    return e + U * (np.nan_to_num(ref, nan=0.0) + e + 2.0)


def euclidean_bound(a, b, precision):
    """Per-element bound on |kernel (|a|^2 + |b|^2) - 2 a.b - float64 squared distance| for finite rows: the operands'
    planes and the GEMM, the fp32 row norms and the final add and subtract."""
    a, b = _f64(a), _f64(b)
    D = a.shape[1]
    Dp = -(-D // 64) * 64
    e, S = _dot_error(a, b, 0.0, 0.0, precision, Dp)
    with np.errstate(invalid="ignore", over="ignore"):
        a2 = np.nan_to_num((a * a).sum(1), nan=0.0, posinf=0.0)[:, None]
        b2 = np.nan_to_num((b * b).sum(1), nan=0.0, posinf=0.0)[None, :]
    g = sum_bound(Dp)
    e = 2 * e + g * (a2 + b2)
    return e + U * (1 + g) * (a2 + b2) + U * (a2 + b2 + 2 * S + 2 * e)
