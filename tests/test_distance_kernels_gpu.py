"""The appearance-distance kernels (csrc/cosine.cu) and the entry points built on them -- b2_cosine_cost,
b2_distance_matrix, b2_track_pair_cost(_dev), b2_tmot_embedding_distance -- against the float64 references of
tests/distance_oracle.py, in split and fp16 precision.

Shapes: D around the GEMM's 64-deep K blocks and the widths real features have (EfficientDet's fpn_num_filters, OSNet's
512, ResNet-101's 2048); gallery rows around the 128-row padding, detections around the 16-column padding and past
several N tiles; segments of length 0, 1 and the budget's 100.  Values: zero rows, rows of norm below 1e-12, exact
duplicates (distance ~0, all cancellation), NaN and +-inf components, components at 65504, 65519 and 65520, ties.

Three kinds of check:
  * bit-exact: the epilogue kernels (distance_finish, cosine_segmin, pair_segmin) are single IEEE fp32 ops and must
    equal the float32 restatement exactly, NaN where it is NaN; rows_to_planes' planes are the split of each input;
  * error-bounded: each finite result within the per-element bound of distance_oracle (it scales with sum_k |a_k b_k|
    and, for squared distances, with |a|^2 + |b|^2), which the fp16-precision result must break on a generic case;
  * non-finite: a result is NaN exactly where the float64 reference is NaN and finite where it is finite.
"""
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

import distance_oracle as do

pytestmark = pytest.mark.gpu

PRECISIONS = ["split", "fp16"]
DS = [1, 7, 33, 63, 64, 65, 88, 112, 160, 224, 288, 384, 512, 2048]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _engine():
    from object_detection_tracking_b200 import engine
    return engine


def _lib():
    from object_detection_tracking_b200 import _lib
    return _lib


def cosine_cost(g, seg, dets, precision):
    return _engine().cosine_cost(g, seg, dets, precision=precision)


def distance_matrix(a, b, metric, precision):
    from object_detection_tracking_b200.reid import compute_distance_matrix
    return compute_distance_matrix(a, b, metric, precision=precision).numpy()


def pair_cost(a, seg_a, b, seg_b, precision, gate=None, fill=999.0):
    lib = _lib()
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    sa, sb = np.ascontiguousarray(seg_a, np.int32), np.ascontiguousarray(seg_b, np.int32)
    g = None if gate is None else np.ascontiguousarray(gate, np.uint8)
    out = np.empty((len(sa) - 1, len(sb) - 1), np.float32)
    lib.check(lib.load().b2_track_pair_cost(0, lib.ptr(a), lib.ptr(sa), len(sa) - 1, lib.ptr(b), lib.ptr(sb), len(sb) - 1,
                                            a.shape[1], lib.ptr(g), float(fill), {"fp16": 0, "split": 1}[precision],
                                            lib.ptr(out)), "b2_track_pair_cost")
    return out


def jde_distance(a, b, precision):
    from object_detection_tracking_b200.tmot import embedding_distance
    return embedding_distance(a, b, precision=precision)


def rows(rng, n, D, specials=()):
    """n Gaussian rows with special rows at the given (index, kind) places."""
    x = rng.standard_normal((n, D)).astype(np.float32)
    for i, kind in specials:
        if not 0 <= i < n:
            continue
        if kind == "zero":
            x[i] = 0.0
        elif kind == "tiny":                       # norm 1e-13, below F.normalize's eps
            x[i] = x[i] / np.linalg.norm(x[i]) * np.float32(1e-13)
        elif kind == "nan":
            x[i, (7 * i) % D] = np.nan
        elif kind == "big":                        # the largest components the fp16 hi plane holds finite
            x[i, 0] = 65504.0
            x[i, -1] = -65519.0
        elif kind == "dup":                        # a copy of row 0
            x[i] = x[0]
    return x


def check(got, ref, bnd, what):
    """NaN exactly where ref is NaN, finite where ref is finite, and within bnd there."""
    got = np.asarray(got, np.float64)
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    nan_got, nan_ref = np.isnan(got), np.isnan(ref)
    if (nan_got != nan_ref).any():
        i = tuple(np.argwhere(nan_got != nan_ref)[0])
        raise AssertionError("%s: NaN pattern differs at %s: got %r, reference %r" % (what, i, got[i], ref[i]))
    fin = np.isfinite(ref)
    assert np.isfinite(got[fin]).all(), "%s: non-finite result where the reference is finite" % what
    err = np.where(fin, np.abs(got - np.where(fin, ref, 0.0)), 0.0)
    bnd = np.broadcast_to(bnd, ref.shape)
    ok = ~fin | (err <= bnd)
    if not ok.all():
        i = tuple(np.argwhere(~ok)[0])
        raise AssertionError("%s: element %s |err| %.3g > bound %.3g (ref %.9g, got %.9g)" % (what, i, err[i], bnd[i],
                                                                                            ref[i], got[i]))


def same_values(got, exp, what):
    """Equal values, NaN where exp is NaN (+0 and -0 compare equal)."""
    got, exp = np.asarray(got), np.asarray(exp)
    assert got.shape == exp.shape, (what, got.shape, exp.shape)
    bad = (np.isnan(got) != np.isnan(exp)) | (~np.isnan(exp) & (got != exp))
    if bad.any():
        i = tuple(np.argwhere(bad)[0])
        raise AssertionError("%s: %d elements differ, first %s: got %r expected %r" % (what, bad.sum(), i, got[i], exp[i]))


def seg_of(lengths):
    return np.concatenate([[0], np.cumsum(lengths)]).astype(np.int32)


def block_max(e, seg_a, seg_b=None):
    """Bound of a minimum over segments: the largest element bound of the segment (min is 1-Lipschitz)."""
    r = do.seg_reduce(e, seg_a, 0, np.maximum, 0.0)
    return r if seg_b is None else do.seg_reduce(r, seg_b, 1, np.maximum, 0.0)


# ---- operand conversion ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", DS)
def test_rows_to_planes_are_the_split_of_each_input(D):
    rng = np.random.default_rng(D)
    x = rows(rng, 40, D, [(1, "zero"), (2, "tiny"), (3, "nan"), (4, "big"), (5, "dup")])
    x[6, 0], x[7, D - 1] = np.inf, -np.inf
    x[8] *= 1e-6                                   # fp16 subnormal hi, lo planes
    for ld in (D, -(-D // 64) * 64, -(-D // 64) * 64 + 64):
        hi, lo, sq, flag = _engine().op_distance_operand(x, ld=ld)
        eh, el = do.planes_raw(x, ld)
        same_values(hi.view(np.float16), eh.view(np.float16), "hi D=%d ld=%d" % (D, ld))
        same_values(lo.view(np.float16), el.view(np.float16), "lo D=%d ld=%d" % (D, ld))
        assert flag == 0
        x64 = x.astype(np.float64)
        with np.errstate(invalid="ignore", over="ignore"):
            ref = (x64 * x64).sum(1)
        check(sq, ref, do.sum_bound(ld) * np.nan_to_num(ref, posinf=0.0), "sqnorm D=%d ld=%d" % (D, ld))
        assert np.isposinf(sq[6]) and np.isposinf(sq[7])


@pytest.mark.parametrize("value", [65520.0, -65520.0, 70000.0, -3.0e38])
def test_rows_to_planes_flags_finite_values_beyond_fp16(value):
    rng = np.random.default_rng(1)
    x = rows(rng, 33, 65, [(4, "big")])
    x[5, 0], x[6, 1] = np.nan, np.inf             # non-finite values are not range errors
    assert _engine().op_distance_operand(x)[3] == 0
    x[31, 64] = value
    hi, lo, _, flag = _engine().op_distance_operand(x, ld=128)
    assert flag == 1 and do.out_of_range(x)
    assert np.isinf(hi[31, 64].view(np.float16))


@pytest.mark.parametrize("eps", [0.0, 1e-12])
@pytest.mark.parametrize("D", DS)
def test_normalized_rows_within_bound_and_eps_semantics(D, eps):
    rng = np.random.default_rng(100 + D)
    x = rows(rng, 37, D, [(1, "zero"), (2, "tiny"), (3, "nan"), (4, "big"), (5, "dup")])
    x[6, 0] = np.inf
    ld = -(-D // 64) * 64
    hi, lo, sq, flag = _engine().op_distance_operand(x, ld=ld, normalize=True, eps=eps)
    assert sq is None and flag is None
    got = hi.view(np.float16).astype(np.float64) + lo.view(np.float16).astype(np.float64) / 2048.0
    ref = np.zeros((len(x), ld))
    ref[:, :D] = do.normalize(x, eps)
    bnd = (do.norm_rel(D) + 2.0 ** -22) * np.abs(np.nan_to_num(ref)) + 2.0 ** -36
    check(got, ref, bnd, "normalized D=%d eps=%g" % (D, eps))
    if eps == 0.0:
        assert np.isnan(got[1, :D]).all()          # 0 / 0, as nn_matching
    else:
        assert (got[1] == 0).all()                 # 0 / 1e-12, as F.normalize
        assert np.linalg.norm(got[2]) == pytest.approx(0.1, rel=1e-5)
    assert (got[:, D:][np.isfinite(ref[:, D:])] == 0).all()


# ---- epilogues, bit-exact ------------------------------------------------------------------------------------------
def special_dots(rng, rows_, ld, cols):
    """Products with NaN, +-inf, -0.0, values that cancel against 1 or the norms, and garbage (NaN) past `cols`."""
    d = rng.uniform(-1.5, 1.5, (rows_, ld)).astype(np.float32)
    flat = d[:, :cols].reshape(-1)
    idx = rng.permutation(flat.size)
    k = max(1, flat.size // 40)
    flat[idx[:k]] = np.nan
    flat[idx[k:2 * k]] = np.inf
    flat[idx[2 * k:3 * k]] = -np.inf
    flat[idx[3 * k:4 * k]] = -0.0
    flat[idx[4 * k:5 * k]] = 1.0
    flat[idx[5 * k:6 * k]] = np.float32(1.0) - np.float32(2.0 ** -24)
    d[:, :cols] = flat.reshape(rows_, cols)
    d[:, cols:] = np.nan
    return d


@pytest.mark.parametrize("cols", [1, 15, 16, 17, 600])
def test_distance_finish_is_bit_exact(cols):
    rng = np.random.default_rng(cols)
    for rows_ in (1, 127, 129):
        ld = cols + 16
        d = special_dots(rng, rows_, ld, cols)
        na2 = np.abs(rng.standard_normal(rows_)).astype(np.float32)
        nb2 = np.abs(rng.standard_normal(cols)).astype(np.float32)
        na2[0], nb2[-1] = np.nan, np.inf
        na2[rows_ // 2] = 0.75                     # (na2 + nb2) - 2 d cancels to 0 against d = 0.5 ...
        nb2[0] = 0.25
        d[rows_ // 2, 0] = 0.5
        got = _engine().op_distance_epilogue("cosine", d, cols=cols)
        same_values(got, do.finish_f32(d[:, :cols], 0), "1 - d rows=%d cols=%d" % (rows_, cols))
        got = _engine().op_distance_epilogue("euclidean", d, cols=cols, na2=na2, nb2=nb2)
        exp = do.finish_f32(d[:, :cols], 1, na2, nb2)
        same_values(got, exp, "a2 + b2 - 2d rows=%d cols=%d" % (rows_, cols))
        if rows_ > 1:
            assert exp[rows_ // 2, 0] == 0.0 and got[rows_ // 2, 0] == 0.0


@pytest.mark.parametrize("cols", [1, 15, 16, 17, 600])
def test_cosine_segmin_is_bit_exact_and_keeps_nan(cols):
    rng = np.random.default_rng(200 + cols)
    lengths = [1, 0, 100, 3, 0, 1, 24]
    seg = seg_of(lengths)
    n = int(seg[-1])
    d = rng.uniform(-1, 1, (n, cols + 5)).astype(np.float32)
    d[:, cols:] = np.nan                           # padding columns are never read
    d[seg[2] + 7, 0] = np.nan                      # one NaN row entry in the 100-row segment
    d[seg[3]:seg[4], :] = 0.25                     # equal minima across a segment's rows
    d[seg[6] + 3, cols - 1] = np.inf               # 1 - inf = -inf is a valid minimum
    d[seg[6] + 4, cols // 2] = -np.inf             # 1 + inf = inf never wins
    got = _engine().op_distance_epilogue("cosine_segmin", d, cols=cols, seg_a=seg)
    exp = do.cosine_segmin_f32(d[:, :cols], seg)
    same_values(got, exp, "cosine_segmin cols=%d" % cols)
    assert np.isnan(got[2, 0]) and (got[1] == do.EMPTY_SEGMENT).all() and (got[4] == do.EMPTY_SEGMENT).all()
    assert (got[3] == 0.75).all() and got[6, cols - 1] == -np.inf


@pytest.mark.parametrize("n_cols", [1, 15, 16, 17, 600])
def test_pair_segmin_is_bit_exact_keeps_nan_and_gates(n_cols):
    rng = np.random.default_rng(300 + n_cols)
    seg_a = seg_of([1, 0, 100, 2, 33])
    lb = [1] if n_cols == 1 else [1, 0, n_cols - 1] if n_cols < 110 else [1, 0, 100] + [1] * (n_cols - 101)
    seg_b = seg_of(lb)
    R, C = int(seg_a[-1]), int(seg_b[-1])
    assert C == n_cols
    d = rng.uniform(-1, 1, (R, C + 3)).astype(np.float32)
    d[:, C:] = np.nan                              # padding columns are never read
    na2 = np.abs(rng.standard_normal(R)).astype(np.float32) + 2.0
    nb2 = np.abs(rng.standard_normal(C)).astype(np.float32) + 2.0
    N, M = len(seg_a) - 1, len(seg_b) - 1
    d[seg_a[2] + 50, seg_b[M - 1]] = np.nan        # a NaN inside a 100-row block
    d[seg_a[3]:seg_a[4], :] = 10.0                 # negative squared distances clamp to 0: ties at 0
    na2[seg_a[4] + 5] = np.nan                     # a NaN row norm
    gate = (rng.uniform(size=(N, M)) < 0.7).astype(np.uint8)
    gate[2, M - 1] = gate[3, M - 1] = gate[4, M - 1] = 1
    for g, fill in ((None, 999.0), (gate, -7.0)):
        got = _engine().op_distance_epilogue("pair_segmin", d, cols=C, na2=na2, nb2=nb2, seg_a=seg_a, seg_b=seg_b,
                                             gate=g, fill=fill)
        exp = do.pair_segmin_f32(d[:, :C], na2, nb2, seg_a, seg_b, g, fill)
        same_values(got, exp, "pair_segmin cols=%d gate=%s" % (n_cols, g is not None))
        assert np.isnan(got[2, M - 1]) and (got[1] == fill).all() and got[3, M - 1] == 0.0
        assert np.isnan(got[4, M - 1])


def test_epilogue_refuses_offsets_outside_the_products():
    d = np.zeros((4, 8), np.float32)
    with pytest.raises(RuntimeError, match="seg_a"):
        _engine().op_distance_epilogue("cosine_segmin", d, seg_a=[0, 5])
    with pytest.raises(RuntimeError, match="seg_b"):
        _engine().op_distance_epilogue("pair_segmin", d, na2=np.zeros(4), nb2=np.zeros(8), seg_a=[0, 4],
                                       seg_b=[0, 3, 2])


# ---- entry points against float64 ----------------------------------------------------------------------------------
SHAPES = [(1, 1), (127, 15), (128, 16), (129, 17)]


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("D", DS)
def test_cosine_cost_within_bound(D, precision):
    """b2_cosine_cost = DeepSORT's _nn_cosine_distance per track: tiny-norm rows and duplicates within the bound, and a
    NaN row makes its track's (or detection's) costs NaN."""
    rng = np.random.default_rng(400 + D)
    for S, N in SHAPES:
        lengths = [1] if S == 1 else [1, 0, 100, S - 101]
        seg = seg_of(lengths)
        g = rows(rng, S, D, [(S - 1, "tiny"), (S - 2, "dup"), (S - 3, "big")])
        dets = rows(rng, N, D, [(N - 1, "dup"), (N - 2, "tiny")])
        dets[0] = g[0] if N > 3 else dets[0]
        got = cosine_cost(g, seg, dets, precision)
        ref = do.nn_cosine(g, seg, dets)
        bnd = block_max(do.cosine_bound(g, dets, 0.0, precision), seg)
        check(got, ref, bnd, "cosine_cost D=%d S=%d N=%d %s" % (D, S, N, precision))
        if S > 1:
            assert (got[1] == do.EMPTY_SEGMENT).all()


@pytest.mark.parametrize("metric", ["cosine", "euclidean"])
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("D", DS)
def test_distance_matrix_within_bound(D, precision, metric):
    rng = np.random.default_rng(500 + D)
    for na, nb in SHAPES + [(33, 600)]:
        a = rows(rng, na, D, [(na - 1, "tiny"), (na - 2, "zero"), (na - 3, "big"), (na - 4, "dup")])
        b = rows(rng, nb, D, [(nb - 1, "dup"), (nb - 2, "zero"), (nb - 3, "tiny")])
        got = distance_matrix(a, b, metric, precision)
        if metric == "cosine":
            ref, bnd = do.cosine_matrix(a, b, do.TORCHREID_EPS), do.cosine_bound(a, b, do.TORCHREID_EPS, precision)
        else:
            ref, bnd = do.sq_euclidean(a, b), do.euclidean_bound(a, b, precision)
        check(got, ref, bnd, "distance_matrix %s D=%d %dx%d %s" % (metric, D, na, nb, precision))


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("D", DS)
def test_pair_cost_and_jde_distance_within_bound(D, precision):
    rng = np.random.default_rng(600 + D)
    for S, N in SHAPES:
        la = [S] if S < 3 else [1, 0, S - 1]
        lb = [N] if N < 3 else [1, 0, N - 1]
        sa, sb = seg_of(la), seg_of(lb)
        a = rows(rng, S, D, [(S - 1, "tiny"), (S - 2, "big"), (S - 3, "zero")])
        b = rows(rng, N, D, [(N - 1, "dup"), (N - 2, "zero")])
        gate = np.ones((len(la), len(lb)), np.uint8)
        gate[-1, 0] = 0
        got = pair_cost(a, sa, b, sb, precision, gate=gate, fill=999.0)
        ref = do.feature_dist(a, sa, b, sb, gate, fill=999.0)
        e = do.euclidean_bound(a, b, precision)
        check(got, ref, block_max(e, sa, sb), "pair_cost D=%d S=%d N=%d %s" % (D, S, N, precision))
        from object_detection_tracking_b200.tracking import euclidean_cost
        got = euclidean_cost(a, sa, b, precision=precision)
        check(got, do.nn_euclidean(a, sa, b), block_max(e, sa), "nn_euclidean D=%d %s" % (D, precision))
        got = jde_distance(a, b, precision)
        a64, b64 = a.astype(np.float64), b.astype(np.float64)
        n2 = (a64 * a64).sum(1)[:, None] + (b64 * b64).sum(1)[None, :]
        check(got, do.jde_cdist(a, b), np.sqrt(e + 1e-15 * n2), "jde D=%d S=%d N=%d %s" % (D, S, N, precision))


@pytest.mark.parametrize("precision", PRECISIONS)
def test_large_cosine_cost_200_tracks_of_100_rows_D2048(precision):
    rng = np.random.default_rng(7)
    D, T, N = 2048, 200, 130
    g = np.abs(rng.standard_normal((T * 100, D))).astype(np.float32)
    dets = np.abs(rng.standard_normal((N, D))).astype(np.float32)
    dets[:5] = g[[0, 150, 1999, 10050, 19999]]
    seg = (np.arange(T + 1) * 100).astype(np.int32)
    got = cosine_cost(g, seg, dets, precision)
    check(got, do.nn_cosine(g, seg, dets), block_max(do.cosine_bound(g, dets, 0.0, precision), seg),
          "cosine_cost 200x100 D=2048 %s" % precision)


@pytest.mark.parametrize("precision", PRECISIONS)
def test_large_pair_cost_3000_by_3000_crops(precision):
    rng = np.random.default_rng(8)
    D = 512
    sa = seg_of(rng.integers(1, 60, 100))
    sb = seg_of(rng.integers(1, 60, 100))
    a = rng.standard_normal((int(sa[-1]), D)).astype(np.float32)
    b = rng.standard_normal((int(sb[-1]), D)).astype(np.float32)
    b[:40] = a[:40]
    assert 2000 < sa[-1] < 4000 and 2000 < sb[-1] < 4000
    gate = (rng.uniform(size=(100, 100)) < 0.8).astype(np.uint8)
    got = pair_cost(a, sa, b, sb, precision, gate=gate, fill=999.0)
    ref = do.feature_dist(a, sa, b, sb, gate, fill=999.0)
    check(got, ref, block_max(do.euclidean_bound(a, b, precision), sa, sb), "pair_cost 3000x3000 %s" % precision)


@pytest.mark.parametrize("what", ["cosine_cost", "cosine", "euclidean", "pair_cost"])
def test_split_bound_is_sharp_fp16_breaks_it(what):
    """The split-precision bound is tight enough to catch a dropped lo plane: on a generic case the fp16-precision
    result breaks it, the split result does not."""
    rng = np.random.default_rng(9)
    D = 128
    a = rng.standard_normal((129, D)).astype(np.float32)
    b = rng.standard_normal((33, D)).astype(np.float32)
    seg = seg_of([1, 100, 28])
    sb = np.arange(len(b) + 1, dtype=np.int32)
    outcome = {}
    for precision in PRECISIONS:
        if what == "cosine_cost":
            got, ref, bnd = cosine_cost(a, seg, b, precision), do.nn_cosine(a, seg, b), block_max(
                do.cosine_bound(a, b, 0.0, "split"), seg)
        elif what == "cosine":
            got, ref = distance_matrix(a, b, "cosine", precision), do.cosine_matrix(a, b, do.TORCHREID_EPS)
            bnd = do.cosine_bound(a, b, do.TORCHREID_EPS, "split")
        elif what == "euclidean":
            got, ref, bnd = distance_matrix(a, b, "euclidean", precision), do.sq_euclidean(a, b), do.euclidean_bound(
                a, b, "split")
        else:
            got = pair_cost(a, seg, b, sb, precision)
            ref = do.feature_dist(a, seg, b, sb)
            bnd = block_max(do.euclidean_bound(a, b, "split"), seg, sb)
        try:
            check(got, ref, bnd, "%s %s" % (what, precision))
            outcome[precision] = True
        except AssertionError:
            outcome[precision] = False
    assert outcome == {"split": True, "fp16": False}, outcome


# ---- the non-finite cases each entry point used to get wrong ---------------------------------------------------------
@pytest.mark.parametrize("precision", PRECISIONS)
def test_zero_gallery_row_makes_its_track_nan(precision):
    """A zero gallery row divides 0 by 0 in nn_matching and np.min keeps the NaN: the track's costs are NaN (the kernel
    used to drop the NaN and return the minimum over the other rows)."""
    rng = np.random.default_rng(10)
    g = rows(rng, 10, 88, [(4, "zero")])
    dets = rows(rng, 5, 88)
    seg = seg_of([3, 4, 3])
    got = cosine_cost(g, seg, dets, precision)
    ref = do.nn_cosine(g, seg, dets)
    assert np.isnan(ref[1]).all()
    check(got, ref, block_max(do.cosine_bound(g, dets, 0.0, precision), seg), "zero gallery row")


@pytest.mark.parametrize("precision", PRECISIONS)
def test_zero_detection_row_is_nan_not_the_sentinel(precision):
    rng = np.random.default_rng(11)
    g = rows(rng, 10, 160)
    dets = rows(rng, 17, 160, [(16, "zero"), (3, "zero")])
    seg = seg_of([3, 4, 3])
    got = cosine_cost(g, seg, dets, precision)
    assert np.isnan(got[:, [3, 16]]).all() and np.isfinite(np.delete(got, [3, 16], axis=1)).all()
    check(got, do.nn_cosine(g, seg, dets), block_max(do.cosine_bound(g, dets, 0.0, precision), seg), "zero detection")


@pytest.mark.parametrize("precision", PRECISIONS)
def test_zero_row_torchreid_cosine_is_exactly_one(precision):
    """F.normalize clamps the norm at 1e-12: a zero row is at distance exactly 1 (it used to be 0/0 = NaN)."""
    rng = np.random.default_rng(12)
    a = rows(rng, 6, 512, [(2, "zero"), (3, "tiny")])
    b = rows(rng, 9, 512, [(0, "zero"), (5, "tiny")])
    got = distance_matrix(a, b, "cosine", precision)
    assert (got[2] == 1.0).all() and (got[:, 0] == 1.0).all()
    check(got, do.cosine_matrix(a, b, do.TORCHREID_EPS), do.cosine_bound(a, b, do.TORCHREID_EPS, precision), "zero row")


@pytest.mark.parametrize("precision", PRECISIONS)
def test_nan_embedding_is_nan_not_a_perfect_match(precision):
    """A NaN component: _pdist and the torchreid distance are NaN; the pair cost used to clamp it to 0."""
    rng = np.random.default_rng(13)
    D = 224
    a = rows(rng, 12, D, [(5, "nan")])
    b = rows(rng, 7, D, [(2, "nan")])
    sa, sb = seg_of([4, 4, 4]), seg_of([2, 2, 3])
    got = pair_cost(a, sa, b, sb, precision)
    ref = do.feature_dist(a, sa, b, sb)
    assert np.isnan(ref[1]).all() and np.isnan(ref[:, 1]).all()
    check(got, ref, block_max(do.euclidean_bound(a, b, precision), sa, sb), "pair cost NaN")
    from object_detection_tracking_b200.tracking import euclidean_cost
    got = euclidean_cost(a, sa, b, precision=precision)
    check(got, do.nn_euclidean(a, sa, b), block_max(do.euclidean_bound(a, b, precision), sa), "nn_euclidean NaN")
    got = distance_matrix(a, b, "euclidean", precision)
    check(got, do.sq_euclidean(a, b), do.euclidean_bound(a, b, precision), "distance_matrix NaN")
    got = distance_matrix(a, b, "cosine", precision)
    check(got, do.cosine_matrix(a, b, do.TORCHREID_EPS), do.cosine_bound(a, b, do.TORCHREID_EPS, precision),
          "torchreid cosine NaN")


@pytest.mark.parametrize("precision", PRECISIONS)
def test_tmot_distance_keeps_nan(precision):
    """np.maximum(0, cdist) keeps NaN; sqrt(std::max(0.0, NaN)) used to return 0, the best possible match."""
    rng = np.random.default_rng(14)
    a = rows(rng, 5, 288, [(1, "nan")])
    b = rows(rng, 4, 288, [(3, "nan"), (0, "dup")])
    got = jde_distance(a, b, precision)
    ref = do.jde_cdist(a, b)
    assert np.isnan(ref[1]).all() and np.isnan(ref[:, 3]).all()
    a64, b64 = a.astype(np.float64), b.astype(np.float64)
    n2 = np.nan_to_num((a64 * a64).sum(1)[:, None] + (b64 * b64).sum(1)[None, :])
    check(got, ref, np.sqrt(do.euclidean_bound(a, b, precision) + 1e-15 * n2), "jde NaN")


@pytest.mark.parametrize("precision", PRECISIONS)
def test_inf_components_never_give_a_finite_distance(precision):
    """A +-inf component: every cosine distance of the row is NaN, as the reference's inf / inf; every euclidean
    distance of the row is non-finite (NaN in split precision, where the lo plane of inf is NaN) while the reference's
    is inf or NaN.  Rows without one are unaffected."""
    rng = np.random.default_rng(15)
    D = 112
    a = rows(rng, 9, D)
    b = rows(rng, 6, D)
    a[2, 5], b[4, 0] = np.inf, -np.inf
    seg = seg_of([2, 3, 4])
    got = cosine_cost(a, seg, b, precision)
    check(got, do.nn_cosine(a, seg, b), block_max(do.cosine_bound(a, b, 0.0, precision), seg), "cosine_cost inf")
    got = distance_matrix(a, b, "cosine", precision)
    check(got, do.cosine_matrix(a, b, do.TORCHREID_EPS), do.cosine_bound(a, b, do.TORCHREID_EPS, precision), "cos inf")
    got = distance_matrix(a, b, "euclidean", precision)
    ref = do.sq_euclidean(a, b)
    assert not np.isfinite(ref[2]).any() and not np.isfinite(ref[:, 4]).any()
    fin = np.isfinite(ref)
    assert not np.isfinite(got[~fin]).any()
    if precision == "split":
        assert np.isnan(got[~fin]).all()
    check(np.where(fin, got, 0.0), np.where(fin, ref, 0.0), do.euclidean_bound(a, b, precision), "euclidean inf")


@pytest.mark.parametrize("value", [65504.0, 65519.0, 65520.0])
@pytest.mark.parametrize("precision", PRECISIONS)
def test_fp16_limit_components(value, precision):
    """Components up to 65519 are held finite by the planes and give finite distances within the bound; a finite 65520
    rounds to an fp16 inf, and every un-normalised entry point fails loudly instead of returning a NaN or a 0 cost.
    Normalised (cosine) rows are unaffected."""
    rng = np.random.default_rng(16)
    D = 64
    a = rows(rng, 6, D)
    b = rows(rng, 5, D)
    a[3, 7] = value
    sa, sb = seg_of([2, 4]), seg_of([5])
    check(cosine_cost(a, sa, b, precision), do.nn_cosine(a, sa, b),
          block_max(do.cosine_bound(a, b, 0.0, precision), sa), "cosine_cost %g" % value)
    check(distance_matrix(a, b, "cosine", precision), do.cosine_matrix(a, b, do.TORCHREID_EPS),
          do.cosine_bound(a, b, do.TORCHREID_EPS, precision), "cosine %g" % value)
    calls = {
        "b2_distance_matrix": lambda: (distance_matrix(a, b, "euclidean", precision), do.sq_euclidean(a, b),
                                       do.euclidean_bound(a, b, precision)),
        "b2_track_pair_cost": lambda: (pair_cost(a, sa, b, sb, precision), do.feature_dist(a, sa, b, sb),
                                       block_max(do.euclidean_bound(a, b, precision), sa, sb)),
        "b2_tmot_embedding_distance": lambda: (jde_distance(a, b, precision), do.jde_cdist(a, b),
                                               np.sqrt(do.euclidean_bound(a, b, precision) + 1e-15 * value ** 2)),
    }
    for name, call in calls.items():
        if value >= do.FP16_INF_FROM:
            with pytest.raises(RuntimeError, match="outside the fp16-plane range"):
                call()
        else:
            got, ref, bnd = call()
            check(got, ref, bnd, "%s %g %s" % (name, value, precision))
    # the failed call leaves nothing behind: the next one on the same workspace is clean
    check(distance_matrix(b, b, "euclidean", precision), do.sq_euclidean(b, b), do.euclidean_bound(b, b, precision),
          "after")


# ---- workspace reuse and the device-pointer path ---------------------------------------------------------------------
_SEQUENCE = r"""
import numpy as np, sys
sys.path.insert(0, %(root)r)
from object_detection_tracking_b200.engine import cosine_cost
from object_detection_tracking_b200.reid import compute_distance_matrix
from object_detection_tracking_b200.tracking import euclidean_cost
rng = np.random.default_rng(0)
out = {}
# D, gallery rows, detections: growing and shrinking D, Sp and Np; every other call has NaN, zero and inf rows
for k, (D, S, N) in enumerate([(64, 5, 7), (2048, 300, 40), (7, 129, 600), (512, 3, 2), (288, 128, 17), (33, 1, 1),
                              (2048, 257, 16), (65, 40, 90)]):
    g = rng.standard_normal((S, D)).astype(np.float32)
    d = rng.standard_normal((N, D)).astype(np.float32)
    if k %% 2:
        g[-1] = np.nan
        g[0, 0] = np.inf
        d[-1] = 0.0
        if N > 2:
            d[1, -1] = np.nan
    seg = np.array(sorted({0, S} | set(rng.integers(0, S, 3).tolist())), np.int32)
    for p in ("split", "fp16"):
        out["cos%%d%%s" %% (k, p)] = cosine_cost(g, seg, d, precision=p)
        out["cdm%%d%%s" %% (k, p)] = compute_distance_matrix(d, g, "cosine", precision=p).numpy()
        out["euc%%d%%s" %% (k, p)] = compute_distance_matrix(g, d, "euclidean", precision=p).numpy()
        out["pair%%d%%s" %% (k, p)] = euclidean_cost(g, seg, d, precision=p)
np.savez(sys.argv[1], **out)
"""


def test_workspace_reuse_equals_the_per_call_path_with_nonfinite_leftovers():
    """The persistent workspaces (grow-only buffers, cached plans) return the bits of a private workspace per call
    (B2_NO_WS=1) over a sequence that grows and shrinks D, the padded gallery rows and the padded columns, with calls
    whose inputs are NaN, inf or zero in between: leftover operand rows are harmless even when they are not finite."""
    res = []
    with tempfile.TemporaryDirectory() as tmp:
        for i, env in enumerate([{"B2_NO_WS": "1"}, {}]):
            path = os.path.join(tmp, "o%d.npz" % i)
            subprocess.run([sys.executable, "-c", _SEQUENCE % {"root": ROOT}, path], check=True,
                           env=dict(os.environ, **env), timeout=600)
            res.append(dict(np.load(path)))
    assert set(res[0]) == set(res[1]) and len(res[0]) == 64
    nan_seen = 0
    for k in res[0]:
        assert res[0][k].shape == res[1][k].shape, k
        np.testing.assert_array_equal(res[0][k], res[1][k], err_msg=k)   # NaN in the same places, equal elsewhere
        nan_seen += int(np.isnan(res[0][k]).any())
    assert nan_seen >= 16


@pytest.mark.parametrize("precision", PRECISIONS)
def test_pair_cost_dev_equals_host_path(precision):
    from object_detection_tracking_b200.reid import SharedGallery
    lib = _lib()
    rng = np.random.default_rng(17)
    for D, la, lb in ((88, [3, 0, 100, 1], [1, 15, 1]), (2048, [129], [16, 1]), (7, [1], [1]), (512, [40] * 20, [30] * 20)):
        sa, sb = seg_of(la), seg_of(lb)
        a = rows(rng, int(sa[-1]), D, [(0, "nan"), (2, "zero")])
        b = rows(rng, int(sb[-1]), D, [(1, "dup")])
        gate = (rng.uniform(size=(len(la), len(lb))) < 0.8).astype(np.uint8)
        ga, gb = SharedGallery(a), SharedGallery(b)
        try:
            out = np.empty((len(la), len(lb)), np.float32)
            lib.check(lib.load().b2_track_pair_cost_dev(0, ga.ptr, lib.ptr(sa), len(la), gb.ptr, lib.ptr(sb), len(lb), D,
                                                        lib.ptr(gate), 999.0, {"fp16": 0, "split": 1}[precision],
                                                        lib.ptr(out)), "b2_track_pair_cost_dev")
        finally:
            ga.close()
            gb.close()
        host = pair_cost(a, sa, b, sb, precision, gate=gate, fill=999.0)
        np.testing.assert_array_equal(out, host)
        check(out, do.feature_dist(a, sa, b, sb, gate, 999.0),
              block_max(do.euclidean_bound(a, b, precision), sa, sb), "dev D=%d %s" % (D, precision))
    big = rows(rng, 4, 64)
    big[1, 3] = 65520.0
    g = SharedGallery(big)
    try:
        s = seg_of([4])
        out = np.empty((1, 1), np.float32)
        with pytest.raises(RuntimeError, match="b2_track_pair_cost_dev.*outside the fp16-plane range"):
            lib.check(lib.load().b2_track_pair_cost_dev(0, g.ptr, lib.ptr(s), 1, g.ptr, lib.ptr(s), 1, 64, None, 0.0,
                                                        {"fp16": 0, "split": 1}[precision], lib.ptr(out)),
                      "b2_track_pair_cost_dev")
    finally:
        g.close()
