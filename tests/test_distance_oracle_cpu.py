"""tests/distance_oracle.py against the code it restates, on the values where distance kernels go wrong: zero rows, rows
with a norm below 1e-12, exact duplicates, NaN and +-inf components, components at the fp16 limit.  The references here
are oracle/nn_matching (DeepSORT's metric), torch's F.normalize on the CPU (torchreid's cosine distance), sklearn's
euclidean_distances (compute_feature_dist) and scipy's cdist (the JDE embedding distance)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import conv_oracle as co
import distance_oracle as do
from oracle import nn_matching


def adversarial(rng, D=16):
    """Rows: generic, zero, norm 1e-13, duplicate of row 0, NaN component, +inf, -inf, fp16-limit components."""
    x = rng.standard_normal((9, D)).astype(np.float32)
    x[1] = 0.0
    x[2] = (x[2] / np.linalg.norm(x[2]) * 1e-13).astype(np.float32)
    x[3] = x[0]
    x[4, 3] = np.nan
    x[5, 1] = np.inf
    x[6, 2] = -np.inf
    x[7, :3] = [65504.0, 65519.0, -65520.0]
    return x


def same(got, exp, rtol=1e-12, atol=0.0):
    got, exp = np.asarray(got, np.float64), np.asarray(exp, np.float64)
    assert got.shape == exp.shape
    np.testing.assert_array_equal(np.isnan(got), np.isnan(exp))
    m = ~np.isnan(exp)
    np.testing.assert_allclose(got[m], exp[m], rtol=rtol, atol=atol)


def test_nn_cosine_and_euclidean_match_nn_matching():
    rng = np.random.default_rng(0)
    g = adversarial(rng)
    dets = np.concatenate([adversarial(rng)[[0, 1, 3, 4, 5]], g[:2]])
    seg = np.array([0, 1, 2, 4, 5, 9], np.int32)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        for metric, fn in (("cosine", do.nn_cosine), ("euclidean", do.nn_euclidean)):
            m = nn_matching.NearestNeighborDistanceMetric(metric, 0.5)
            m.samples = {t: list(g[seg[t]:seg[t + 1]].astype(np.float64)) for t in range(len(seg) - 1)}
            same(fn(g, seg, dets), m.distance(dets.astype(np.float64), list(range(len(seg) - 1))), atol=1e-9)
    cos = do.nn_cosine(g, seg, dets)
    assert np.isnan(cos[1]).all() and np.isnan(cos[:, 1]).all()            # zero gallery row / zero detection
    assert np.isfinite(cos[2, [0, 2]]).all() and np.isfinite(cos[0, [0, 2]]).all()   # tiny-norm row, duplicate
    assert np.isnan(cos[4]).all()                                           # NaN and inf rows poison their track


def test_empty_segment_is_the_kernels_sentinel():
    g = np.ones((2, 4), np.float32)
    out = do.nn_cosine(g, [0, 0, 2], g)
    assert (out[0] == do.EMPTY_SEGMENT).all() and (out[1] == 0).all()
    assert (do.cosine_segmin_f32(np.zeros((2, 3), np.float32), [0, 2, 2])[1] == do.EMPTY_SEGMENT).all()


def test_torchreid_cosine_matches_f_normalize():
    rng = np.random.default_rng(1)
    a = adversarial(rng)
    b = np.concatenate([adversarial(rng), a[:3]])
    at, bt = torch.from_numpy(a.astype(np.float64)), torch.from_numpy(b.astype(np.float64))
    ref = (1 - F.normalize(at, p=2, dim=1) @ F.normalize(bt, p=2, dim=1).t()).numpy()
    got = do.cosine_matrix(a, b, do.TORCHREID_EPS)
    same(got, ref, atol=1e-12)
    assert (got[1, np.isfinite(got[1])] == 1.0).all() and np.isfinite(got[1, [0, 1, 2]]).all()   # zero row: exactly 1
    # norm 1e-13 < eps: x / 1e-12 has norm 0.1, so the distance is within 0.1 of 1
    assert np.linalg.norm(do.normalize(a[2:3], do.TORCHREID_EPS)) == pytest.approx(0.1, rel=1e-6)
    assert abs(got[2, 0] - 1.0) <= 0.1 + 1e-12
    assert np.isnan(got[4]).all() and np.isnan(got[5]).all() and np.isnan(got[6]).all()


def test_squared_euclidean_matches_torch_and_sklearn():
    from sklearn.metrics.pairwise import euclidean_distances
    rng = np.random.default_rng(2)
    a = adversarial(rng)
    b = np.concatenate([adversarial(rng), a[:4]])
    at, bt = torch.from_numpy(a.astype(np.float64)), torch.from_numpy(b.astype(np.float64))
    ref = (at.pow(2).sum(1, keepdim=True) + bt.pow(2).sum(1, keepdim=True).t() - 2 * at @ bt.t()).numpy()
    got = do.sq_euclidean(a, b)
    fin = np.isfinite(a).all(1)[:, None] & np.isfinite(b).all(1)[None, :]
    same(got[fin], ref[fin], rtol=1e-12, atol=1e-4)
    assert np.isnan(got[4]).all() and not np.isfinite(got[5]).any()
    ra, rb = np.isfinite(a).all(1), np.isfinite(b).all(1)
    sk = euclidean_distances(a[ra].astype(np.float64), b[rb].astype(np.float64), squared=True)
    np.testing.assert_allclose(np.maximum(got[np.ix_(ra, rb)], 0), sk, rtol=1e-9, atol=1e-3)
    assert got[0, 9 + 3] == pytest.approx(0.0, abs=1e-12)                   # duplicate rows


def test_feature_dist_matches_sklearn_loop_and_gates():
    from sklearn.metrics.pairwise import euclidean_distances
    rng = np.random.default_rng(3)
    a = rng.standard_normal((10, 8)).astype(np.float32)
    b = np.concatenate([rng.standard_normal((6, 8)), a[[2]]]).astype(np.float32)
    sa, sb = np.array([0, 3, 3, 10]), np.array([0, 1, 4, 7])
    gate = np.array([[1, 1, 0], [1, 1, 1], [1, 0, 1]], np.uint8)
    got = do.feature_dist(a, sa, b, sb, gate, fill=999.0)
    for i in range(3):
        for j in range(3):
            if gate[i, j] == 0 or sa[i] == sa[i + 1]:
                assert got[i, j] == 999.0
            else:
                exp = euclidean_distances(a[sa[i]:sa[i + 1]].astype(np.float64), b[sb[j]:sb[j + 1]].astype(np.float64),
                                          squared=True).min()
                assert got[i, j] == pytest.approx(exp, rel=1e-9, abs=1e-9)
    a[5, 0] = np.nan
    got = do.feature_dist(a, sa, b, sb, gate, fill=999.0)
    assert np.isnan(got[2, [0, 2]]).all() and got[2, 1] == 999.0 and np.isfinite(got[:2]).all()


def test_jde_cdist_matches_scipy():
    from scipy.spatial.distance import cdist
    rng = np.random.default_rng(4)
    a, b = adversarial(rng), adversarial(rng)
    with np.errstate(invalid="ignore"):
        same(do.jde_cdist(a, b), np.maximum(0, cdist(a.astype(np.float64), b.astype(np.float64))))
    assert np.isnan(do.jde_cdist(a, b)[4]).all()


def test_f32_epilogues_are_single_roundings_of_float64():
    """Each step of the float32 restatements is one IEEE op: a float32 add, subtract or multiply of float32 operands is
    the float64 result rounded once to float32."""
    rng = np.random.default_rng(5)
    d = (rng.standard_normal((7, 9)) * 10.0 ** rng.integers(-8, 8, (7, 9))).astype(np.float32)
    na2, nb2 = np.abs(rng.standard_normal(7) * 100).astype(np.float32), np.abs(rng.standard_normal(9)).astype(np.float32)
    np.testing.assert_array_equal(do.finish_f32(d, 0), (1.0 - d.astype(np.float64)).astype(np.float32))
    s = (na2[:, None].astype(np.float64) + nb2[None, :]).astype(np.float32)
    np.testing.assert_array_equal(do.finish_f32(d, 1, na2, nb2), (s.astype(np.float64) - 2.0 * d).astype(np.float32))
    d[2, 4] = np.nan
    cs = do.cosine_segmin_f32(d, [0, 3, 3, 7])
    assert np.isnan(cs[0, 4]) and (cs[1] == do.EMPTY_SEGMENT).all() and np.isfinite(np.delete(cs[0], 4)).all()
    ps = do.pair_segmin_f32(d, na2, nb2, [0, 3, 7], [0, 5, 5, 9], np.array([[1, 1, 1], [0, 1, 1]], np.uint8), fill=-1.0)
    assert np.isnan(ps[0, 0]) and ps[0, 1] == -1.0 and ps[1, 0] == -1.0 and (ps[:, 2] >= 0).all()


def test_range_flag_and_planes():
    x = np.array([[65504.0, 65519.0, -65519.0, np.inf, np.nan, -np.inf]], np.float32)
    assert not do.out_of_range(x)
    assert do.out_of_range(np.array([[0.0, -65520.0]], np.float32))
    assert do.out_of_range(np.array([[3e38]], np.float32))
    hi, lo = do.planes_raw(x, ld=8)
    assert hi.shape == (1, 8) and (hi[0, 6:] == 0).all() and (lo[0, 6:] == 0).all()
    assert hi[0, 1].view(np.float16) == 65504 and lo[0, 1].view(np.float16) == 15 * 2048


def test_split_bound_holds_for_the_plane_arithmetic_and_fp16_breaks_it():
    """The split planes' dot product (in float64) lies within the bound of a generic case; the fp16 plane alone does not
    (the GPU suite repeats this with the kernels)."""
    rng = np.random.default_rng(6)
    a = rng.standard_normal((64, 128)).astype(np.float32)
    b = rng.standard_normal((48, 128)).astype(np.float32)
    ref = do.sq_euclidean(a, b)
    bnd = do.euclidean_bound(a, b, "split")
    for prec, ok in (("split", True), ("fp16", False)):
        ra, rb = co.represent(a, prec == "split"), co.represent(b, prec == "split")
        got = (a.astype(np.float64) ** 2).sum(1)[:, None] + (b.astype(np.float64) ** 2).sum(1)[None] - 2 * ra @ rb.T
        assert bool((np.abs(got - ref) <= bnd).all()) == ok, prec
