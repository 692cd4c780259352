"""Tracklet re-linking on the GPU: b2_tracklet_dist_dev against a float64 evaluation within the split-precision (and
fp16) error bound of tests/distance_oracle.py, its refusals, and relink.reid end to end on the synthetic video of
tests/relink_inputs.py against the reference's outputs in tests/golden/relink.npz."""
import json
import os

import numpy as np
import pytest

import distance_oracle as do
import relink_inputs as ri
from test_distance_kernels_gpu import block_max, check, rows, seg_of

pytestmark = pytest.mark.gpu


def dev(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda()


def tracklet_dist(q, sq, g, sg, pairs, method="min_all", precision="split"):
    from object_detection_tracking_b200 import relink
    return relink.tracklet_dist(dev(q), sq, dev(g), sg, pairs, method, precision)


def pair_ref(d, sq, sg, pairs):
    """min over each pair's block of the float64 matrix d (NaN kept)."""
    return np.array([np.min(d[sq[i]:sq[i + 1], sg[j]:sg[j + 1]]) for i, j in pairs])


def mean_f32(x, seg):
    """segment_mean_kernel restated: float32 sum in row order, divided by the count."""
    out = np.zeros((len(seg) - 1, x.shape[1]), np.float32)
    for s in range(len(seg) - 1):
        acc = np.zeros(x.shape[1], np.float32)
        for r in range(seg[s], seg[s + 1]):
            acc = acc + x[r]
        out[s] = acc / np.float32(seg[s + 1] - seg[s])
    return out


@pytest.mark.parametrize("precision", ["split", "fp16"])
@pytest.mark.parametrize("D", [512, 2048])
def test_min_all_within_bound(D, precision):
    rng = np.random.default_rng(D)
    lq, lg = [1, 500, 3, 1, 37], [500, 1, 2, 64, 1, 17]
    sq, sg = seg_of(lq), seg_of(lg)
    q = rows(rng, int(sq[-1]), D, [(1, "dup")])
    g = rows(rng, int(sg[-1]), D)
    g[0] = q[0]                                                      # a duplicate across the two tables
    pairs = [(i, j) for i in range(len(lq)) for j in range(len(lg))]
    pairs = pairs[::-1] + [(1, 0), (0, 0), (1, 0)]                  # unordered and repeated
    got = tracklet_dist(q, sq, g, sg, pairs, "min_all", precision)
    e = do.euclidean_bound(q, g, precision)
    bnd = np.array([block_max(e, sq, sg)[i, j] for i, j in pairs])
    check(got, pair_ref(do.sq_euclidean(q, g), sq, sg, pairs), bnd, "min_all D=%d %s" % (D, precision))


def test_thousands_of_pairs():
    rng = np.random.default_rng(5)
    lq, lg = rng.integers(1, 6, 300), rng.integers(1, 6, 200)
    sq, sg = seg_of(lq), seg_of(lg)
    q, g = rows(rng, int(sq[-1]), 512), rows(rng, int(sg[-1]), 512)
    pairs = np.stack([rng.integers(0, 300, 5000), rng.integers(0, 200, 5000)], 1)
    got = tracklet_dist(q, sq, g, sg, pairs)
    bm = block_max(do.euclidean_bound(q, g, "split"), sq, sg)
    check(got, pair_ref(do.sq_euclidean(q, g), sq, sg, pairs), bm[pairs[:, 0], pairs[:, 1]], "5000 pairs")


def test_duplicates_keep_their_sign_and_nan_propagates():
    rng = np.random.default_rng(9)
    D = 512
    base = rows(rng, 64, D)
    q = base[:32].copy()
    g = base[:32].copy()                                            # every query row has an exact duplicate
    sq, sg = seg_of([1] * 32), seg_of([1] * 32)
    pairs = [(i, i) for i in range(32)]
    got = tracklet_dist(q, sq, g, sg, pairs)
    bnd = np.diag(do.euclidean_bound(q, g, "split"))
    assert (np.abs(got) <= bnd).all()
    assert (got < 0).any() or (got == 0).all()                      # unclamped: a negative rounding survives
    qn = q.copy()
    qn[3, 5] = np.nan
    got = tracklet_dist(qn, seg_of([4, 28]), g, seg_of([2, 30]), [(0, 0), (0, 1), (1, 0), (1, 1)])
    assert np.isnan(got[:2]).all() and np.isfinite(got[2:]).all()


@pytest.mark.parametrize("D", [512, 2048])
def test_avg_is_the_distance_of_the_means(D):
    rng = np.random.default_rng(D + 1)
    lq, lg = [1, 500, 7], [3, 1, 500, 2]
    sq, sg = seg_of(lq), seg_of(lg)
    q, g = rows(rng, int(sq[-1]), D), rows(rng, int(sg[-1]), D)
    mq, mg = mean_f32(q, sq), mean_f32(g, sg)
    for m, x, s in ((mq, q, sq), (mg, g, sg)):                       # the restated means against float64 means
        m64 = np.stack([x[s[i]:s[i + 1]].astype(np.float64).mean(0) for i in range(len(s) - 1)])
        n = np.diff(s)[:, None]
        assert (np.abs(m - m64) <= (n + 1) * do.U * np.abs(x).max()).all()
    pairs = [(i, j) for i in range(3) for j in range(4)] + [(2, 2), (0, 0)]
    got = tracklet_dist(q, sq, g, sg, pairs, "avg")
    e = do.euclidean_bound(mq, mg, "split")
    ref = do.sq_euclidean(mq, mg)
    idx = np.asarray(pairs)
    check(got, ref[idx[:, 0], idx[:, 1]], e[idx[:, 0], idx[:, 1]], "avg D=%d" % D)


def test_refusals():
    from object_detection_tracking_b200 import relink
    rng = np.random.default_rng(1)
    q, g = dev(rows(rng, 6, 64)), dev(rows(rng, 6, 64))
    ok = seg_of([3, 3])
    cases = [(seg_of([3, 3])[::-1].copy(), ok, [(0, 0)], "min_all", "start at 0|monotone"),
             (np.array([0, 4, 3, 6], np.int32), np.array([0, 2, 4, 6], np.int32), [(0, 0)], "min_all", "monotone"),
             (np.array([0, 3, 3, 6], np.int32), ok, [(0, 0)], "min_all", "empty query segment"),
             (ok, np.array([0, 0, 6], np.int32), [(0, 0)], "min_all", "empty gallery segment"),
             (ok, ok, [(2, 0)], "min_all", "out of range"),
             (ok, ok, [(0, -1)], "avg", "out of range")]
    for sq, sg, pairs, method, msg in cases:
        with pytest.raises(RuntimeError, match="b2_tracklet_dist_dev.*(%s)" % msg):
            relink.tracklet_dist(q, sq, g, sg, pairs, method)
    with pytest.raises(ValueError):
        relink.tracklet_dist(q, ok, g, ok, [(0, 0)], "max")
    from object_detection_tracking_b200 import _lib
    out = np.zeros(1, np.float32)
    pr = np.zeros(2, np.int32)
    with pytest.raises(RuntimeError, match="method"):
        _lib.check(_lib.load().b2_tracklet_dist_dev(0, q.data_ptr(), _lib.ptr(ok), 2, g.data_ptr(), _lib.ptr(ok), 2, 64,
                                                    _lib.ptr(pr), 1, 2, 1, _lib.ptr(out)), "b2_tracklet_dist_dev")
    big = rows(rng, 6, 64)
    big[2, 7] = 65520.0
    with pytest.raises(RuntimeError, match="b2_tracklet_dist_dev.*outside the fp16-plane range"):
        relink.tracklet_dist(dev(big), ok, g, ok, [(0, 0)])


# ---- end to end ------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def golden(golden_dir):
    z = np.load(os.path.join(golden_dir, "relink.npz"))
    runs = []
    for r in range(len(ri.RUNS)):
        info = json.loads(str(z["run%d_json" % r]))
        info["Person"] = z["run%d_Person" % r].tobytes()
        info["Vehicle"] = z["run%d_Vehicle" % r].tobytes()
        runs.append(info)
    return runs


@pytest.fixture(scope="module")
def extractors():
    from object_detection_tracking_b200.reid import FeatureExtractor
    from object_detection_tracking_b200.synth import synth_osnet_state, synth_resnet101_reid_state
    p_state, v_state = synth_osnet_state(4321), synth_resnet101_reid_state(2468)
    out = {}
    for b in (4, 32):
        out[b] = (FeatureExtractor("osnet_x1_0", image_size=(256, 128), batch=b, state_dict=p_state),
                  FeatureExtractor("resnet101", image_size=(128, 256), batch=b, state_dict=v_state))
    return out


@pytest.fixture(scope="module")
def video():
    return ri.frames()


def run_reid(tmp, run, exts, video, frames_per_call, feat_max):
    from object_detection_tracking_b200 import relink
    pf = ri.write_track_file(os.path.join(tmp, "p.txt"), ri.track_rows("p"))
    vf = ri.write_track_file(os.path.join(tmp, "v.txt"), ri.track_rows("v"))
    _, pd, pc = relink.preprocess(pf, ri.TOL, ri.EXPAND_W, ri.EXPAND_H)
    _, vd, vc = relink.preprocess(vf, ri.TOL, ri.EXPAND_W, ri.EXPAND_H)
    box_num, gap, thr, method = run["params"]
    orig = relink.tracklet_dist

    def spy(qf, sq, gf, sg, pairs, m, p):                            # the features' scale, for the distance tolerance
        feat_max.append((float(max(qf.abs().max(), gf.abs().max())), int(qf.shape[1]),
                         float(max((qf.double() ** 2).sum(1).max(), (gf.double() ** 2).sum(1).max()))))
        return orig(qf, sq, gf, sg, pairs, m, p)
    relink.tracklet_dist = spy
    try:
        new_p, new_v = relink.reid(ri.frame_iter(video), exts[0], exts[1], pd, pc, vd, vc, feature_box_num=box_num,
                                   feature_box_gap=gap, reject_dist_thres=thr, compare_method=method,
                                   frames_per_call=frames_per_call)
    finally:
        relink.tracklet_dist = orig
    files = {}
    for cat, new in (("Person", new_p), ("Vehicle", new_v)):
        relink.save_new_track(cat, new, tmp, "video.mp4")
        files[cat] = open(os.path.join(tmp, "video.mp4", cat, "video.txt"), "rb").read()
    return {"p": pc, "v": vc}, files


def test_reid_end_to_end_matches_reference(golden, extractors, video, tmp_path):
    for r, run in enumerate(golden):
        scale = []
        cands, files = run_reid(str(tmp_path / ("r%d" % r)), run, extractors[32], video, 8, scale)
        assert files["Person"] == run["Person"] and files["Vehicle"] == run["Vehicle"], "run %d" % r
        for k, cls in enumerate("pv"):
            fmax, D, sq = scale[k]
            e = (2e-5 if cls == "p" else 3e-5) * fmax                   # per-component feature tolerance (test_reid*)
            got = [[q, [list(map(float, row)) for row in rows_]] for q, rows_ in cands[cls].items()]
            exp = run["after"][cls]
            assert [(q, [row[:3] for row in rs]) for q, rs in got] == [(q, [row[:3] for row in rs]) for q, rs in exp]
            for (_, rg), (_, re_) in zip(got, exp):
                for a, b in zip(rg, re_):
                    tol = 4 * np.sqrt(max(b[3], 0.0)) * e * np.sqrt(D) + 4 * e * e * D + 8e-7 * sq
                    assert abs(a[3] - b[3]) <= tol, (r, cls, a, b, tol)


def test_reid_is_independent_of_chunking(golden, extractors, video, tmp_path):
    run = golden[0]
    results = []
    for b, fpc in ((32, 8), (32, 1), (4, 8), (4, 1)):
        cands, files = run_reid(str(tmp_path / ("b%d_f%d" % (b, fpc))), run, extractors[b], video, fpc, [])
        results.append(({c: [(q, [list(map(float, row)) for row in rs]) for q, rs in cands[c].items()] for c in "pv"},
                        files))
    for other in results[1:]:
        assert other == results[0]
