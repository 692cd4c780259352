"""Tracklet re-linking (object_detection_tracking_b200/relink.py) without a GPU, against the reference's own outputs in
tests/golden/relink.npz (make_golden_relink.py) on the synthetic video of tests/relink_inputs.py, and against a float32
transcription of single_video_reid.py:99-136 on random track sets: the candidate search, the planning of the needed
boxes, the merge fed the golden distances, the written files, and the reference's errors."""
import json
import os
import types

import numpy as np
import pytest

import relink_inputs as ri
from object_detection_tracking_b200 import relink


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
def track_files(tmp_path_factory):
    d = tmp_path_factory.mktemp("relink")
    return (ri.write_track_file(str(d / "p.txt"), ri.track_rows("p")),
            ri.write_track_file(str(d / "v.txt"), ri.track_rows("v")))


def as_json(c):
    return [[float(q), [[float(v) for v in row] for row in c[q]]] for q in c]


def same_distance_sign_free(a, b):
    """Candidate lists equal; distances compared exactly (golden-fed merges)."""
    assert len(a) == len(b)
    for (qa, ra), (qb, rb) in zip(a, b):
        assert qa == qb
        assert ra == rb, (qa, ra, rb)


# ---- single_video_reid.py:99-136 transcribed (float32 scalars, as the driver computes them under NumPy 2) -------------
def search_loop(track_ids, track_data, tol, wp, hp):
    def expand(t):
        left, top, width, height = t
        return [left - width * wp * 0.5, top - height * hp * 0.5, width * (1. + wp), height * (1. + hp)]

    def inter(t1, t2):
        l1, t1_, w1, h1 = t1
        l2, t2_, w2, h2 = t2
        xx1, yy1 = np.maximum(l1, l2), np.maximum(t1_, t2_)
        xx2, yy2 = np.minimum(l1 + w1, l2 + w2), np.minimum(t1_ + h1, t2_ + h2)
        with np.errstate(invalid="ignore", divide="ignore"):
            return (np.maximum(0, xx2 - xx1) * np.maximum(0, yy2 - yy1)) / (w2 * h2)

    pairs = {}
    for i1, a in enumerate(track_ids):
        end1 = track_data[a][-1, 0]
        e = expand(track_data[a][-1, 2:6])
        for i2 in range(i1 + 1, len(track_ids)):
            b = track_ids[i2]
            start2 = track_data[b][0, 0]
            if start2 <= end1 or not start2 - end1 < tol:
                continue
            if inter(e, track_data[b][0, 2:6]) > 0:
                if a not in pairs:
                    pairs[a] = [[b, start2, end1]]
                elif start2 == pairs[a][0][1]:
                    pairs[a].append([b, start2, end1])
    return pairs


def test_preprocess_matches_golden(golden, track_files):
    for cls, f in zip("pv", track_files):
        n, data, pairs = relink.preprocess(f, ri.TOL, ri.EXPAND_W, ri.EXPAND_H)
        assert n == len(data)
        assert as_json(pairs) == golden[0]["before"][cls]
        for q in pairs:                                              # the reference's element types
            for row in pairs[q]:
                assert type(row[0]) is float and row[1].dtype == np.float32 and row[2].dtype == np.float32
    _, _, p = relink.preprocess(track_files[0], ri.TOL, ri.EXPAND_W, ri.EXPAND_H)
    assert [r[0] for r in p[16.0]] == [17.0, 19.0]                   # 18 starts earlier but is not first-found
    assert 20.0 not in p and 22.0 not in p                           # touching boxes, a gap of exactly tol


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_preprocess_matches_transcription_on_random_tracks(tmp_path, seed):
    rng = np.random.default_rng(seed)
    n = 1500
    start = rng.integers(0, 3000, n)
    length = rng.integers(1, 40, n)
    rows = []
    for t in range(n):
        x, y = rng.uniform(0, 400), rng.uniform(0, 300)
        w, h = rng.choice([rng.uniform(0, 3), rng.uniform(10, 200), 0.0]), rng.uniform(0, 300)
        for f in range(int(start[t]), int(start[t] + length[t])):
            rows.append((f, t + 1, round(x, 2), round(y, 2), round(w, 2), round(h, 2), 0.9))
            x += rng.normal(0, 3)
            y += rng.normal(0, 3)
    rows.sort()
    path = ri.write_track_file(str(tmp_path / "t.txt"), rows)
    total = 0
    for tol, wp, hp in ((200, 2.0, 0.5), (30, 0.1, 0.1), (7, 0.0, 0.0)):
        _, data, pairs = relink.preprocess(path, tol, wp, hp)
        ref = search_loop(sorted(data), data, tol, wp, hp)
        assert list(pairs) == list(ref)
        for q in ref:
            assert [[r[0], float(r[1]), float(r[2])] for r in pairs[q]] == [[r[0], float(r[1]), float(r[2])]
                                                                               for r in ref[q]]
        total += sum(len(v) for v in ref.values())
    assert total > 200


def test_planned_boxes_match_golden(golden, track_files):
    for run in golden:
        box_num, gap = run["params"][:2]
        _, pd, pc = relink.preprocess(track_files[0], ri.TOL, ri.EXPAND_W, ri.EXPAND_H)
        _, vd, vc = relink.preprocess(track_files[1], ri.TOL, ri.EXPAND_W, ri.EXPAND_H)
        needed = {}
        relink.plan_boxes(needed, pd, pc, box_num, gap)
        relink.plan_boxes(needed, vd, vc, box_num, gap)
        assert [[k, [[float(x) for x in b] for b in v]] for k, v in needed.items()] == run["needed"]
    # the shared keys: vehicle 7 re-planned "query_7.0", "gallery_8.0" kept person 8's boxes
    assert dict(golden[0]["needed"])["query_7.0"][0][2] == 10.0
    assert dict(golden[0]["needed"])["gallery_8.0"][0][3] == 40.0
    _, pd, _ = relink.preprocess(track_files[0], ri.TOL, ri.EXPAND_W, ri.EXPAND_H)
    gap = golden[1]["params"][1]                                             # feature_box_num <= 0: every gap-th box
    assert len(dict(golden[1]["needed"])["query_16.0"]) == -(-len(pd[16.0]) // gap) == 4


def golden_fed_reid(run, track_files):
    """reid() with the crops' validity and the distances taken from the golden run instead of the GPU."""
    _, pd, pc = relink.preprocess(track_files[0], ri.TOL, ri.EXPAND_W, ri.EXPAND_H)
    _, vd, vc = relink.preprocess(track_files[1], ri.TOL, ri.EXPAND_W, ri.EXPAND_H)
    got = {k: set(v) for k, v in run["valid"].items()}
    out = {}
    for cls, data, cands in (("p", pd, pc), ("v", vd, vc)):
        dist_of = {(q, r[0]): np.float32(r[3]) for q, rows in run["after"][cls] for r in rows}
        live, remove = relink.prune_candidates(cands, got)
        dist = [dist_of[(q, r[0])] for q in live for r in cands[q]]
        relink.attach_distances(cands, live, remove, dist)
        out[cls] = (cands, data, relink.merge_candidates(cands, data, run["params"][2]))
    return out


def test_merge_fed_golden_distances_matches_golden(golden, track_files, tmp_path):
    for r, run in enumerate(golden):
        out = golden_fed_reid(run, track_files)
        for cls, cat in (("p", "Person"), ("v", "Vehicle")):
            cands, data, new = out[cls]
            same_distance_sign_free(as_json(cands), run["after"][cls])
            assert sorted(new) == run["new_ids"][cls]
            relink.save_new_track(cat, new, str(tmp_path / ("r%d" % r)), "video.mp4")
            raw = open(str(tmp_path / ("r%d" % r) / "video.mp4" / cat / "video.txt"), "rb").read()
            assert raw == run[cat]
        p_c, p_data, p_new = out["p"]
        assert 9.0 not in p_c and 14.0 not in p_c                          # queries without a valid crop removed
        assert [row[0] for row in p_c[11.0]] == [13.0]                      # gallery 12 has no valid crop
        assert set(p_new) >= {1.0, 4.0, 7.0, 8.0, 24.0} and 3.0 not in p_new and 6.0 not in p_new and 26.0 not in p_new
        assert (p_new[1.0][:, 1] == 1.0).all() and len(p_new[1.0]) == 30  # the chain 1 <- 2 <- 3
        assert (p_data[3.0][:, 1] == 1.0).all()                           # written through the caller's arrays
        assert 5.0 in p_new and 25.0 in p_new                               # the losing claims stay apart


def test_nan_distance_never_matches(track_files):
    _, pd, pc = relink.preprocess(track_files[0], ri.TOL, ri.EXPAND_W, ri.EXPAND_H)
    cands = {1.0: [[2.0, 13, 9, np.float32(np.nan)]]}
    new = relink.merge_candidates(cands, {1.0: pd[1.0], 2.0: pd[2.0]}, 1e9)
    assert sorted(new) == [1.0, 2.0]


def test_reference_errors(tmp_path, track_files):
    with pytest.raises(TypeError):
        relink.preprocess(track_files[0], ri.TOL, ri.EXPAND_W, ri.EXPAND_H, reject_track_conf_thres=0.1)
    with pytest.raises(TypeError):
        relink.preprocess(track_files[0], ri.TOL, ri.EXPAND_W, ri.EXPAND_H, reject_track_conf_thres=0.99)
    assert relink.preprocess(ri.write_track_file(str(tmp_path / "e.txt"), []))[:2] == (0, [])

    def no_gpu(*a, **k):
        raise AssertionError("nothing should be embedded")
    ext = types.SimpleNamespace(batch=4, engine=types.SimpleNamespace(feat_dim=512, device=0, embed_boxes_dev=no_gpu))
    video = ri.frames()
    _, pd, pc = relink.preprocess(track_files[0], ri.TOL, ri.EXPAND_W, ri.EXPAND_H)
    _, vd, vc = relink.preprocess(track_files[1], ri.TOL, ri.EXPAND_W, ri.EXPAND_H)
    with pytest.raises(KeyError):                                        # needed frames that never arrive
        relink.reid(ri.frame_iter(video, []), ext, ext, pd, pc, vd, vc)
    rows = [(0, 1, 10, 10, 0.5, 30, 0.9), (1, 1, 10, 10, 0.5, 30, 0.9), (3, 2, 10, 10, 8, 30, 0.9)]
    path = ri.write_track_file(str(tmp_path / "z.txt"), rows)
    _, zd, zc = relink.preprocess(path, 10, 0.1, 0.1)
    assert list(zc) == [1.0]
    with pytest.raises(ValueError, match="empty"):                       # valid_box passes, int(w) == 0
        relink.reid(ri.frame_iter(video, [0, 1, 2, 3]), ext, ext, zd, zc, {}, {}, frames_per_call=8)
