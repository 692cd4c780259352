"""Times tracklet re-linking (relink.reid) end to end on a synthetic 1080p video generated on the fly, against the
reference's loop structure (single_video_reid.py:156-365: host crops kept per key, every gallery embedded again for each
query that lists it, one distance matrix and torch.min per candidate pair) run with this package's host-crop
FeatureExtractor.__call__ and reid.compute_distance_matrix.  Both must give the same merges before anything is timed.

    python tools/bench_relink.py [--frames 240] [--persons 150] [--vehicles 50] [--repeat 3]
Prints one JSON line with the card name and power limit read in the same run.
"""
import argparse
import json
import operator
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import relink_inputs as ri  # noqa: E402
from object_detection_tracking_b200 import relink  # noqa: E402
from object_detection_tracking_b200.reid import compute_distance_matrix  # noqa: E402

H, W = 1080, 1920


def scene(n_frames, n_p, n_v, seed=0):
    """Tracklets in pairs: each identity leaves and re-enters once (a gap of 3-8 frames), boxes drift slowly."""
    rng = np.random.default_rng(seed)
    tracks, tid = [], 1
    for cls, n, (bw, bh) in (("p", n_p, (60, 150)), ("v", n_v, (220, 110))):
        for k in range(n // 2):
            ident = (1 if cls == "p" else 1000) + k
            x, y = int(rng.integers(0, W - bw - 40)), int(rng.integers(0, H - bh - 10))
            f0 = int(rng.integers(0, n_frames - 60))
            l1 = int(rng.integers(15, 30))
            gap = int(rng.integers(3, 9))
            l2 = int(rng.integers(15, 30))
            tracks.append((cls, tid, ident, f0, f0 + l1 - 1, x, y, bw, bh))
            tracks.append((cls, tid + 1, ident, f0 + l1 + gap, min(f0 + l1 + gap + l2, n_frames) - 1, x + 6, y, bw, bh))
            tid += 2
    return tracks


def rows_of(tracks, cls):
    return sorted((f, t, x + (f % 5), y, w, h + f % 3, 0.9) for c, t, _, f0, f1, x, y, w, h in tracks if c == cls
                  for f in range(f0, f1 + 1))


def frame_source(tracks, n_frames):
    bg = ri.background(H, W)
    sprites = {}
    for c, _, ident, *_ in tracks:
        if ident not in sprites:
            sprites[ident] = ri.sprite(ident, 48, 24) if c == "p" else ri.sprite(ident, 24, 48)

    def make(f):
        img = bg.copy()
        for c, _, ident, f0, f1, x, y, w, h in tracks:
            if f0 <= f <= f1:
                ri.paint(img, sprites[ident], x + (f % 5), y, w, h + f % 3)
        return img
    return make


def reference_loop(frames, p_ext, v_ext, pd, pc, vd, vc, box_num, box_gap, thr):
    """single_video_reid.py:156-365 with the package's host-crop extractor and distance matrix (min_all)."""
    needed = {}
    relink.plan_boxes(needed, pd, pc, box_num, box_gap)
    relink.plan_boxes(needed, vd, vc, box_num, box_gap)
    frame_data = {}
    for key in needed:
        for bi, box in enumerate(needed[key]):
            frame_data.setdefault(box[0], []).append((box[2:6], key, bi))
    imgs = {}
    for f, image in enumerate(frames):
        if f in frame_data:
            for tlwh, key, bi in frame_data[f]:
                imgs.setdefault(key, {})
                if relink.valid_box(tlwh, image):
                    x, y, w, h = (int(v) for v in tlwh)
                    imgs[key][bi] = np.ascontiguousarray(image[y:y + h, x:x + w, ::-1])

    def compare(cands, ext):
        import torch
        remove = {}
        for q in cands:
            qb = imgs["query_%s" % q]
            if not qb:
                remove[q] = 1
                continue
            qf = ext([qb[i] for i in sorted(qb)])
            temp = [c for c in cands[q] if imgs["gallery_%s" % c[0]]]
            if not temp:
                remove[q] = 1
                continue
            cands[q] = temp
            dist = torch.zeros((1, len(temp)))
            for i, (g, _, _) in enumerate(temp):
                gb = imgs["gallery_%s" % g]
                gf = ext([gb[k] for k in sorted(gb)])
                dist[0, i] = torch.min(compute_distance_matrix(qf, gf, "euclidean"))
            dist = dist.numpy()
            for i in range(dist.shape[1]):
                cands[q][i].append(dist[0, i])
            cands[q].sort(key=operator.itemgetter(-1))
        for q in remove:
            del cands[q]
    compare(pc, p_ext)
    compare(vc, v_ext)
    return relink.merge_candidates(pc, pd, thr), relink.merge_candidates(vc, vd, thr)


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:       # the timing itself still needs the GPU
        return "unknown (%s)" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=240)
    ap.add_argument("--persons", type=int, default=150)
    ap.add_argument("--vehicles", type=int, default=50)
    ap.add_argument("--box_num", type=int, default=5)
    ap.add_argument("--box_gap", type=int, default=3)
    ap.add_argument("--repeat", type=int, default=3)
    a = ap.parse_args()
    import torch
    from object_detection_tracking_b200.reid import FeatureExtractor
    from object_detection_tracking_b200.synth import synth_osnet_state, synth_resnet101_reid_state
    p_ext = FeatureExtractor("osnet_x1_0", image_size=(256, 128), batch=32, state_dict=synth_osnet_state(4321))
    v_ext = FeatureExtractor("resnet101", image_size=(128, 256), batch=32, state_dict=synth_resnet101_reid_state(2468))
    tracks = scene(a.frames, a.persons, a.vehicles)
    make = frame_source(tracks, a.frames)
    frames = [make(f) for f in range(a.frames)]
    tmp = tempfile.mkdtemp()
    pf = ri.write_track_file(os.path.join(tmp, "p.txt"), rows_of(tracks, "p"))
    vf = ri.write_track_file(os.path.join(tmp, "v.txt"), rows_of(tracks, "v"))
    thr = 2.0

    def run_gpu():
        _, pd, pc = relink.preprocess(pf, 10, 0.5, 0.5)
        _, vd, vc = relink.preprocess(vf, 10, 0.5, 0.5)
        it = ([[(frames[f], 1.0, f)] for f in range(a.frames)], a.frames)
        out = relink.reid(it, p_ext, v_ext, pd, pc, vd, vc, a.box_num, a.box_gap, thr, "min_all")
        torch.cuda.synchronize()
        return out, pc, vc

    def run_ref():
        _, pd, pc = relink.preprocess(pf, 10, 0.5, 0.5)
        _, vd, vc = relink.preprocess(vf, 10, 0.5, 0.5)
        return reference_loop(frames, p_ext, v_ext, pd, pc, vd, vc, a.box_num, a.box_gap, thr), pc, vc

    (gp, gv), gpc, gvc = run_gpu()
    (rp, rv), rpc, rvc = run_ref()
    merges = lambda d: sorted((float(k), len(v)) for k, v in d.items())
    assert merges(gp) == merges(rp) and merges(gv) == merges(rv), "the two paths merge differently"
    n_pairs = sum(len(v) for v in gpc.values()) + sum(len(v) for v in gvc.values())
    t_gpu, t_ref = [], []
    for _ in range(a.repeat):                       # alternate the two paths
        t0 = time.perf_counter()
        run_gpu()
        t_gpu.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        run_ref()
        t_ref.append(time.perf_counter() - t0)
    print(json.dumps({"bench": "relink", "gpu": gpu_info(), "frames": a.frames, "size": [H, W],
                      "tracks": [a.persons, a.vehicles], "compared_pairs": n_pairs,
                      "merged_tracks": [a.persons - len(gp), a.vehicles - len(gv)],
                      "gpu_reid_s_median": float(np.median(t_gpu)), "reference_loop_s_median": float(np.median(t_ref)),
                      "speedup": float(np.median(t_ref) / np.median(t_gpu)), "gpu_reid_s": t_gpu,
                      "reference_loop_s": t_ref}))


if __name__ == "__main__":
    main()
