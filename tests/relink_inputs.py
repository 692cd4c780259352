"""The synthetic video of the tracklet re-linking tests (tests/golden/make_golden_relink.py, test_relink_cpu.py,
test_relink_gpu.py): 40 frames of 240x320 built with integer arithmetic only, so that every test regenerates them
bit for bit instead of storing them, and the person / vehicle MOT track tables painted into them.

Each identity has a blocky sprite (an integer hash per 4x4 block and channel) that is pasted, nearest-neighbour, into
each of its boxes: crops of one identity are close in feature space and different identities are far apart.

Person tracks (tol_num_frame 10, expand 0.5 / 0.5), one scenario per cell:
  1 -> 2 -> 3        one identity, gaps of 4 frames: a merge chain (3 merges into 1 through 2)
  4, 5 -> 6          two queries claim gallery 6; the longer query (4) wins
  7 -> 8             different identities: the distance is above the threshold (7 and 8 are vehicle ids too)
  9 -> 10            every box of query 9 leaves the frame: the query is removed
  11 -> 12, 13       gallery 12's boxes are too small (area <= 10): dropped from 11's list, 11 merges with 13
  14 -> 15           the only gallery has no valid crop: query 14 is removed
  16 -> 17, 18, 19   17 (start 19) is found first; 18 starts earlier (18) but is dropped; 19 shares 17's start
  20, 21             21's first box touches 20's expanded last box: no candidate
  22, 23             23 starts exactly tol frames after 22 ends: no candidate
  24, 25 -> 26       two queries of equal length claim 26: the first (24) wins
Vehicle tracks: 7 -> 8 (one identity, but the reference's crop keys are shared with persons 7 and 8), 30 -> 31 (merge),
32 -> 33 (different identities).
"""
import os

import numpy as np

H, W, NUM_FRAMES = 240, 320, 40
TOL, EXPAND_W, EXPAND_H = 10, 0.5, 0.5


def _cell(k):
    return (k % 6) * 53 + 16, 40 + (k // 6) * 80


def _tracks():
    """[(class, track id, identity, first frame, last frame, x, y, w, h)]"""
    t = []
    x, y = _cell(0)
    t += [("p", 1, 1, 0, 9, x, y, 16, 40), ("p", 2, 1, 13, 22, x, y, 16, 42), ("p", 3, 1, 26, 35, x + 2, y, 17, 40)]
    x, y = _cell(1)
    t += [("p", 4, 2, 0, 11, x, y, 16, 40), ("p", 5, 2, 3, 11, x + 14, y, 16, 40), ("p", 6, 2, 14, 25, x + 8, y, 16, 42)]
    x, y = _cell(2)
    t += [("p", 7, 3, 0, 9, x, y, 16, 40), ("p", 8, 4, 12, 20, x, y, 16, 40)]
    x, y = _cell(6)
    t += [("p", 9, 5, 0, 9, -6, y, 16, 40), ("p", 10, 5, 12, 20, 2, y, 16, 40)]
    x, y = _cell(7)
    t += [("p", 11, 6, 0, 9, x, y, 16, 40), ("p", 12, 6, 12, 20, x - 3, y - 8, 2, 4), ("p", 13, 6, 12, 22, x, y, 16, 41)]
    x, y = _cell(3)
    t += [("p", 14, 7, 0, 9, x, y, 16, 40), ("p", 15, 7, 12, 20, x + 2, y + 2, 3, 3)]
    x, y = _cell(4)
    t += [("p", 16, 8, 0, 15, x, y, 16, 40), ("p", 17, 8, 19, 30, x, y, 16, 41), ("p", 18, 8, 18, 30, x + 16, y + 20, 16, 40),
          ("p", 19, 9, 19, 30, x - 16, y - 31, 16, 40)]
    x, y = _cell(8)
    t += [("p", 20, 10, 0, 9, x, y, 16, 40), ("p", 21, 10, 12, 20, x + 20, y, 16, 40)]
    x, y = _cell(9)
    t += [("p", 22, 11, 0, 9, x, y, 16, 40), ("p", 23, 11, 19, 27, x, y, 16, 40)]
    x, y = _cell(10)
    t += [("p", 24, 12, 0, 9, x, y, 16, 40), ("p", 25, 12, 0, 9, x + 14, y, 16, 40), ("p", 26, 12, 12, 21, x + 8, y, 16, 42)]
    t += [("v", 7, 101, 0, 9, 10, 195, 60, 30), ("v", 8, 101, 12, 22, 12, 195, 60, 30),
          ("v", 30, 102, 0, 11, 110, 195, 60, 30), ("v", 31, 102, 14, 25, 112, 196, 62, 30),
          ("v", 32, 103, 0, 9, 210, 195, 60, 30), ("v", 33, 104, 12, 20, 212, 195, 60, 30)]
    return t


def _height(w, h, f, tid):
    """Box heights vary by 0-2 pixels from frame to frame (not for the too-small boxes), so that one track's crops differ."""
    return h if w < 4 else h + (5 * f + tid) % 3


def track_rows(cls):
    """MOT rows [frame, id, left, top, width, height, conf] of one class ("p" / "v"), sorted by (frame, id)."""
    rows = []
    for c, tid, _, f0, f1, x, y, w, h in _tracks():
        if c == cls:
            rows += [(f, tid, x, y, w, _height(w, h, f, tid), 0.5 + 0.01 * ((f * 7 + tid) % 50)) for f in range(f0, f1 + 1)]
    return sorted(rows)


def write_track_file(path, rows):
    d = os.path.dirname(path)
    if d and not os.path.exists(d):
        os.makedirs(d)
    with open(path, "w") as f:
        for r in rows:
            f.write("%d,%d,%g,%g,%g,%g,%.4f,-1,-1,-1\n" % tuple(r))
    return path


def _hash(k, by, bx, c):
    v = (k * 2654435761 + by * 40503 + bx * 9973 + c * 65599) & 0xFFFFFFFF
    v ^= v >> 13
    v = (v * 1274126177) & 0xFFFFFFFF
    return (v >> 16) & 0xFF


def sprite(identity, h=48, w=24):
    """uint8 BGR sprite of one identity: 4x4 blocks of hashed colours."""
    s = np.empty((h, w, 3), np.uint8)
    for by in range(h // 4):
        for bx in range(w // 4):
            for c in range(3):
                s[by * 4:by * 4 + 4, bx * 4:bx * 4 + 4, c] = _hash(identity, by, bx, c)
    return s


def paint(frame, spr, x, y, w, h):
    """Pastes `spr` nearest-neighbour into the box (x, y, w, h) of `frame`, clipped to the frame (integer arithmetic)."""
    Hf, Wf = frame.shape[:2]
    sh, sw = spr.shape[:2]
    ys = np.arange(max(y, 0), min(y + h, Hf))
    xs = np.arange(max(x, 0), min(x + w, Wf))
    if ys.size and xs.size:
        frame[ys[:, None], xs[None, :]] = spr[((ys - y) * sh // h)[:, None], ((xs - x) * sw // w)[None, :]]


def background(h, w):
    yy, xx = np.mgrid[0:h, 0:w]
    return np.stack([(3 * xx + 2 * yy + 50 * c) % 256 for c in range(3)], -1).astype(np.uint8)


def frames():
    """[NUM_FRAMES, H, W, 3] uint8 BGR."""
    bg = background(H, W)
    sprites = {}
    out = np.empty((NUM_FRAMES, H, W, 3), np.uint8)
    tracks = _tracks()
    for f in range(NUM_FRAMES):
        out[f] = bg
        for c, tid, ident, f0, f1, x, y, w, h in tracks:
            if f0 <= f <= f1:
                if ident not in sprites:
                    sprites[ident] = sprite(ident, 48, 24) if c == "p" else sprite(ident, 24, 48)
                paint(out[f], sprites[ident], x, y, w, _height(w, h, f, tid))
    return out


def frame_iter(video, order=None):
    """The reference's (batches, count) pair: batch[0] = (image, scale, frame_idx)."""
    order = range(len(video)) if order is None else order
    return ([[(video[f], 1.0, f)] for f in order], len(order))


# The parameter sets of the golden runs: (feature_box_num, feature_box_gap, compare_method); reject_dist_thres per method
RUNS = [(5, 3, "min_all"), (-1, 4, "min_all"), (4, 2, "avg")]
THRESHOLD = {"min_all": 2.0, "avg": 2.0}
