"""Drop-ins for the reference's TMOT tracker (tmot/multitracker.py, tmot/matching.py) over libb200det's native
association code (csrc/tmot.cpp).  The per-frame embedding distance is one tensor-core GEMM on the GPU; everything else is
float64 host code, as in the reference.  No CPU fallback for the embedding distance: without an H100 only the `cost_fn` hook
(used by the CPU parity tests with the oracle) can supply it."""
from __future__ import annotations

import ctypes
import weakref

import numpy as np

from . import _lib
from .tracking import _COST_FN


class TrackState(object):          # tmot/basetrack.py:5-9
    New, Tracked, Lost, Removed = 0, 1, 2, 3


class STrack(object):
    """Read-only view of one track after JDETracker.update (multitracker.py:13-174: the attributes the drivers read,
    obj_detect_tracking_multi_queuer_tmot.py:572-582)."""
    __slots__ = ("track_id", "state", "is_activated", "frame_id", "start_frame", "tracklet_len", "tlwh", "cur_det_tlwh",
                 "cur_det_conf", "score", "mean", "covariance")

    def __init__(self, **kw):
        for k, v in kw.items():
            setattr(self, k, v)

    @property
    def end_frame(self):
        return self.frame_id

    @property
    def tlbr(self):
        r = self.tlwh.copy()
        r[2:] += r[:2]
        return r

    def __repr__(self):
        return "OT_{}_({}-{})".format(self.track_id, self.start_frame, self.end_frame)


class _IdGroup(object):
    """BaseTrack._count is a class attribute: every JDETracker of the process draws ids from one counter and reset()
    zeroes it (basetrack.py:13,34-37; multitracker.py:215).  Trackers created with the same group share a native counter."""

    def __init__(self):
        self.members = []          # weak references to the trackers of the group that own a native handle

    def live_handle(self):
        self.members = [w for w in self.members if w() is not None and w()._h is not None]
        return self.members[0]()._h if self.members else None


_DEFAULT_GROUP = _IdGroup()


class JDETracker(object):
    """Drop-in for tmot.multitracker.JDETracker (multitracker.py:176-358): same constructor, `update(detections)` with
    detections = [(tlwh, conf, feature), ...] and the list of activated tracks as the result, `reset()`."""

    def __init__(self, conf_thres, track_max_second_lost=4.0, emb_max_dist=0.7, iou_max_dist1=0.8, iou_max_dist2=0.9,
                 emb_smooth_alpha=0.9, frame_gap=8., frame_rate=30., device=0, precision="split", cost_fn=None,
                 id_group=_DEFAULT_GROUP):
        self._args = (float(conf_thres), float(track_max_second_lost), float(emb_max_dist), float(iou_max_dist1),
                      float(iou_max_dist2), float(emb_smooth_alpha), float(frame_gap), float(frame_rate))
        self.device = device
        self._precision = {"fp16": 0, "split": 1}[precision]
        self._lib = _lib.load()
        self._h = None
        self._dim = None
        self._user_cost = cost_fn
        self._cb = None
        self._group = id_group
        self.frame_id = 0

    def _create(self, dim):
        h = ctypes.c_void_p()
        _lib.check(self._lib.b2_jde_create(ctypes.byref(h), int(self.device), *self._args, int(dim), self._precision,
                                           self._group.live_handle()), "b2_jde_create")
        self._h, self._dim = h, dim
        self._group.members.append(weakref.ref(self))
        if self._user_cost is not None:
            fn = self._user_cost

            def _cb(user, gal, seg, T, dets, N, D, cost):
                try:
                    a = np.ctypeslib.as_array(gal, shape=(T, D)).copy()
                    b = np.ctypeslib.as_array(dets, shape=(N, D)).copy()
                    np.ctypeslib.as_array(cost, shape=(T, N))[:, :] = np.asarray(fn(a, b), dtype=np.float32).reshape(T, N)
                    return 0
                except Exception:      # an exception must not cross the C ABI
                    return -1
            self._cb = _COST_FN(_cb)
            _lib.check(self._lib.b2_jde_set_cost_fn(self._h, ctypes.cast(self._cb, ctypes.c_void_p), None),
                       "b2_jde_set_cost_fn")

    def close(self):
        if self._h is not None:
            self._lib.b2_jde_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def reset(self):
        """multitracker.py:206-215: clears this tracker's lists and ALWAYS zeroes the id counter of the whole process
        (BaseTrack._count = 0) -- also when this tracker has not seen a detection yet and owns no native state."""
        self.frame_id = 0
        if self._h is not None:
            _lib.check(self._lib.b2_jde_reset(self._h), "b2_jde_reset")
        else:
            h = self._group.live_handle()
            if h is not None:
                _lib.check(self._lib.b2_jde_reset_ids(h), "b2_jde_reset_ids")

    def update(self, detections):
        n = len(detections)
        self.frame_id += 1
        if self._h is None:
            if n == 0:
                return []
            self._create(int(np.asarray(detections[0][2]).shape[-1]))
            for _ in range(self.frame_id - 1):       # frames that had no detection before the first one
                self._lib.b2_jde_update(self._h, None, None, None, 0)
        tlwh = np.ascontiguousarray([d[0] for d in detections], dtype=np.float64).reshape(n, 4)
        conf = np.ascontiguousarray([d[1] for d in detections], dtype=np.float64).reshape(n)
        feat = np.ascontiguousarray([d[2] for d in detections], dtype=np.float32).reshape(n, self._dim)
        got = self._lib.b2_jde_update(self._h, _lib.ptr(tlwh), _lib.ptr(conf), _lib.ptr(feat), n)
        if got < 0:
            _lib.check(got, "b2_jde_update")
        return self.get_tracks(0, full=False)

    def get_tracks(self, which=0, full=True):
        """which: 0 = the list update() returns, 1 = tracked_stracks, 2 = lost_stracks.  full=False skips the Kalman
        state (mean / covariance stay None): what the drivers read per frame is the id, the boxes and the confidence."""
        if self._h is None:
            return []
        n = self._lib.b2_jde_get_tracks(self._h, which, 0, *([None] * 12))
        if n == 0:
            return []
        ints = np.zeros((6, n), np.int32)                       # ids, state, is_activated, frame_id, start_frame, tracklet_len
        tlwh, dtlwh = np.zeros((n, 4)), np.zeros((n, 4))
        dconf, score = np.zeros(n), np.zeros(n)
        mean, cov = (np.zeros((n, 8)), np.zeros((n, 8, 8))) if full else (None, None)
        got = self._lib.b2_jde_get_tracks(self._h, which, n, *[_lib.ptr(a) for a in (ints[0], ints[1], ints[2], ints[3], ints[4],
                                                                                     ints[5], tlwh, dtlwh, dconf, score, mean, cov)])
        if got != n:
            _lib.check(-1, "b2_jde_get_tracks")
        ids, st, act, fid, sf, tl = ints.tolist()
        dconf_l, score_l = dconf.tolist(), score.tolist()
        # the arrays are fresh per call, so row views do not alias anything that outlives this list
        return [STrack(track_id=ids[k], state=st[k], is_activated=bool(act[k]), frame_id=fid[k], start_frame=sf[k],
                       tracklet_len=tl[k], tlwh=tlwh[k], cur_det_tlwh=dtlwh[k], cur_det_conf=dconf_l[k], score=score_l[k],
                       mean=mean[k] if full else None, covariance=cov[k] if full else None)
                for k in range(n)]

    @property
    def tracked_stracks(self):
        return self.get_tracks(1)

    @property
    def lost_stracks(self):
        return self.get_tracks(2)


# ---- tmot/matching.py ---------------------------------------------------------------------------------------------

def lapjv(cost, extend_cost=True, cost_limit=np.inf):
    """lap.lapjv(cost, extend_cost=True, cost_limit=...) as the reference calls it (matching.py:32, multi_video_reid.py:512):
    (matched cost, x, y) with -1 for unmatched rows / columns."""
    c = np.ascontiguousarray(cost, dtype=np.float64)
    if c.ndim != 2:
        raise ValueError("2-dimensional array expected")
    if not np.isfinite(cost_limit):
        raise NotImplementedError("only the cost_limit form the reference uses is provided")
    nr, nc = c.shape
    x, y = np.zeros(nr, np.int32), np.zeros(nc, np.int32)
    opt = ctypes.c_double(0)
    _lib.check(_lib.load().b2_lapjv(_lib.ptr(c), nr, nc, float(cost_limit), _lib.ptr(x), _lib.ptr(y), ctypes.byref(opt)),
               "b2_lapjv")
    return opt.value, x.astype(np.int64), y.astype(np.int64)


def linear_assignment(cost_matrix, thresh):          # matching.py:28-38
    cost_matrix = np.asarray(cost_matrix, dtype=np.float64)
    if cost_matrix.size == 0:
        return np.empty((0, 2), dtype=int), tuple(range(cost_matrix.shape[0])), tuple(range(cost_matrix.shape[1]))
    _, x, y = lapjv(cost_matrix, extend_cost=True, cost_limit=thresh)
    matches = np.asarray([[ix, mx] for ix, mx in enumerate(x) if mx >= 0])
    return matches, np.where(x < 0)[0], np.where(y < 0)[0]


def _tlbrs(tracks):
    if len(tracks) > 0 and not isinstance(tracks[0], np.ndarray):
        tracks = [t.tlbr for t in tracks]
    return np.ascontiguousarray(tracks, dtype=np.float64).reshape(-1, 4)


def iou_distance(atracks, btracks):                  # matching.py:57-77
    a, b = _tlbrs(atracks), _tlbrs(btracks)
    out = np.zeros((len(a), len(b)), dtype=np.float64)
    if out.size:
        _lib.check(_lib.load().b2_tmot_iou_distance(_lib.ptr(a), len(a), _lib.ptr(b), len(b), _lib.ptr(out)),
                   "b2_tmot_iou_distance")
    return out


def embedding_distance(track_features, det_features, device=0, precision="split"):     # matching.py:80-94
    """Euclidean distances between [T,D] smoothed track embeddings and [N,D] detection embeddings (float64 [T,N])."""
    a = np.ascontiguousarray(track_features, dtype=np.float32)
    b = np.ascontiguousarray(det_features, dtype=np.float32)
    T = a.shape[0] if a.ndim == 2 else 0
    N = b.shape[0] if b.ndim == 2 else 0
    out = np.zeros((T, N), dtype=np.float64)
    if out.size:
        _lib.check(_lib.load().b2_tmot_embedding_distance(int(device), _lib.ptr(a), T, _lib.ptr(b), N, a.shape[1],
                                                          {"fp16": 0, "split": 1}[precision], _lib.ptr(out)),
                   "b2_tmot_embedding_distance")
    return out


def fuse_motion(means, covariances, cost_matrix, measurements_xyah, only_position=False, lambda_=0.98):   # matching.py:97-109
    """In the reference's argument order minus the Kalman filter object: track means [T,8] / covariances [T,8,8], the
    cost matrix [T,N] and the detections' (x, y, a, h) [N,4]."""
    cost = np.array(cost_matrix, dtype=np.float64, order="C")
    if cost.size == 0:
        return cost
    m = np.ascontiguousarray(means, dtype=np.float64).reshape(-1, 8)
    c = np.ascontiguousarray(covariances, dtype=np.float64).reshape(-1, 64)
    z = np.ascontiguousarray(measurements_xyah, dtype=np.float64).reshape(-1, 4)
    _lib.check(_lib.load().b2_tmot_fuse_motion(_lib.ptr(m), _lib.ptr(c), len(m), _lib.ptr(z), len(z), _lib.ptr(cost),
                                               int(bool(only_position)), float(lambda_)), "b2_tmot_fuse_motion")
    return cost
