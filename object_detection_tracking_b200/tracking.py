"""GPU drop-in for the DeepSORT appearance metric.

`GpuNearestNeighborDistanceMetric` has the constructor, attributes and methods of the reference's
`deep_sort.nn_matching.NearestNeighborDistanceMetric` (deep_sort/nn_matching.py:99-177), so
`Tracker(metric)` (deep_sort/tracker.py:40-48, obj_detect_tracking.py:553-558) takes it unchanged.
`distance()` replaces the per-track Python loop of tiny NumPy GEMMs (:174-177) by ONE tensor-core GEMM
over the concatenated galleries plus a segmented row-min (b2_cosine_cost; the 'euclidean' metric of the same class,
nn_matching.py:57-75, runs as b2_track_pair_cost).  No CPU fallback.
"""
from __future__ import annotations

import numpy as np

from .engine import cosine_cost


class GpuNearestNeighborDistanceMetric(object):
    def __init__(self, metric, matching_threshold, budget=None, device=0, precision="split"):
        if metric not in ("cosine", "euclidean"):
            raise ValueError("Invalid metric; must be either 'euclidean' or 'cosine'")       # nn_matching.py:123-129
        self.metric = metric
        self.matching_threshold = matching_threshold
        self.budget = budget
        self.samples = {}
        self.device = device
        self.precision = precision

    def partial_fit(self, features, targets, active_targets):
        """deep_sort/nn_matching.py:137-154 (host bookkeeping, unchanged semantics)."""
        for feature, target in zip(features, targets):
            self.samples.setdefault(target, []).append(feature)
            if self.budget is not None:
                self.samples[target] = self.samples[target][-self.budget:]
        self.samples = {k: self.samples[k] for k in active_targets}

    def distance(self, features, targets):
        """Returns the float64 [len(targets), len(features)] cost matrix of :156-177."""
        T, N = len(targets), len(features)
        cost = np.zeros((T, N))
        if T == 0 or N == 0:
            return cost
        feats = np.asarray(features, dtype=np.float32)
        seg = np.zeros(T + 1, dtype=np.int32)
        rows = []
        for i, t in enumerate(targets):
            g = np.asarray(self.samples[t], dtype=np.float32).reshape(-1, feats.shape[1])
            rows.append(g)
            seg[i + 1] = seg[i] + g.shape[0]
        gallery = np.concatenate(rows, axis=0)
        if self.metric == "cosine":
            cost[:, :] = cosine_cost(gallery, seg, feats, device=self.device, precision=self.precision)
        else:
            cost[:, :] = euclidean_cost(gallery, seg, feats, device=self.device, precision=self.precision)
        return cost


def euclidean_cost(gallery, seg, feats, device=0, precision="split"):
    """_nn_euclidean_distance (nn_matching.py:57-75) for every (track, detection): min over the track's gallery rows of
    the squared distance, clamped at 0 -- the track-pair cost with every detection as a one-row segment (one GEMM +
    segmented min on the GPU).  float32 [T, N]."""
    from . import _lib
    gallery = np.ascontiguousarray(gallery, dtype=np.float32)
    feats = np.ascontiguousarray(feats, dtype=np.float32)
    seg = np.ascontiguousarray(seg, dtype=np.int32)
    T, N = len(seg) - 1, len(feats)
    det_seg = np.arange(N + 1, dtype=np.int32)
    out = np.zeros((T, N), dtype=np.float32)
    _lib.check(_lib.load().b2_track_pair_cost(int(device), _lib.ptr(gallery), _lib.ptr(seg), T, _lib.ptr(feats),
                                              _lib.ptr(det_seg), N, feats.shape[1], None, 0.0,
                                              {"fp16": 0, "split": 1}[precision], _lib.ptr(out)),
               "b2_track_pair_cost")
    return out


def _metric_kind(metric):
    """'cosine' / 'euclidean' of a NearestNeighborDistanceMetric-like object: ours carries `.metric`, the reference's
    class only keeps the chosen function in `._metric` (nn_matching.py:123-129)."""
    kind = getattr(metric, "metric", None)
    if kind is None:
        fn = getattr(metric, "_metric", None)
        name = getattr(fn, "__name__", "")
        kind = "euclidean" if "euclid" in name else "cosine"
    if kind not in ("cosine", "euclidean"):
        raise ValueError("Invalid metric; must be either 'euclidean' or 'cosine'")
    return kind


# ----------------------------------------------------------------------------------------------------------------
# Native association loop (SURVEY 8f rank 2): same surface as deep_sort.tracker.Tracker / deep_sort.track.Track.
# ----------------------------------------------------------------------------------------------------------------
import ctypes  # noqa: E402

from . import _lib  # noqa: E402


class TrackState(object):            # deep_sort/track.py:5-16
    Tentative = 1
    Confirmed = 2
    Deleted = 3


class Track(object):
    """Read-only view of one live track of the native tracker (deep_sort/track.py:19-166 attribute names)."""

    __slots__ = ("mean", "covariance", "track_id", "hits", "age", "time_since_update", "state")

    def __init__(self, mean, covariance, track_id, hits, age, time_since_update, state):
        self.mean, self.covariance, self.track_id = mean, covariance, track_id
        self.hits, self.age, self.time_since_update, self.state = hits, age, time_since_update, state

    def to_tlwh(self):
        ret = self.mean[:4].copy()
        ret[2] *= ret[3]
        ret[:2] -= ret[2:] / 2
        return ret

    def to_tlbr(self):
        ret = self.to_tlwh()
        ret[2:] = ret[:2] + ret[2:]
        return ret

    def is_tentative(self):
        return self.state == TrackState.Tentative

    def is_confirmed(self):
        return self.state == TrackState.Confirmed

    def is_deleted(self):
        return self.state == TrackState.Deleted


_COST_FN = ctypes.CFUNCTYPE(ctypes.c_int, ctypes.c_void_p, ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_int32),
                            ctypes.c_int, ctypes.POINTER(ctypes.c_float), ctypes.c_int, ctypes.c_int,
                            ctypes.POINTER(ctypes.c_float))


class Tracker(object):
    """Drop-in for deep_sort.tracker.Tracker (tracker.py:10-138): `Tracker(metric, max_iou_distance, max_age, n_init)`,
    `predict()`, `update(detections)`, `.tracks`.  The whole association step (Kalman filter in float64, matching cascade,
    IoU matching, linear assignment, track management, gallery bookkeeping) runs in libb200det (csrc/tracker.cpp); the
    appearance cost matrices come from b2_cosine_cost on the GPU.

    `metric` supplies the parameters exactly as in the reference: an object with `matching_threshold` and `budget`
    (nn_matching.NearestNeighborDistanceMetric or GpuNearestNeighborDistanceMetric); its own sample store is not used --
    the native tracker keeps the per-track galleries.  `cost_fn(gallery, seg_offsets, dets) -> [T,N]` replaces the GPU
    appearance cost (tests pass the CPU oracle there); without it an H100 is required.
    Detections need `.tlwh`, `.confidence`, `.feature` (deep_sort/detection.py:27-42)."""

    def __init__(self, metric, max_iou_distance=0.5, max_age=60, n_init=1, device=0, precision="split", cost_fn=None):
        self.metric = metric
        self.max_iou_distance, self.max_age, self.n_init = max_iou_distance, max_age, n_init
        self.device = getattr(metric, "device", device)
        self._precision = {"fp16": 0, "split": 1}[getattr(metric, "precision", precision)]
        self._lib = _lib.load()
        self._h = None
        self._dim = None
        self._user_cost = cost_fn
        if cost_fn is None and _metric_kind(metric) == "euclidean":
            # the reference Tracker asks metric.distance() (tracker.py:98-104), so the metric kind is honoured there; the
            # native cascade's built-in cost is the cosine one, the euclidean one is installed as its cost function
            dev, prec = self.device, getattr(metric, "precision", precision)
            self._user_cost = lambda gal, seg, dets: euclidean_cost(gal, seg, dets, device=dev, precision=prec)
        self._cb = None
        self._tracks = []
        self._stale = False

    @property
    def tracks(self):
        """The live tracks (deep_sort/tracker.py:38), materialised from the native state on first access after a
        predict() / update(): the drivers read them once per frame, after update() (obj_detect_tracking.py:670)."""
        if self._stale:
            self._refresh()
        return self._tracks

    def _create(self, dim):
        h = ctypes.c_void_p()
        budget = self.metric.budget if getattr(self.metric, "budget", None) is not None else 0
        _lib.check(self._lib.b2_tracker_create(ctypes.byref(h), int(self.device), float(self.max_iou_distance),
                                               int(self.max_age), int(self.n_init),
                                               float(self.metric.matching_threshold), int(budget), int(dim),
                                               self._precision), "b2_tracker_create")
        self._h, self._dim = h, dim
        if self._user_cost is not None:
            fn = self._user_cost

            def _cb(user, gal, seg, T, dets, N, D, cost):
                try:
                    seg_a = np.ctypeslib.as_array(seg, shape=(T + 1,)).copy()
                    gal_a = np.ctypeslib.as_array(gal, shape=(int(seg_a[-1]), D)).copy()
                    det_a = np.ctypeslib.as_array(dets, shape=(N, D)).copy()
                    out = np.asarray(fn(gal_a, seg_a, det_a), dtype=np.float32).reshape(T, N)
                    np.ctypeslib.as_array(cost, shape=(T, N))[:, :] = out
                    return 0
                except Exception:      # an exception must not cross the C ABI
                    return -1
            self._cb = _COST_FN(_cb)
            _lib.check(self._lib.b2_tracker_set_cost_fn(self._h, ctypes.cast(self._cb, ctypes.c_void_p), None),
                       "b2_tracker_set_cost_fn")

    def close(self):
        if self._h is not None:
            self._lib.b2_tracker_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def predict(self):
        if self._h is not None:
            _lib.check(self._lib.b2_tracker_predict(self._h), "b2_tracker_predict")
            self._stale = True

    def update(self, detections):
        n = len(detections)
        if self._h is None:
            if n == 0:
                return
            self._create(int(np.asarray(detections[0].feature).shape[-1]))
        tlwh = np.ascontiguousarray([d.tlwh for d in detections], dtype=np.float64).reshape(n, 4)
        conf = np.ascontiguousarray([d.confidence for d in detections], dtype=np.float64).reshape(n)
        feat = np.ascontiguousarray([d.feature for d in detections], dtype=np.float32).reshape(n, self._dim)
        _lib.check(self._lib.b2_tracker_update(self._h, _lib.ptr(tlwh), _lib.ptr(conf), _lib.ptr(feat), n),
                   "b2_tracker_update")
        self._stale = True

    def _refresh(self):
        n = self._lib.b2_tracker_num_tracks(self._h)
        ids, st, hits, age, tsu = (np.zeros(n, np.int32) for _ in range(5))
        mean = np.zeros((n, 8), np.float64)
        cov = np.zeros((n, 8, 8), np.float64)
        got = self._lib.b2_tracker_get_tracks(self._h, n, _lib.ptr(ids), _lib.ptr(st), _lib.ptr(hits), _lib.ptr(age),
                                              _lib.ptr(tsu), _lib.ptr(mean), _lib.ptr(cov))
        if got != n:
            _lib.check(-1, "b2_tracker_get_tracks")
        self._tracks = [Track(mean[k], cov[k], int(ids[k]), int(hits[k]), int(age[k]), int(tsu[k]), int(st[k]))
                        for k in range(n)]
        self._stale = False


def linear_sum_assignment(cost_matrix):
    """scipy.optimize.linear_sum_assignment restated natively (the solver the tracker uses; exported for the parity tests)."""
    c = np.ascontiguousarray(cost_matrix, dtype=np.float64)
    nr, nc = c.shape
    k = min(nr, nc)
    rows, cols = np.zeros(k, np.int32), np.zeros(k, np.int32)
    got = _lib.load().b2_linear_sum_assignment(_lib.ptr(c), nr, nc, _lib.ptr(rows), _lib.ptr(cols))
    if got < 0:
        _lib.check(got, "b2_linear_sum_assignment")
    return rows[:got].astype(np.int64), cols[:got].astype(np.int64)


def non_max_suppression(boxes, max_bbox_overlap, scores=None):
    """application_util/preprocessing.py:6-74 (pre-tracker NMS over tlwh boxes): kept indices in pick order."""
    boxes = np.ascontiguousarray(boxes, dtype=np.float64).reshape(-1, 4)
    n = len(boxes)
    if n == 0:
        return []
    sc = None if scores is None else np.ascontiguousarray(scores, dtype=np.float64).reshape(n)
    keep = np.zeros(n, np.int32)
    got = _lib.load().b2_track_nms(_lib.ptr(boxes), _lib.ptr(sc), n, float(max_bbox_overlap), _lib.ptr(keep))
    if got < 0:
        _lib.check(got, "b2_track_nms")
    return [int(i) for i in keep[:got]]


# ----------------------------------------------------------------------------------------------------------------
# Detector output -> tracker input (SURVEY 8a row a21): host glue of the reference drivers, vectorised.
# ----------------------------------------------------------------------------------------------------------------
class Detection(object):
    """deep_sort/detection.py:5-49: tlwh float64, confidence float, feature float32."""

    def __init__(self, tlwh, confidence, feature):
        self.tlwh = np.asarray(tlwh, dtype=np.float64)
        self.confidence = float(confidence)
        self.feature = np.asarray(feature, dtype=np.float32)

    def to_tlbr(self):
        ret = self.tlwh.copy()
        ret[2:] += ret[:2]
        return ret

    def to_xyah(self):
        ret = self.tlwh.copy()
        ret[:2] += ret[2:] / 2
        ret[2] /= ret[3]
        return ret


def _select_detections(final_boxes, final_probs, final_labels, box_feats, targetid2class, tracking_objs, min_confidence,
                       scale, is_coco_model, coco_to_actev_mapping):
    """Common body of deep_sort/utils.py:5-35 and obj_detect_tracking_multi_queuer_tmot.py:456-488: boxes / scale, class
    filter (with the COCO -> ActEV name mapping), round(prob, 7) >= min_confidence, x1y1x2y2 -> xywh in the boxes' own
    dtype, feature = mean over the 7x7 grid unless the detector already returned pooled features (feat_mode 1)."""
    boxes = np.asarray(final_boxes) / scale
    probs = np.asarray(final_probs)
    feats = np.asarray(box_feats)
    keep, confs = [], []
    for j, label in enumerate(final_labels):
        cat_name = targetid2class[label]
        if is_coco_model:
            if cat_name not in coco_to_actev_mapping:
                continue
            cat_name = coco_to_actev_mapping[cat_name]
        conf = float(round(probs[j], 7))
        if cat_name not in tracking_objs or conf < min_confidence:
            continue
        keep.append(j)
        confs.append(conf)
    keep = np.asarray(keep, dtype=np.int64)
    xywh = boxes[keep].copy() if len(keep) else np.zeros((0, 4), boxes.dtype)
    xywh[:, 2] -= xywh[:, 0]
    xywh[:, 3] -= xywh[:, 1]
    f = feats[keep] if len(keep) else np.zeros((0,) + feats.shape[1:], feats.dtype)
    if f.ndim > 2:                                   # [R, C, 7, 7] -> [R, C]
        f = np.mean(f, axis=(2, 3))
    return xywh, confs, f


def create_obj_infos(cur_frame, final_boxes, final_probs, final_labels, box_feats, targetid2class, tracking_objs,
                     min_confidence, min_detection_height, scale, is_coco_model=False, coco_to_actev_mapping=None):
    """Drop-in for deep_sort.utils.create_obj_infos (deep_sort/utils.py:5-44) -> list of Detection."""
    xywh, confs, f = _select_detections(final_boxes, final_probs, final_labels, box_feats, targetid2class, tracking_objs,
                                        min_confidence, scale, is_coco_model, coco_to_actev_mapping)
    # (the reference builds Python lists here; Detection converts to float64 / float32 arrays either way)
    return [Detection(xywh[k], confs[k], f[k]) for k in range(len(confs)) if not xywh[k, 3] < min_detection_height]


def preprocess_detections(final_boxes, final_probs, final_labels, box_feats, targetid2class, tracking_objs, min_confidence,
                          scale, is_coco_model=False, coco_to_actev_mapping=None):
    """Drop-in for the TMOT driver's preprocess_detections (obj_detect_tracking_multi_queuer_tmot.py:456-488) ->
    [(xywh, confidence, feature), ...] as JDETracker.update takes them."""
    xywh, confs, f = _select_detections(final_boxes, final_probs, final_labels, box_feats, targetid2class, tracking_objs,
                                        min_confidence, scale, is_coco_model, coco_to_actev_mapping)
    return [(xywh[k], confs[k], f[k]) for k in range(len(confs))]


# ----------------------------------------------------------------------------------------------------------------
# Per-video post-processing of the track table (deep_sort/utils.py:47-113; obj_detect_tracking.py:800-801).
# Rows are [frame, track id, x, y, w, h, ...]; host numpy, once per video -- not on the per-frame path.
# ----------------------------------------------------------------------------------------------------------------
def linear_inter_bbox(tracking_data, frame_gap):
    """deep_sort/utils.py:47-91: fills the frames a track skipped (detection runs every `frame_gap` frames) by linear
    interpolation between its neighbouring rows, rounded to 2 decimals, unless the hole is longer than 10 * frame_gap."""
    tracking_data = np.asarray(tracking_data)
    if tracking_data.shape[0] == 0:
        return tracking_data
    ids = tracking_data[:, 1].astype(np.int64)
    extra = []
    for tid in np.unique(ids):
        rows = tracking_data[ids == tid]
        frames = rows[:, 0]
        for k in range(len(rows) - 1):
            f0, f1 = frames[k], frames[k + 1]
            if f1 - f0 <= 1 or f1 - f0 > 10 * frame_gap:
                continue
            missing = np.arange(int(f0) + 1, int(np.ceil(f1)))
            missing = missing[(missing > f0) & (missing < f1)]
            if not len(missing):
                continue
            ratio = (missing - f0) / (f1 - f0)
            vals = np.around(rows[k, 2:][None, :] + (rows[k + 1, 2:] - rows[k, 2:])[None, :] * ratio[:, None], decimals=2)
            extra.append(np.concatenate([missing[:, None].astype(np.float64), np.full((len(missing), 1), float(tid)), vals], 1))
    if extra:
        tracking_data = np.concatenate([tracking_data] + extra, axis=0)
    order = np.lexsort((tracking_data[:, 1], tracking_data[:, 0]))
    return tracking_data[order]


def filter_short_objs(tracking_data):
    """deep_sort/utils.py:94-113: drops tracks with fewer than two rows; rows sorted by (frame, id)."""
    tracking_data = np.asarray(tracking_data)
    if tracking_data.shape[0] == 0:
        return tracking_data
    ids = tracking_data[:, 1].astype(np.int64)
    uniq, counts = np.unique(ids, return_counts=True)
    keep = np.isin(ids, uniq[counts >= 2])
    out = tracking_data[keep]
    return out[np.lexsort((out[:, 1], out[:, 0]))]
