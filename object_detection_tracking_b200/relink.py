"""GPU drop-in for the reference's single-video tracklet re-linking (single_video_reid.py): `preprocess` finds the
tracklets one object may have left and re-entered, `reid` compares their crops with the person / vehicle ReID extractors
and merges the matches into one track id, `save_new_track` writes the merged MOT file.

What runs where:
  * the candidate search is vectorised numpy over the float32 track table (the reference loops over all track pairs);
  * the crops are resized and embedded on the GPU (ReidEngine.embed_boxes_dev, Pillow-exact), once per needed box and
    class, into a per-class float32 CUDA table that never visits the host; only the crops' pixels are uploaded;
  * every candidate pair of a class is scored by one b2_tracklet_dist_dev call (one GEMM + one pair kernel) on rows
    compacted from that table;
  * the merge decisions are the reference's own list / dict logic on the host.
The reference's quirks are kept on purpose (DESIGN.md section 4, "Tracklet re-linking"): the "first-found" candidate
rule, the query / gallery crop keys the two classes share, the in-place mutation of `candidates` and of the caller's
track arrays, and its errors.  No CPU fallback: a missing library or GPU raises.
"""
from __future__ import annotations

import operator
import os
from ctypes import c_void_p

import numpy as np

from . import _lib

METHODS = {"min_all": 0, "avg": 1}


# ---- utils.py:44-57, 148-180, with the reference's dtypes ----------------------------------------------------------
def valid_box(tlwh, img, min_area=10):
    """utils.py:44-57."""
    x, y, w, h = tlwh
    area = w * h
    height, width, _ = img.shape
    return bool(x >= 0 and y >= 0 and w >= 0 and h >= 0 and x <= width and y <= height and x + w <= width
                and y + h <= height and area > min_area)


def _expand_tlwh(L, T, W, H, w_p, h_p):
    """utils.py:172-180 on float32 columns.  Under NumPy 2 (NEP 50) a Python float meets a float32 scalar as float32, so
    each product below is a float32 operation, in the reference's order."""
    return (L - W * np.float32(w_p) * np.float32(0.5), T - H * np.float32(h_p) * np.float32(0.5),
            W * np.float32(1. + w_p), H * np.float32(1. + h_p))


def _intersection_positive(e, L2, T2, W2, H2):
    """tlwh_intersection(e, tlwh2) > 0 (utils.py:148-169) for one expanded box `e` against float32 columns."""
    l1, t1, w1, h1 = e
    xx1 = np.maximum(l1, L2)
    yy1 = np.maximum(t1, T2)
    xx2 = np.minimum(l1 + w1, L2 + W2)
    yy2 = np.minimum(t1 + h1, T2 + H2)
    w = np.maximum(np.float32(0), xx2 - xx1)
    h = np.maximum(np.float32(0), yy2 - yy1)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        return (w * h) / (W2 * H2) > 0


# ---- single_video_reid.py:68-138 ---------------------------------------------------------------------------------
def read_tracks(track_file):
    """The MOT rows of `track_file` as float32 [N, 7] (frame, id, left, top, width, height, conf), or None if empty."""
    data = []
    with open(track_file, "r") as f:
        for line in f:
            frame_idx, track_id, left, top, width, height, conf, _, _, _ = line.strip().split(",")
            data.append([frame_idx, track_id, left, top, width, height, conf])
    if not data:
        return None
    return np.array(data, dtype="float32")


def preprocess(track_file, tol_num_frame=30, expand_width_p=0.1, expand_height_p=0.1, reject_track_conf_thres=-1):
    """single_video_reid.py:68-138 -> (ori_track_num, track_data {id: float32 [K, 7]}, possible_pairs {id: [[id2,
    start2, end1], ...]}), the same pairs in the same order.  A candidate needs start2 > end1, start2 - end1 < tol and a
    positive intersection of the query's expanded last box with the candidate's first box; after a track's first
    candidate only those starting on that candidate's frame are kept."""
    data = read_tracks(track_file)
    if data is None:
        return 0, [], {}
    track_ids = np.unique(data[:, 1]).tolist()
    track_data = {}
    for track_id in track_ids:
        track_data[track_id] = data[data[:, 1] == track_id, :]
    ori_track_num = len(track_data)
    if reject_track_conf_thres > 0.:
        good_track_ids = [t for t in track_data if np.mean(track_data[t][:, 6]) > reject_track_conf_thres]
        track_data = {track_data[t] for t in good_track_ids}      # :97 -- a set of arrays: TypeError (unhashable)
        track_data[track_ids[0]]                                  # no good track: the search's subscript fails
    n = len(track_ids)
    first = np.stack([track_data[t][0] for t in track_ids])      # [n, 7]
    last = np.stack([track_data[t][-1] for t in track_ids])
    S, E = first[:, 0], last[:, 0]
    ex = _expand_tlwh(last[:, 2], last[:, 3], last[:, 4], last[:, 5], expand_width_p, expand_height_p)
    possible_pairs = {}
    for i in range(n - 1):
        j = np.arange(i + 1, n)
        s2 = S[i + 1:]
        ok = (s2 > E[i]) & ((s2 - E[i]) < tol_num_frame)
        j, s2 = j[ok], s2[ok]
        if j.size == 0:
            continue
        f = first[j]
        ok = _intersection_positive(tuple(c[i] for c in ex), f[:, 2], f[:, 3], f[:, 4], f[:, 5])
        j, s2 = j[ok], s2[ok]
        if j.size == 0:
            continue
        keep = s2 == s2[0]                                       # :131-136, the first-found candidate's start
        possible_pairs[track_ids[i]] = [[track_ids[k], S[k], E[i]] for k in j[keep]]
    return ori_track_num, track_data, possible_pairs


# ---- single_video_reid.py:156-206 ---------------------------------------------------------------------------------
def plan_boxes(needed_track_boxes, track_data, candidates, feature_box_num, feature_box_gap):
    """get_track_boxes (:156-194): the last boxes of each query and the first of each gallery, every feature_box_gap-th,
    at most feature_box_num (<= 0: no limit).  Keys are "query_<id>" / "gallery_<id>" in one dict for both classes: a
    query key is planned again by every class that lists it, a gallery key only by the first."""
    for query_track_id in candidates:
        query_key = "query_%s" % query_track_id
        needed_track_boxes[query_key] = []
        rows = track_data[query_track_id]
        limit = len(rows) if feature_box_num <= 0 else feature_box_num
        idx = 1
        while idx <= len(rows) and len(needed_track_boxes[query_key]) < limit:
            needed_track_boxes[query_key].append(rows[-idx])
            idx += feature_box_gap
        for gallery_track_id, _, _ in candidates[query_track_id]:
            gallery_key = "gallery_%s" % gallery_track_id
            if gallery_key in needed_track_boxes:
                continue
            needed_track_boxes[gallery_key] = []
            rows = track_data[gallery_track_id]
            limit = len(rows) if feature_box_num <= 0 else feature_box_num
            idx = 0
            while idx < len(rows) and len(needed_track_boxes[gallery_key]) < limit:
                needed_track_boxes[gallery_key].append(rows[idx])
                idx += feature_box_gap
    return needed_track_boxes


def _class_keys(candidates):
    keys = set()
    for q in candidates:
        keys.add("query_%s" % q)
        for g, _, _ in candidates[q]:
            keys.add("gallery_%s" % g)
    return keys


class _FeatureTable(object):
    """One class's crop features on the GPU: rows appended in embedding order to a float32 CUDA tensor (grown by
    doubling), and (key, box_idx) -> row, where a later crop of the same box replaces the earlier one."""

    def __init__(self, extractor, keys):
        self.extractor = extractor
        self.engine = extractor.engine
        self.keys = keys          # the query / gallery keys this class compares
        self.rows = 0
        self.buf = None           # allocated by the first embed pass
        self.row_of = {}

    def embed(self, crops, slots):
        """crops: [n] uint8 BGR arrays image[y:y+h, x:x+w]; slots: [(key, box_idx)] * n.  Each chunk of the extractor's
        batch goes to the engine as one padded [k, hmax, wmax, 3] array with box (i, 0, 0, w, h) for crop i: the
        resize reads the crop's own pixels only, so only the crops are uploaded, not the frames."""
        import torch
        n = len(slots)
        if n == 0:
            return
        if self.buf is None:
            self.buf = torch.empty((max(64, n), self.engine.feat_dim), dtype=torch.float32,
                                   device="cuda:%d" % self.engine.device)
        if self.rows + n > self.buf.shape[0]:
            cap = self.buf.shape[0]
            while cap < self.rows + n:
                cap *= 2
            grown = torch.empty((cap, self.buf.shape[1]), dtype=torch.float32, device=self.buf.device)
            grown[:self.rows] = self.buf[:self.rows]
            torch.cuda.current_stream(self.buf.device).synchronize()    # the engine writes on its own stream
            self.buf = grown
        b = self.extractor.batch
        for i in range(0, n, b):
            part = crops[i:i + b]
            k = len(part)
            packed = np.zeros((k, max(c.shape[0] for c in part), max(c.shape[1] for c in part), 3), np.uint8)
            boxes = np.zeros((k, 5), np.int64)
            for j, c in enumerate(part):
                packed[j, :c.shape[0], :c.shape[1]] = c
                boxes[j] = (j, 0, 0, c.shape[1], c.shape[0])
            self.engine.embed_boxes_dev(packed, boxes, self.buf[self.rows + i:self.rows + i + k])
        for i, slot in enumerate(slots):
            self.row_of[slot] = self.rows + i
        self.rows += n


def _stream_crops(frame_iter, frame_data, tables, frames_per_call):
    """:208-227 on the GPU: for every needed frame, valid_box on its shape, int() the tlwh and queue the crop for each
    class table that uses its key; every `frames_per_call` frames with queued crops, one embed pass per class.  Returns
    {key: {box_idx}} of the valid crops, with an entry (maybe empty) for every key whose frame arrived."""
    got = {}
    queued = {c: ([], []) for c in tables}
    pending = 0

    def flush():
        for c, (crops, slots) in queued.items():
            tables[c].embed(crops, slots)
            crops.clear()
            slots.clear()

    for batch in frame_iter[0]:
        image, scale, frame_idx = batch[0]
        if frame_idx not in frame_data:
            continue
        image = image.astype("uint8")
        used = False
        for tlwh, key, box_idx in frame_data[frame_idx]:
            if key not in got:
                got[key] = set()
            if not valid_box(tlwh, image):
                continue
            x, y, w, h = (int(v) for v in tlwh)
            if w < 1 or h < 1:
                raise ValueError("%s box %d %r: the integer crop [%d:%d, %d:%d] is empty (the reference fails in "
                                 "cv2.cvtColor)" % (key, box_idx, tuple(tlwh), y, y + h, x, x + w))
            got[key].add(box_idx)
            for c in tables:
                if key in tables[c].keys:
                    queued[c][0].append(image[y:y + h, x:x + w])
                    queued[c][1].append((key, box_idx))
                    used = True
        pending += used
        if pending >= frames_per_call:
            flush()
            pending = 0
    flush()
    return got


def tracklet_dist(q_feats, seg_q, g_feats, seg_g, pairs, method="min_all", precision="split"):
    """b2_tracklet_dist_dev on float32 CUDA tensors q_feats [seg_q[-1], D] and g_feats [seg_g[-1], D]: for each (query
    segment, gallery segment) of pairs [P, 2] the minimum squared euclidean distance over the two segments' rows
    ("min_all", unclamped) or the distance of their means ("avg") -> float32 [P]."""
    if method not in METHODS:
        raise ValueError("compare_method must be 'min_all' or 'avg', got %r" % (method,))
    seg_q = np.ascontiguousarray(seg_q, np.int32)
    seg_g = np.ascontiguousarray(seg_g, np.int32)
    pairs = np.ascontiguousarray(np.asarray(pairs, np.int32).reshape(-1, 2))
    for t in (q_feats, g_feats):
        assert t.is_cuda and t.is_contiguous() and str(t.dtype) == "torch.float32" and t.dim() == 2, t.shape
    assert q_feats.shape[1] == g_feats.shape[1]
    import torch
    torch.cuda.current_stream(q_feats.device).synchronize()           # the call reads them on its own stream
    out = np.empty(len(pairs), np.float32)
    _lib.check(_lib.load().b2_tracklet_dist_dev(q_feats.device.index or 0, c_void_p(q_feats.data_ptr()), _lib.ptr(seg_q),
                                                len(seg_q) - 1, c_void_p(g_feats.data_ptr()), _lib.ptr(seg_g),
                                                len(seg_g) - 1, int(q_feats.shape[1]), _lib.ptr(pairs), len(pairs),
                                                METHODS[method], {"fp16": 0, "split": 1}[precision], _lib.ptr(out)),
               "b2_tracklet_dist_dev")
    return out


def prune_candidates(candidates, got):
    """The first half of get_features_and_compare (:238-262): a query without a valid crop, or whose galleries have none,
    is listed for removal; the others keep only the galleries with a valid crop (candidates[q] is replaced).  `got` is
    {key: valid box indices}; a key whose frames never arrived raises the reference's KeyError (:241, :255).  Returns
    (queries to compare, queries to remove)."""
    remove_track_ids = {}
    live = []
    for query_track_id in candidates:
        query_boxes = got["query_%s" % query_track_id]
        if not query_boxes:
            remove_track_ids[query_track_id] = 1
            continue
        temp_list = [[g, o, c] for g, o, c in candidates[query_track_id] if got["gallery_%s" % g]]
        if not temp_list:
            remove_track_ids[query_track_id] = 1
            continue
        candidates[query_track_id] = temp_list
        live.append(query_track_id)
    return live, remove_track_ids


def attach_distances(candidates, live, remove_track_ids, dist):
    """The second half (:301-308): dist holds one distance per (query, candidate) of `live` in list order; each is
    appended to its candidate row, every list is sorted by it (stable) and the removed queries are deleted."""
    p = 0
    for q in live:
        for row in candidates[q]:
            row.append(dist[p])
            p += 1
        candidates[q].sort(key=operator.itemgetter(-1))
    for track_id in remove_track_ids:
        del candidates[track_id]


def _compare(candidates, table, got, method, precision):
    """get_features_and_compare (:233-310) with every remaining pair of the class scored in one b2_tracklet_dist_dev call
    on rows compacted from the class's feature table, in sorted box_idx order (:246, :269)."""
    import torch
    live, remove_track_ids = prune_candidates(candidates, got)
    dist = []
    if live:
        rows_q, seg_q, rows_g, seg_g, gal_idx, pairs = [], [0], [], [0], {}, []
        for qi, q in enumerate(live):
            key = "query_%s" % q
            rows_q += [table.row_of[(key, i)] for i in sorted(got[key])]
            seg_q.append(len(rows_q))
            for g, _, _ in candidates[q]:
                key = "gallery_%s" % g
                if key not in gal_idx:
                    gal_idx[key] = len(seg_g) - 1
                    rows_g += [table.row_of[(key, i)] for i in sorted(got[key])]
                    seg_g.append(len(rows_g))
                pairs.append((qi, gal_idx[key]))
        idx = lambda r: torch.as_tensor(r, dtype=torch.int64, device=table.buf.device)
        dist = tracklet_dist(table.buf.index_select(0, idx(rows_q)), seg_q, table.buf.index_select(0, idx(rows_g)), seg_g,
                             pairs, method, precision)
    attach_distances(candidates, live, remove_track_ids, dist)


def merge_candidates(candidates, track_data, reject_dist_thres):
    """:316-365: a query's best candidate below the threshold claims that gallery; of several claims the longest query
    wins (ties: the first); merges follow chains through merge_map.  The new track id is written through a view into
    the caller's arrays, as the reference does."""
    merge_map = {}
    reverse_candidates = {}
    for query_track_id in candidates:
        match_list = [(o[0], o[-1]) for o in candidates[query_track_id] if o[-1] < reject_dist_thres]
        if match_list:
            match_track_id, dist = match_list[0]
            if match_track_id not in reverse_candidates:
                reverse_candidates[match_track_id] = []
            reverse_candidates[match_track_id].append((query_track_id, dist, len(track_data[query_track_id])))
    for track_id in reverse_candidates:
        if len(reverse_candidates[track_id]) > 1:
            reverse_candidates[track_id].sort(key=operator.itemgetter(2), reverse=True)
        matched_prev_track_id, _, _ = reverse_candidates[track_id][0]
        while matched_prev_track_id in merge_map:
            matched_prev_track_id = merge_map[matched_prev_track_id]
        assert track_id not in merge_map
        assert matched_prev_track_id not in merge_map
        merge_map[track_id] = matched_prev_track_id
    new_track_data = {}
    for track_id in track_data:
        this_track_data = track_data[track_id][:, :]
        if track_id in merge_map:
            track_id = merge_map[track_id]
            this_track_data[:, 1] = track_id
        if track_id in new_track_data:
            new_track_data[track_id] = np.concatenate([new_track_data[track_id], this_track_data], axis=0)
        else:
            new_track_data[track_id] = this_track_data
    return new_track_data


def reid(frame_iter, p_extractor, v_extractor, p_track_data, p_candidates, v_track_data, v_candidates,
         feature_box_num=5, feature_box_gap=20, reject_dist_thres=200, compare_method="min_all", frames_per_call=8,
         precision="split"):
    """single_video_reid.py:141-370 -> (new person track data, new vehicle track data).  `frame_iter` is the reference's
    (iterable of batches, count) pair with batch[0] = (image, scale, frame_idx); the extractors are reid.FeatureExtractor
    (osnet_x1_0 and resnet101).  `p_candidates` / `v_candidates` are mutated in place as the reference does (queries and
    galleries without a valid crop removed, rows become [id, start, end, dist] sorted by dist), and so are the track
    arrays of merged tracks (their id column)."""
    if compare_method not in METHODS:
        raise AssertionError("compare_method must be 'min_all' or 'avg'")
    if frames_per_call < 1:
        raise ValueError("frames_per_call must be >= 1")
    needed_track_boxes = {}
    plan_boxes(needed_track_boxes, p_track_data, p_candidates, feature_box_num, feature_box_gap)
    plan_boxes(needed_track_boxes, v_track_data, v_candidates, feature_box_num, feature_box_gap)
    frame_data = {}
    for key in needed_track_boxes:
        for box_idx, box in enumerate(needed_track_boxes[key]):
            frame_idx = box[0]
            if frame_idx not in frame_data:
                frame_data[frame_idx] = []
            frame_data[frame_idx].append((box[2:6], key, box_idx))
    tables = {}
    for c, cands, ext in (("p", p_candidates, p_extractor), ("v", v_candidates, v_extractor)):
        if cands:
            tables[c] = _FeatureTable(ext, _class_keys(cands))
    got = _stream_crops(frame_iter, frame_data, tables, frames_per_call)
    for c, cands in (("p", p_candidates), ("v", v_candidates)):
        if c in tables:
            _compare(cands, tables[c], got, compare_method, precision)
    return (merge_candidates(p_candidates, p_track_data, reject_dist_thres),
            merge_candidates(v_candidates, v_track_data, reject_dist_thres))


def save_new_track(cat_name, track_data, out_dir, videoname):
    """:373-388: the rows of every track sorted by (frame, id), written as the MOT text file
    out_dir/videoname/cat_name/<videoname without extension>.txt."""
    track_results = sorted([l.tolist() for t in track_data for l in track_data[t]], key=lambda x: (x[0], x[1]))
    out_file_dir = os.path.join(out_dir, videoname, cat_name)
    if not os.path.exists(out_file_dir):
        os.makedirs(out_file_dir)
    out_file = os.path.join(out_file_dir, os.path.splitext(videoname)[0] + ".txt")
    with open(out_file, "w") as fw:
        for row in track_results:
            line = "%d,%d,%.2f,%.2f,%.2f,%.2f,%.4f,-1,-1,-1" % (row[0], row[1], row[2], row[3], row[4], row[5], row[6])
            fw.write(line + "\n")


def relink_video(person_track_file, vehicle_track_file, frame_iter, p_extractor, v_extractor, out_dir, videoname,
                 tol_num_frame=200, expand_width_p=2.0, expand_height_p=0.5, feature_box_num=500, feature_box_gap=20,
                 reject_dist_thres=150, compare_method="min_all", frames_per_call=8):
    """One video of the driver's loop (single_video_reid.py:476-510, defaults from its argparse): preprocess both track
    files, reid, write Person/ and Vehicle/ files under out_dir/videoname.  Decoding the video stays with the caller:
    `frame_iter` is (iterable of batches, count) as for reid.  Returns the track counts
    ((person before, after), (vehicle before, after))."""
    ori_p, p_data, p_cand = preprocess(person_track_file, tol_num_frame, expand_width_p, expand_height_p)
    ori_v, v_data, v_cand = preprocess(vehicle_track_file, tol_num_frame, expand_width_p, expand_height_p)
    new_p, new_v = reid(frame_iter, p_extractor, v_extractor, p_data, p_cand, v_data, v_cand,
                        feature_box_num=feature_box_num, feature_box_gap=feature_box_gap,
                        reject_dist_thres=reject_dist_thres, compare_method=compare_method,
                        frames_per_call=frames_per_call)
    save_new_track("Person", new_p, out_dir, videoname)
    save_new_track("Vehicle", new_v, out_dir, videoname)
    return (ori_p, len(new_p)), (ori_v, len(new_v))
