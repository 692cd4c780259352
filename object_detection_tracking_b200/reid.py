"""GPU drop-in for the reference's ReID embedding API and distance matrices.

`FeatureExtractor` mirrors torchreid.utils.FeatureExtractor (torchreid/feature_extractor.py:121-252): same
constructor arguments, callable on a list of HWC RGB uint8 arrays / a single array / image paths, returns a
`torch.Tensor [B, 512]`.  `__call__` keeps the PIL resize of the reference's transform pipeline on the host (it is the
reference's own library call); ToTensor + Normalize + the whole OSNet-x1.0 forward run in libb200det
(b2_reid_embed).  `extract_boxes` takes the frame and the track boxes instead and cuts, converts and resizes them on
the GPU bit-exactly as Pillow does (b2_reid_embed_boxes).  `compute_distance_matrix` mirrors
torchreid/distance.py:6-46.  No CPU fallback.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import c_char_p, c_int64, c_void_p

import numpy as np

from . import _lib


class ReidEngine:
    """Owner of a b2_reid context for one crop batch size."""

    MODELS = {"osnet_x1_0": (0, (256, 128), 512), "resnet101": (1, (128, 256), 2048)}   # id, crop (h, w), feature width

    def __init__(self, batch: int, device: int = 0, precision: str = "split", model: str = "osnet_x1_0"):
        self.lib = _lib.load()
        self.batch = int(batch)
        self.model = model
        self.device = int(device)
        self.model_id, self.image_size, self.feat_dim = self.MODELS[model]
        self._ctx = c_void_p(0)
        _lib.check(self.lib.b2_reid_create_model(ctypes.byref(self._ctx), int(device), self.batch,
                                                 {"fp16": 0, "split": 1}[precision], self.model_id), "b2_reid_create_model")

    def close(self):
        if getattr(self, "_ctx", None) is not None and self._ctx.value:
            self.lib.b2_reid_destroy(self._ctx)
            self._ctx = c_void_p(0)

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def load_state(self, state: dict):
        names = sorted(k for k in state if not k.startswith("classifier") and not k.endswith("num_batches_tracked"))
        arrs = [np.ascontiguousarray(np.asarray(state[k]), dtype=np.float32) for k in names]
        n = len(names)
        _lib.check(self.lib.b2_reid_load_weights(self._ctx, (c_char_p * n)(*[k.encode() for k in names]),
                                                 (c_void_p * n)(*[a.ctypes.data for a in arrs]),
                                                 (c_int64 * n)(*[a.size for a in arrs]), n), "b2_reid_load_weights")

    def embed(self, crops_u8: np.ndarray) -> np.ndarray:
        """crops_u8: [n, h, w, 3] RGB uint8 already resized to the model's crop size (256x128 osnet_x1_0, 128x256
        resnet101), n <= batch -> [n, 512 | 2048] float32."""
        crops_u8 = np.ascontiguousarray(crops_u8, dtype=np.uint8)
        n = crops_u8.shape[0]
        assert crops_u8.shape[1:] == self.image_size + (3,), crops_u8.shape
        out = np.empty((n, self.feat_dim), dtype=np.float32)
        _lib.check(self.lib.b2_reid_embed(self._ctx, _lib.ptr(crops_u8), n, _lib.ptr(out)), "b2_reid_embed")
        return out

    def embed_dev(self, crops_u8: np.ndarray, out_dev) -> None:
        """Same pass with the [n, feat_dim] features written into `out_dev` -- a float32 torch CUDA tensor (or a slice of
        one: e.g. this camera's rows of the gallery buffer the NCCL all-gather sends) on this engine's GPU; nothing comes
        back to the host (b2_reid_embed_dev)."""
        crops_u8 = np.ascontiguousarray(crops_u8, dtype=np.uint8)
        n = crops_u8.shape[0]
        assert crops_u8.shape[1:] == self.image_size + (3,), crops_u8.shape
        assert out_dev.is_cuda and out_dev.is_contiguous() and tuple(out_dev.shape) == (n, self.feat_dim), out_dev.shape
        assert str(out_dev.dtype) == "torch.float32"
        _lib.check(self.lib.b2_reid_embed_dev(self._ctx, _lib.ptr(crops_u8), n, c_void_p(out_dev.data_ptr())),
                   "b2_reid_embed_dev")

    def _boxes_args(self, frames, boxes):
        frames = np.asarray(frames)
        if frames.dtype != np.uint8:
            raise ValueError("frames must be uint8 BGR, got %s" % frames.dtype)
        frames = np.ascontiguousarray(frames)
        if frames.ndim == 3:
            frames = frames[None]
        if frames.ndim != 4 or frames.shape[3] != 3:
            raise ValueError("frames must be [h, w, 3] or [F, h, w, 3] uint8 BGR, got shape %s" % (frames.shape,))
        boxes = np.asarray(boxes)
        if boxes.ndim != 2 or boxes.shape[1] != 5 or not np.issubdtype(boxes.dtype, np.integer):
            raise ValueError("boxes must be an integer [n, 5] table (frame, x, y, w, h), got %s %s" % (boxes.dtype,
                                                                                                      boxes.shape))
        if boxes.size and (boxes.min() < np.iinfo(np.int32).min or boxes.max() > np.iinfo(np.int32).max):
            raise ValueError("box coordinates do not fit int32")
        return frames, np.ascontiguousarray(boxes, dtype=np.int32)

    def embed_boxes(self, frames, boxes) -> np.ndarray:
        """frames: [h, w, 3] or [F, h, w, 3] uint8 BGR; boxes: int [n, 5] rows (frame index, x, y, w, h), 1 <= n <= batch,
        each inside its frame -> [n, feat_dim] float32, the features of
        Image.fromarray(frame[y:y+h, x:x+w, ::-1]).resize(crop size, BILINEAR) for every box, cut out and resized on the
        GPU (b2_reid_embed_boxes).  A bad box raises RuntimeError before anything is launched."""
        frames, boxes = self._boxes_args(frames, boxes)
        out = np.empty((boxes.shape[0], self.feat_dim), dtype=np.float32)
        _lib.check(self.lib.b2_reid_embed_boxes(self._ctx, _lib.ptr(frames), frames.shape[0], frames.shape[1],
                                                frames.shape[2], _lib.ptr(boxes), boxes.shape[0], _lib.ptr(out)),
                   "b2_reid_embed_boxes")
        return out

    def embed_boxes_dev(self, frames, boxes, out_dev) -> None:
        """embed_boxes with the [n, feat_dim] features written into `out_dev`, a contiguous float32 torch CUDA tensor on
        this engine's GPU, as embed_dev (b2_reid_embed_boxes_dev)."""
        frames, boxes = self._boxes_args(frames, boxes)
        n = boxes.shape[0]
        assert out_dev.is_cuda and out_dev.is_contiguous() and tuple(out_dev.shape) == (n, self.feat_dim), out_dev.shape
        assert str(out_dev.dtype) == "torch.float32"
        _lib.check(self.lib.b2_reid_embed_boxes_dev(self._ctx, _lib.ptr(frames), frames.shape[0], frames.shape[1],
                                                    frames.shape[2], _lib.ptr(boxes), n, c_void_p(out_dev.data_ptr())),
                   "b2_reid_embed_boxes_dev")

    def get_activation(self, name: str) -> np.ndarray:
        """fp32 NHWC copy of a named intermediate of the last pass (parity tests)."""
        shape = (c_int64 * 4)()
        cap = self.batch * 131 * 64 * 64 * 4 * (4 if self.model_id == 1 else 1) + 1024
        buf = np.empty(cap // 4, dtype=np.float32)
        _lib.check(self.lib.b2_reid_get_activation(self._ctx, name.encode(), _lib.ptr(buf), buf.nbytes, shape),
                   "b2_reid_get_activation")
        shp = tuple(int(v) for v in shape)
        return buf[:int(np.prod(shp))].reshape(shp).copy()

    def num_launches(self) -> int:
        return int(self.lib.b2_reid_num_launches(self._ctx))


class FeatureExtractor(object):
    """torchreid/feature_extractor.py:121-252 with model_name='osnet_x1_0' (person, image_size (256, 128)) or 'resnet101'
    (vehicle, image_size (128, 256): single_video_reid.py:404-415)."""

    def __init__(self, model_name="osnet_x1_0", model_path="", image_size=(256, 128),
                 pixel_mean=(0.485, 0.456, 0.406), pixel_std=(0.229, 0.224, 0.225), pixel_norm=True,
                 device="cuda", verbose=False, batch=32, precision="split", state_dict=None):
        if model_name not in ReidEngine.MODELS:
            raise NotImplementedError("the GPU path implements osnet_x1_0 (person) and resnet101 (vehicle), the two "
                                      "extractors the drivers build (single_video_reid.py:404-415)")
        if tuple(image_size) != ReidEngine.MODELS[model_name][1] or not pixel_norm \
                or tuple(pixel_mean) != (0.485, 0.456, 0.406) or tuple(pixel_std) != (0.229, 0.224, 0.225):
            raise NotImplementedError("only the drivers' settings are built: 256x128 for osnet_x1_0, 128x256 for "
                                      "resnet101, ImageNet mean/std")
        dev = 0
        if isinstance(device, str) and ":" in device:
            dev = int(device.split(":")[1])
        self.image_size = tuple(image_size)
        self.engine = ReidEngine(batch, dev, precision, model_name)
        self.batch = batch
        if state_dict is None and model_path and os.path.isfile(model_path):
            import torch
            ckpt = torch.load(model_path, map_location="cpu")
            state_dict = ckpt.get("state_dict", ckpt)
            state_dict = {(k[7:] if k.startswith("module.") else k): v.numpy() for k, v in state_dict.items()}
        if state_dict is None:
            raise RuntimeError("FeatureExtractor needs weights: pass model_path (torchreid checkpoint) or state_dict")
        self.engine.load_state(state_dict)

    def _resize(self, arr):
        from PIL import Image       # T.Resize on a PIL image == Image.resize(bilinear) (feature_extractor.py:190-196)
        img = arr if isinstance(arr, Image.Image) else Image.fromarray(np.asarray(arr, dtype=np.uint8))
        h, w = self.image_size
        return np.asarray(img.convert("RGB").resize((w, h), Image.BILINEAR), dtype=np.uint8)

    def __call__(self, input):
        import torch
        from PIL import Image
        if isinstance(input, (str, np.ndarray)):
            input = [input]
        if not isinstance(input, list):
            raise NotImplementedError("expects a list of HWC uint8 arrays / paths (feature_extractor.py:209-236)")
        crops = [self._resize(Image.open(e) if isinstance(e, str) else e) for e in input]
        feats = []
        for i in range(0, len(crops), self.batch):
            feats.append(self.engine.embed(np.stack(crops[i:i + self.batch])))
        return torch.from_numpy(np.concatenate(feats, 0) if feats else np.zeros((0, self.engine.feat_dim), np.float32))

    def extract_boxes(self, frame_bgr, tlwhs):
        """The drivers' ReID input step (single_video_reid.py:211-227, multi_video_reid.py:212-239) on the GPU: for each
        box tlwh of the uint8 BGR frame [h, w, 3], int() each coordinate, cut image[y:y+h, x:x+w], turn it to RGB and
        resize it as T.Resize does -> torch.Tensor [n, D], the same features as
        self([cv2.cvtColor(crop, cv2.COLOR_BGR2RGB) for crop in crops]).  Boxes go to the engine `batch` at a time.
        Raises ValueError for a box whose integer crop is empty or leaves the frame: callers keep filtering with
        valid_box (utils.py:44-57) first, as the drivers do."""
        import torch
        frame = np.asarray(frame_bgr)
        if frame.ndim != 3 or frame.shape[2] != 3 or frame.dtype != np.uint8:
            raise ValueError("frame_bgr must be a [h, w, 3] uint8 BGR image")
        H, W = frame.shape[:2]
        boxes = np.zeros((len(tlwhs), 5), np.int64)
        for i, tlwh in enumerate(tlwhs):
            x, y, w, h = (int(v) for v in list(tlwh)[:4])
            if w < 1 or h < 1 or x < 0 or y < 0 or x + w > W or y + h > H:
                raise ValueError("box %d %r: the crop [%d:%d, %d:%d] is empty or leaves the %dx%d frame"
                                 % (i, tuple(tlwh), y, y + h, x, x + w, W, H))
            boxes[i, 1:] = (x, y, w, h)
        frame = np.ascontiguousarray(frame)                 # once, not once per chunk
        feats = [self.engine.embed_boxes(frame, boxes[i:i + self.batch]) for i in range(0, len(boxes), self.batch)]
        return torch.from_numpy(np.concatenate(feats, 0) if feats else np.zeros((0, self.engine.feat_dim), np.float32))


def compute_distance_matrix(input1, input2, metric="euclidean", device=0, precision="split"):
    """torchreid/distance.py:6-46: [m,d] x [n,d] -> [m,n]; 'euclidean' is the SQUARED distance (:49-64)."""
    import torch
    a = np.ascontiguousarray(input1.detach().cpu().numpy() if hasattr(input1, "detach") else input1, dtype=np.float32)
    b = np.ascontiguousarray(input2.detach().cpu().numpy() if hasattr(input2, "detach") else input2, dtype=np.float32)
    assert a.ndim == 2 and b.ndim == 2 and a.shape[1] == b.shape[1]
    if metric not in ("euclidean", "cosine"):
        raise ValueError('Unknown distance metric: {}. Please choose either "euclidean" or "cosine"'.format(metric))
    out = np.zeros((a.shape[0], b.shape[0]), dtype=np.float32)
    if out.size:
        lib = _lib.load()
        _lib.check(lib.b2_distance_matrix(device, _lib.ptr(a), a.shape[0], _lib.ptr(b), b.shape[0], a.shape[1],
                                          0 if metric == "cosine" else 1, {"fp16": 0, "split": 1}[precision],
                                          _lib.ptr(out)), "b2_distance_matrix")
    return torch.from_numpy(out)


def allgather_gallery(local_feats, group=None):
    """Multi-camera ReID exchange step (SURVEY section 8e): every rank contributes its stream's gallery
    [rows_i, D]; returns (all_feats [sum rows, D], rows_per_rank).  torch.distributed is the plumbing:
    NCCL over NVLink for CUDA tensors, gloo for CPU tensors in the tests."""
    import torch
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return local_feats, [int(local_feats.shape[0])]
    world = dist.get_world_size(group)
    rows = torch.tensor([local_feats.shape[0]], dtype=torch.int64, device=local_feats.device)
    all_rows = [torch.zeros_like(rows) for _ in range(world)]
    dist.all_gather(all_rows, rows, group=group)
    counts = [int(r.item()) for r in all_rows]
    mx = max(counts)
    padded = torch.zeros((mx, local_feats.shape[1]), dtype=local_feats.dtype, device=local_feats.device)
    padded[:local_feats.shape[0]] = local_feats
    bufs = [torch.zeros_like(padded) for _ in range(world)]
    dist.all_gather(bufs, padded, group=group)
    return torch.cat([b[:c] for b, c in zip(bufs, counts)], 0), counts


def allgather_gallery_dev(local_gallery, rows_cap, group=None):
    """Device-resident exchange step of config 5 (multi_video_reid.py:448-476): `local_gallery` is this camera's
    [rows_cap, D] float32 CUDA tensor (rows beyond the real count are padding); ONE all_gather_into_tensor over NCCL /
    NVLink fills [world, rows_cap, D] on every GPU.  The galleries never visit the host: b2_reid_embed_dev wrote them,
    b2_track_pair_cost_dev reads them.  torch.distributed owns the NCCL communicator (plumbing); the C ABI works on the
    device pointers (INTEGRATION.md)."""
    import torch
    import torch.distributed as dist
    world = dist.get_world_size(group)
    assert local_gallery.is_cuda and local_gallery.is_contiguous() and local_gallery.shape[0] == rows_cap
    out = torch.empty((world,) + tuple(local_gallery.shape), dtype=local_gallery.dtype, device=local_gallery.device)
    dist.all_gather_into_tensor(out, local_gallery, group=group)
    return out


def match_cameras_allgather(tracks_meta, local_gallery, rows_cap, device=0, group=None, frame_offsets=None, tol=50,
                            cost_limit=998., precision="split", ignore_pairs=None, timing=None, object_group=None):
    """Config 5 with the NCCL all-gather (the p2p form is match_cameras_p2p).  Every rank = one camera.
    `tracks_meta` = {track_id: (trajectory rows [K,>=3], number of crop embeddings)} of this camera, whose embeddings sit
    in `local_gallery[:sum(counts)]` (track-id order).  Returns {(i, j): [(id_i, id_j), ...]} for the pairs this rank owns.
    `timing` (dict) receives the all-gather time in ms (CUDA events) and its payload bytes.  `group` carries the gallery
    tensors (NCCL); `object_group` (default: the same) the small host-side metadata -- a gloo group keeps it off the GPU."""
    import torch
    import torch.distributed as dist
    from .tmot import lapjv
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    if object_group is None:
        object_group = group
    ids = sorted(tracks_meta.keys())
    seg = np.zeros(len(ids) + 1, np.int32)
    for k, t in enumerate(ids):
        seg[k + 1] = seg[k] + int(tracks_meta[t][1])
    assert seg[-1] <= rows_cap
    meta = dict(ids=ids, seg=seg, traj={t: np.asarray(tracks_meta[t][0], dtype=np.float64) for t in ids})
    metas = [None] * world
    dist.all_gather_object(metas, meta, group=object_group)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    gathered = allgather_gallery_dev(local_gallery, rows_cap, group)
    e1.record()
    torch.cuda.synchronize()
    if timing is not None:
        timing["allgather_ms"] = e0.elapsed_time(e1)
        timing["allgather_bytes_recv"] = int((world - 1) * local_gallery.numel() * 4)
    dim = int(local_gallery.shape[1])
    result = {}
    for (i, j) in camera_pairs(world, rank, world):
        mi, mj = metas[i], metas[j]
        if not mi["ids"] or not mj["ids"]:
            result[(i, j)] = []
            continue
        fr_i, pt_i, sg_i = _pack_traj({t: (mi["traj"][t], None) for t in mi["ids"]})
        fr_j, pt_j, sg_j = _pack_traj({t: (mj["traj"][t], None) for t in mj["ids"]})
        off = 0 if frame_offsets is None else frame_offsets.get((i, j), 0)
        spatial = np.zeros((len(mi["ids"]), len(mj["ids"])), dtype=np.float64)
        _lib.check(_lib.load().b2_track_spatial_dist(_lib.ptr(fr_i), _lib.ptr(pt_i), _lib.ptr(sg_i), len(mi["ids"]),
                                                     _lib.ptr(fr_j), _lib.ptr(pt_j), _lib.ptr(sg_j), len(mj["ids"]),
                                                     int(off), float(tol), _lib.ptr(spatial)), "b2_track_spatial_dist")
        ign = (ignore_pairs or {}).get((i, j))
        if ign:                                      # multi_video_reid.py:299-303
            for a, t1 in enumerate(mi["ids"]):
                for b, t2 in enumerate(mj["ids"]):
                    if t1 in ign[0] and t2 in ign[1]:
                        spatial[a, b] = 9999.
        feat = pair_cost_device(c_void_p(gathered[i].data_ptr()), mi["seg"], c_void_p(gathered[j].data_ptr()), mj["seg"],
                                dim, spatial, device, precision)
        _, x, _ = lapjv(feat, extend_cost=True, cost_limit=cost_limit)
        result[(i, j)] = [(mi["ids"][a], mj["ids"][int(b)]) for a, b in enumerate(x) if b >= 0]
    return result


# ---- multi-camera track matching (multi_video_reid.py:260-324, 486-534) -----------------------------------------------

def _pack_tracks(tracks):
    """tracks: {track_id: (boxes [K,>=3] with frame id first and the top-down point last, features [K',D])} -> sorted ids,
    trajectory arrays and the concatenated gallery with segment offsets."""
    ids = sorted(tracks.keys())
    frames, pts, seg_t, feats, seg_f = [], [], [0], [], [0]
    for tid in ids:
        data = np.asarray(tracks[tid][0], dtype=np.float64).reshape(len(tracks[tid][0]), -1)
        frames.append(data[:, 0].astype(np.int32))          # int(p[0])
        pts.append(data[:, -2:])
        seg_t.append(seg_t[-1] + len(data))
        f = np.asarray(tracks[tid][1], dtype=np.float32)
        f = f.reshape(-1, f.shape[-1])
        feats.append(f)
        seg_f.append(seg_f[-1] + len(f))
    return (ids, np.ascontiguousarray(np.concatenate(frames)), np.ascontiguousarray(np.concatenate(pts)),
            np.asarray(seg_t, np.int32), np.ascontiguousarray(np.concatenate(feats)), np.asarray(seg_f, np.int32))


def compute_spatial_dist(tracks1, tracks2, frame_offset=0, tol=50, ignore_pairs=([], [])):
    """multi_video_reid.py:260-305 ([N,M] float64, 9999 = not comparable)."""
    ids1, fr1, pt1, seg1, _, _ = _pack_tracks(tracks1)
    ids2, fr2, pt2, seg2, _, _ = _pack_tracks(tracks2)
    out = np.zeros((len(ids1), len(ids2)), dtype=np.float64)
    _lib.check(_lib.load().b2_track_spatial_dist(_lib.ptr(fr1), _lib.ptr(pt1), _lib.ptr(seg1), len(ids1), _lib.ptr(fr2),
                                                 _lib.ptr(pt2), _lib.ptr(seg2), len(ids2), int(frame_offset), float(tol),
                                                 _lib.ptr(out)), "b2_track_spatial_dist")
    for i, t1 in enumerate(ids1):                          # :299-303
        for j, t2 in enumerate(ids2):
            if t1 in ignore_pairs[0] and t2 in ignore_pairs[1]:
                out[i, j] = 9999.
    return out


def compute_feature_dist(tracks1, tracks2, spatial_dist, device=0, precision="split"):
    """multi_video_reid.py:308-324: [N,M] minimum squared crop-embedding distance where spatial_dist < 9999, else 999.
    One GEMM over both cameras' galleries on the GPU instead of one sklearn call per track pair."""
    ids1, _, _, _, f1, s1 = _pack_tracks(tracks1)
    ids2, _, _, _, f2, s2 = _pack_tracks(tracks2)
    gate = np.ascontiguousarray(np.asarray(spatial_dist) < 9999., dtype=np.uint8)
    out = np.zeros((len(ids1), len(ids2)), dtype=np.float32)
    _lib.check(_lib.load().b2_track_pair_cost(int(device), _lib.ptr(f1), _lib.ptr(s1), len(ids1), _lib.ptr(f2), _lib.ptr(s2),
                                              len(ids2), f1.shape[1], _lib.ptr(gate), 999.0,
                                              {"fp16": 0, "split": 1}[precision], _lib.ptr(out)), "b2_track_pair_cost")
    return out.astype(np.float64)


def match_tracks(tracks1, tracks2, frame_offset=0, tol=50, ignore_pairs=([], []), cost_limit=998., device=0,
                 precision="split", feature_dist_fn=None):
    """One camera pair of the bubble compare (multi_video_reid.py:486-534): spatial gate -> feature distance ->
    lap.lapjv(extend_cost=True, cost_limit=998) -> [(track id in camera 1, track id in camera 2), ...].
    `feature_dist_fn(tracks1, tracks2, spatial_dist)` replaces the GPU cost (the CPU tests pass the oracle)."""
    from .tmot import lapjv
    if not tracks1 or not tracks2:
        return []
    spatial = compute_spatial_dist(tracks1, tracks2, frame_offset, tol, ignore_pairs)
    if feature_dist_fn is not None:
        feat = np.asarray(feature_dist_fn(tracks1, tracks2, spatial), dtype=np.float64)
    else:
        feat = compute_feature_dist(tracks1, tracks2, spatial, device, precision)
    _, x, _ = lapjv(feat, extend_cost=True, cost_limit=cost_limit)
    ids1, ids2 = sorted(tracks1.keys()), sorted(tracks2.keys())
    return [(ids1[i], ids2[int(j)]) for i, j in enumerate(x) if j >= 0]


def camera_pairs(n_cameras, rank=0, world_size=1):
    """The bubble-compare pairs (i < j) of multi_video_reid.py:474-476, dealt round-robin to the ranks: after the gallery
    all-gather every GPU scores its share of the pairs (28 pairs on 8 cameras) independently."""
    pairs = [(i, j) for i in range(n_cameras - 1) for j in range(i + 1, n_cameras)]
    return pairs[rank::world_size]


# ---- multi-camera exchange over peer memory (one process per GPU; SURVEY 8e) --------------------------------------------
class SharedGallery(object):
    """One camera's crop embeddings [rows, D] in device memory that the other ranks of the node can map.  Instead of
    all-gathering every gallery into every GPU, each rank opens the galleries of the cameras it has to score against and
    the operand-conversion kernel of the distance GEMM reads them over NVLink in place (b2_track_pair_cost_dev)."""

    def __init__(self, feats, device=0):
        feats = np.ascontiguousarray(feats, dtype=np.float32).reshape(len(feats), -1)
        self.rows, self.dim, self.device = int(feats.shape[0]), int(feats.shape[1]), int(device)
        self._lib = _lib.load()
        self._ptr = c_void_p(0)
        self._handle = (ctypes.c_uint8 * 64)()
        _lib.check(self._lib.b2_gallery_create(self.device, _lib.ptr(feats), self.rows, self.dim, ctypes.byref(self._ptr),
                                               self._handle), "b2_gallery_create")
        self._peers = {}

    @property
    def ptr(self):
        return self._ptr

    @property
    def handle(self) -> bytes:
        return bytes(self._handle)

    def open_peer(self, handle: bytes):
        """Maps another rank's gallery; returns its device pointer on this rank."""
        if handle not in self._peers:
            buf = (ctypes.c_uint8 * 64).from_buffer_copy(handle)
            p = c_void_p(0)
            _lib.check(self._lib.b2_gallery_open(self.device, buf, ctypes.byref(p)), "b2_gallery_open")
            self._peers[handle] = p
        return self._peers[handle]

    def close(self):
        for p in self._peers.values():
            self._lib.b2_gallery_close(self.device, p)
        self._peers = {}
        if self._ptr.value:
            self._lib.b2_gallery_free(self.device, self._ptr)
            self._ptr = c_void_p(0)


def pair_cost_device(ptr1, seg1, ptr2, seg2, dim, spatial_dist=None, device=0, precision="split"):
    """compute_feature_dist (multi_video_reid.py:308-324) on galleries that already live in (own or peer) device memory."""
    seg1 = np.ascontiguousarray(seg1, dtype=np.int32)
    seg2 = np.ascontiguousarray(seg2, dtype=np.int32)
    N, M = len(seg1) - 1, len(seg2) - 1
    gate = None if spatial_dist is None else np.ascontiguousarray(np.asarray(spatial_dist) < 9999., dtype=np.uint8)
    out = np.zeros((N, M), dtype=np.float32)
    _lib.check(_lib.load().b2_track_pair_cost_dev(int(device), ptr1, _lib.ptr(seg1), N, ptr2, _lib.ptr(seg2), M, int(dim),
                                                  _lib.ptr(gate), 999.0, {"fp16": 0, "split": 1}[precision], _lib.ptr(out)),
               "b2_track_pair_cost_dev")
    return out.astype(np.float64)


def match_cameras_p2p(tracks, device=0, group=None, frame_offsets=None, tol=50, cost_limit=998., precision="split",
                      ignore_pairs=None):
    """Config 5 on N ranks = N cameras (one process per GPU): every rank publishes its camera's gallery (SharedGallery),
    the 64-byte handles and the small host-side metadata (track ids, crop counts, trajectories) travel through
    torch.distributed objects, and each rank scores its share of the camera pairs (`camera_pairs`) reading the other
    camera's gallery over NVLink.  `tracks` is this rank's {track_id: (boxes [K,>=3], features [K',D])}.
    `frame_offsets` / `ignore_pairs` are keyed by the camera pair (i, j).
    Returns {(cam_i, cam_j): [(track id in i, track id in j), ...]} for the pairs this rank owns."""
    import torch.distributed as dist
    from .tmot import lapjv
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    ids, _, _, _, feats, seg = _pack_tracks(tracks) if tracks else ([], None, None, None, np.zeros((0, 1), np.float32),
                                                                    np.zeros(1, np.int32))
    gal = SharedGallery(feats, device)
    meta = dict(handle=gal.handle, ids=ids, seg=seg, dim=gal.dim, rows=gal.rows,
                traj={t: np.asarray(tracks[t][0], dtype=np.float64) for t in ids})
    metas = [None] * world
    dist.all_gather_object(metas, meta, group=group)
    result = {}
    try:
        for (i, j) in camera_pairs(world, rank, world):
            mi, mj = metas[i], metas[j]
            if not mi["ids"] or not mj["ids"]:
                result[(i, j)] = []
                continue
            ti = {t: (mi["traj"][t], None) for t in mi["ids"]}
            tj = {t: (mj["traj"][t], None) for t in mj["ids"]}
            off = 0 if frame_offsets is None else frame_offsets.get((i, j), 0)
            fr_i, pt_i, sg_i = _pack_traj(ti)
            fr_j, pt_j, sg_j = _pack_traj(tj)
            spatial = np.zeros((len(mi["ids"]), len(mj["ids"])), dtype=np.float64)
            _lib.check(_lib.load().b2_track_spatial_dist(_lib.ptr(fr_i), _lib.ptr(pt_i), _lib.ptr(sg_i), len(mi["ids"]),
                                                         _lib.ptr(fr_j), _lib.ptr(pt_j), _lib.ptr(sg_j), len(mj["ids"]),
                                                         int(off), float(tol), _lib.ptr(spatial)), "b2_track_spatial_dist")
            ign = (ignore_pairs or {}).get((i, j))
            if ign:                                      # multi_video_reid.py:299-303
                for a, t1 in enumerate(mi["ids"]):
                    for b, t2 in enumerate(mj["ids"]):
                        if t1 in ign[0] and t2 in ign[1]:
                            spatial[a, b] = 9999.
            pi = gal.ptr if i == rank else gal.open_peer(mi["handle"])
            pj = gal.ptr if j == rank else gal.open_peer(mj["handle"])
            feat = pair_cost_device(pi, mi["seg"], pj, mj["seg"], mi["dim"], spatial, device, precision)
            _, x, _ = lapjv(feat, extend_cost=True, cost_limit=cost_limit)
            result[(i, j)] = [(mi["ids"][a], mj["ids"][int(b)]) for a, b in enumerate(x) if b >= 0]
    finally:
        dist.barrier(group=group)          # nobody frees a gallery a peer may still be reading
        gal.close()
    return result


def _pack_traj(tracks):
    ids = sorted(tracks.keys())
    frames, pts, seg = [], [], [0]
    for t in ids:
        d = np.asarray(tracks[t][0], dtype=np.float64)
        d = d.reshape(len(d), -1)
        frames.append(d[:, 0].astype(np.int32))
        pts.append(d[:, -2:])
        seg.append(seg[-1] + len(d))
    return (np.ascontiguousarray(np.concatenate(frames)), np.ascontiguousarray(np.concatenate(pts)),
            np.asarray(seg, np.int32))
