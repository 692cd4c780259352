"""EfficientDet BiFPN + heads + post-processing on the H100 (config 3 of the reference,
efficientdet_wrapper.py:160-474).  Thin host mirror over the C ABI (include/b200det.h, b2_effdet_*); no CPU path."""
from __future__ import annotations

import ctypes

import numpy as np

from . import _lib
from .effdet_config import make_effdet_config  # noqa: F401  (re-export)

# the post-processing's stages (include/b200det.h, b2_effdet_get_stage), and which of them hold int32
POST_STAGES = ("topk_boxes", "topk_scores", "topk_classes", "topk_levels", "topk_count", "final_boxes", "final_scores",
               "final_classes", "final_levels", "final_count", "box_feat", "image_scale")
I32_STAGES = ("topk_classes", "topk_levels", "topk_count", "final_classes", "final_levels", "final_count")


def _c_config(cfg, precision: str, backbone, batch: int = 1) -> _lib.B2EffdetConfig:
    c = _lib.B2EffdetConfig()
    c.backbone = -1 if backbone is None else int(str(backbone)[-1])
    c.image_h, c.image_w = int(cfg.image_size[0]), int(cfg.image_size[1])
    c.min_level, c.max_level = int(cfg.min_level), int(cfg.max_level)
    c.fpn_num_filters = int(cfg.fpn_num_filters)
    c.fpn_cell_repeats = int(cfg.fpn_cell_repeats)
    c.box_class_repeats = int(cfg.box_class_repeats)
    c.num_classes, c.num_scales, c.num_aspects = int(cfg.num_classes), int(cfg.num_scales), len(cfg.aspect_ratios)
    if len(cfg.aspect_ratios) > 3:
        raise ValueError("at most 3 aspect ratios")
    for i, (ax, ay) in enumerate(cfg.aspect_ratios):
        c.aspect_ratios[i][0], c.aspect_ratios[i][1] = float(ax), float(ay)
    c.anchor_scale = float(cfg.anchor_scale)
    c.fpn_weight_method = {"sum": 0, "fastattn": 1}[cfg.fpn_weight_method]
    for i in range(3):
        c.backbone_channels[i] = int(cfg.backbone_channels[i])
    c.max_detection_topk, c.result_per_im = int(cfg.max_detection_topk), int(cfg.result_per_im)
    c.nms_iou_threshold, c.result_score_thres = float(cfg.nms_iou_threshold), float(cfg.result_score_thres)
    c.precision = {"fp16": 0, "split": 1}[precision]
    c.batch = int(batch)
    return c


class EffdetEngine:
    """Feature network + heads + post-processing of one EfficientDet configuration on one GPU."""

    def __init__(self, cfg, weights: dict, device: int = 0, precision: str = "split", backbone=None, batch: int = 1):
        """backbone: None (features in, run_features only) or "efficientnet-b0".."efficientnet-b7" (detect()).
        batch: images per call; with batch > 1 the context runs detect_batch() (up to `batch` frames of any sizes, each
        bit-identical to detect() on a batch-1 context) and its stages carry every image."""
        if int(batch) < 1:
            raise ValueError("batch must be >= 1")
        self.cfg = cfg
        self.batch = int(batch)
        self._lib = _lib.load()
        self._h = ctypes.c_void_p()
        cc = _c_config(cfg, precision, backbone, self.batch)
        _lib.check(self._lib.b2_effdet_create(ctypes.byref(self._h), ctypes.byref(cc), int(device)), "b2_effdet_create")
        self.load_weights(weights)

    def load_weights(self, weights: dict) -> None:
        names = sorted(weights)
        arrs = [np.ascontiguousarray(np.asarray(weights[n], np.float32)).reshape(-1) for n in names]
        c_names = (ctypes.c_char_p * len(names))(*[n.encode() for n in names])
        c_data = (ctypes.c_void_p * len(names))(*[a.ctypes.data for a in arrs])
        c_numel = (ctypes.c_int64 * len(names))(*[a.size for a in arrs])
        _lib.check(self._lib.b2_effdet_load_weights(self._h, c_names, c_data, c_numel, len(names)),
                   "b2_effdet_load_weights")

    def run_features(self, features: dict, image_scale: float = 1.0) -> dict:
        """features: {3,4,5: [C,H,W] fp32} (the oracle's layout) -> final_boxes / final_probs / final_labels /
        levels / fpn_box_feat, rows in NMS selection order."""
        nhwc = [np.ascontiguousarray(np.asarray(features[l], np.float32).transpose(1, 2, 0)) for l in (3, 4, 5)]
        m, f = int(self.cfg.result_per_im), int(self.cfg.fpn_num_filters)
        boxes = np.zeros((m, 4), np.float32)
        scores = np.zeros(m, np.float32)
        classes = np.zeros(m, np.int32)
        levels = np.zeros(m, np.int32)
        feat = np.zeros((m, f), np.float32)
        count = np.zeros(1, np.int32)
        _lib.check(self._lib.b2_effdet_run_features(
            self._h, nhwc[0].ctypes.data, nhwc[1].ctypes.data, nhwc[2].ctypes.data, ctypes.c_float(image_scale),
            boxes.ctypes.data, scores.ctypes.data, classes.ctypes.data, levels.ctypes.data, feat.ctypes.data,
            count.ctypes.data), "b2_effdet_run_features")
        n = int(count[0])
        return dict(final_boxes=boxes[:n], final_probs=scores[:n], final_labels=classes[:n], levels=levels[:n],
                    fpn_box_feat=feat[:n])

    def detect(self, frame_bgr: np.ndarray) -> dict:
        """One BGR uint8 frame [h,w,3] -> detections in frame pixels (efficientdet_wrapper.py:40-111)."""
        frame = np.ascontiguousarray(frame_bgr, np.uint8)
        if frame.ndim != 3 or frame.shape[2] != 3:
            raise ValueError("frame must be [h, w, 3] uint8 BGR")
        m, f = int(self.cfg.result_per_im), int(self.cfg.fpn_num_filters)
        boxes = np.zeros((m, 4), np.float32)
        scores = np.zeros(m, np.float32)
        classes = np.zeros(m, np.int32)
        levels = np.zeros(m, np.int32)
        feat = np.zeros((m, f), np.float32)
        count = np.zeros(1, np.int32)
        scale = np.zeros(1, np.float32)
        _lib.check(self._lib.b2_effdet_detect(
            self._h, frame.ctypes.data, int(frame.shape[0]), int(frame.shape[1]), boxes.ctypes.data, scores.ctypes.data,
            classes.ctypes.data, levels.ctypes.data, feat.ctypes.data, count.ctypes.data, scale.ctypes.data),
            "b2_effdet_detect")
        n = int(count[0])
        return dict(final_boxes=boxes[:n], final_probs=scores[:n], final_labels=classes[:n], levels=levels[:n],
                    fpn_box_feat=feat[:n], image_scale=float(scale[0]))

    def detect_batch(self, frames) -> list:
        """1..batch BGR uint8 frames [h,w,3] of any sizes -> one dict per frame with detect()'s keys, in one pass."""
        frames = [np.ascontiguousarray(f, np.uint8) for f in frames]
        if not 1 <= len(frames) <= self.batch:
            raise ValueError("detect_batch takes 1 to %d frames, got %d" % (self.batch, len(frames)))
        for f in frames:
            if f.ndim != 3 or f.shape[2] != 3:
                raise ValueError("frames must be [h, w, 3] uint8 BGR")
        B, n = self.batch, len(frames)
        m, f = int(self.cfg.result_per_im), int(self.cfg.fpn_num_filters)
        boxes = np.zeros((B, m, 4), np.float32)
        scores = np.zeros((B, m), np.float32)
        classes = np.zeros((B, m), np.int32)
        levels = np.zeros((B, m), np.int32)
        feat = np.zeros((B, m, f), np.float32)
        count = np.zeros(B, np.int32)
        scale = np.zeros(B, np.float32)
        ptrs = (ctypes.c_void_p * n)(*[fr.ctypes.data for fr in frames])
        hs = np.array([fr.shape[0] for fr in frames], np.int32)
        ws = np.array([fr.shape[1] for fr in frames], np.int32)
        _lib.check(self._lib.b2_effdet_detect_batch(
            self._h, ptrs, hs.ctypes.data, ws.ctypes.data, n, boxes.ctypes.data, scores.ctypes.data, classes.ctypes.data,
            levels.ctypes.data, feat.ctypes.data, count.ctypes.data, scale.ctypes.data), "b2_effdet_detect_batch")
        out = []
        for b in range(n):
            r = int(count[b])
            out.append(dict(final_boxes=boxes[b, :r].copy(), final_probs=scores[b, :r].copy(),
                            final_labels=classes[b, :r].copy(), levels=levels[b, :r].copy(),
                            fpn_box_feat=feat[b, :r].copy(), image_scale=float(scale[b])))
        return out

    def replay_ms(self, reps: int = 10) -> float:
        """Mean milliseconds of one replay of the whole-frame graph the last detect call captured (no host copies)."""
        ms = ctypes.c_float()
        _lib.check(self._lib.b2_effdet_replay(self._h, int(reps), ctypes.byref(ms)), "b2_effdet_replay")
        return float(ms.value)

    def stage(self, name: str, real: int = None, image: int = None) -> np.ndarray:
        """'fpn3'..'fpn7' -> [H,W,F]; 'cls3'.. -> [H,W,A*num_classes]; 'box3'.. -> [H,W,A*4]; 'image' -> [H,W,3];
        'stem' / 'block_<i>' / 'c3'..'c5' -> [h,w,C] (pass `real` to drop the operand channel padding);
        post-processing stages (POST_STAGES) -> [n,4] boxes, [n,F] box_feat, else [n] (int32 for I32_STAGES).
        On a batch context: image `image`'s slice, or with image=None every image's, stacked on a leading axis."""
        if image is not None and not 0 <= int(image) < self.batch:
            raise IndexError("image %d of a batch of %d" % (image, self.batch))
        if name in POST_STAGES:
            return self._pick(self._post_stage(name), image)
        na = self.cfg.num_scales * len(self.cfg.aspect_ratios)
        if real is None:
            real = {"fpn": self.cfg.fpn_num_filters, "cls": na * self.cfg.num_classes, "box": na * 4,
                    "ima": 3}.get(name[:3])
            if name in ("c3", "c4", "c5"):
                real = self.cfg.backbone_channels[int(name[1]) - 3]
        cap = int(self.cfg.image_size[0]) * int(self.cfg.image_size[1]) * 64      # stride-2 maps have <= 64 channels
        if name[:3] in ("cls", "box", "fpn") or name in ("c3", "c4", "c5"):
            cap //= 4
        buf = np.zeros(cap * self.batch, np.float32)
        shape = (ctypes.c_int64 * 4)()
        _lib.check(self._lib.b2_effdet_get_stage(self._h, name.encode(), buf.ctypes.data, buf.nbytes, shape),
                   "b2_effdet_get_stage")
        nb, h, w, c = [int(v) for v in shape]
        out = buf[: nb * h * w * c].reshape(nb, h, w, c)
        return self._pick(out if real is None else out[..., :real], image).copy()

    def _pick(self, per_image: np.ndarray, image) -> np.ndarray:
        """[batch, ...] -> one image's [...] (image 0 of a batch-1 context when `image` is None), or all of them."""
        if image is None:
            return per_image[0] if self.batch == 1 else per_image
        return per_image[int(image)]

    def _post_stage(self, name: str) -> np.ndarray:
        """[batch, n, c] ([batch, n] where c is 1)."""
        k, m = int(self.cfg.max_detection_topk), int(self.cfg.result_per_im)
        buf = np.zeros(self.batch * max(4 * k, m * max(4, int(self.cfg.fpn_num_filters)), 8), np.float32)
        shape = (ctypes.c_int64 * 4)()
        _lib.check(self._lib.b2_effdet_get_stage(self._h, name.encode(), buf.ctypes.data, buf.nbytes, shape),
                   "b2_effdet_get_stage")
        nb, n, c = int(shape[0]), int(shape[2]), int(shape[3])
        out = buf[: nb * n * c]
        if name in I32_STAGES:
            out = out.view(np.int32)
        out = out.reshape(nb, n, c)
        if name == "topk_count" and c == 8:          # a batch context exposes each image's [8] top-k state: count at 5
            out = out[:, :, 5:6]
        return (out if out.shape[2] > 1 else out[:, :, 0]).copy()

    def set_stage(self, name: str, value: np.ndarray) -> None:
        """Overwrite a stage with its whole stored shape: 'cls3'.. [H,W,pad16(A*num_classes)], 'box3'.. [H,W,pad16(A*4)],
        'fpn3'.. [H,W,pad64(F)] (float32), 'image_scale' [1], or a post-processing stage (int32 for I32_STAGES); on a
        batch context every image's, stacked on a leading [batch] axis."""
        a = np.ascontiguousarray(value, np.int32 if name in I32_STAGES else np.float32)
        _lib.check(self._lib.b2_effdet_set_stage(self._h, name.encode(), a.ctypes.data, a.nbytes), "b2_effdet_set_stage")

    def run_phases(self, mask: int) -> None:
        """Run the phases in `mask` (_lib.EFFDET_PHASES bits) eagerly on the current stages."""
        _lib.check(self._lib.b2_effdet_run_phases(self._h, int(mask)), "b2_effdet_run_phases")

    def profile_steps(self, reps: int = 5):
        """[(name, kind, ms, flops, bytes)] per launch group of the last pass (CUDA events, eager launches)."""
        cap = 4096
        ms = (ctypes.c_float * cap)()
        n = ctypes.c_int()
        _lib.check(self._lib.b2_effdet_profile_steps(self._h, int(reps), ms, cap, ctypes.byref(n)), "b2_effdet_profile_steps")
        out = []
        for i in range(n.value):
            name = ctypes.create_string_buffer(256)
            fl, by, kind = ctypes.c_double(), ctypes.c_double(), ctypes.c_int()
            _lib.check(self._lib.b2_effdet_step_info(self._h, i, name, 256, ctypes.byref(fl), ctypes.byref(by),
                                                     ctypes.byref(kind)), "b2_effdet_step_info")
            out.append((name.value.decode(), kind.value, float(ms[i]), fl.value, by.value))
        return out

    @property
    def num_launches(self) -> int:
        return int(self._lib.b2_effdet_num_launches(self._h))

    def close(self) -> None:
        if self._h:
            self._lib.b2_effdet_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
