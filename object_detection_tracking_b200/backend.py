"""Drop-in model objects for the reference's detect call surface.

The reference drivers never touch TF ops: they call `models.get_model(...)`, read five tensor
attributes and call `sess.run(fetches, feed_dict=model.get_feed_dict_forward(img))`
(obj_detect_tracking.py:505,610-635; obj_detect_tracking_multi_queuer.py:474-480).  The frozen-graph
classes show that boundary is meant to be swappable ("has the same interface as Mask_RCNN_FPN",
models.py:196-263).  This module provides the same surface on top of libb200det:

    model = get_model(config, gpuid=0, controller="/cpu:0", is_multi=False)     # models.py:97-119
    model.image, model.final_boxes, model.final_labels, model.final_probs, model.fpn_box_feat,
    model.final_valid_indices (batch mode)
    model.get_feed_dict_forward(img) / model.get_feed_dict_forward_multi(imgs)  # models.py:1629,3301
    sess = Session(); sess.run([model.final_boxes, ...], feed_dict=fd)

Outputs follow the reference conventions: fresh, writable numpy arrays owned by the caller; boxes are
x1,y1,x2,y2 in resized-image pixels; labels are 1-based (int64 single image, float32 batch): class ids 1..num_class-1,
or with config.use_partial_classes 1..len(partial_classes), the position in partial_classes plus one, with probabilities
from the (len(partial_classes) + 1)-way softmax (models.py:807-843).
There is no CPU fallback: without the CUDA library or an H100 the calls raise.
"""
from __future__ import annotations

import copy

import numpy as np

from .config import normalize_config
from .engine import Detector


_SLOT_NAMES = ("Adam", "Adam_1", "Adadelta", "Adadelta_1", "Momentum", "beta1_power", "beta2_power")


def check_weights(config, weights: dict) -> dict:
    """The importer's host half (reference: initialize(), obj_detect_tracking.py:392-448).  Accepts a name -> array dict in
    the checkpoint naming with or without the ':0' tensor suffix (utils.get_op_tensor_name, utils.py:708-723); like the
    reference it ignores entries the inference graph has no variable for (optimizer slots, global_step, learning rate, the
    mask / training heads) -- but where the reference silently leaves a MISSING variable at its random initial value, this
    raises, listing every missing or mis-shaped name.  Returns float32 C-contiguous arrays keyed by op name."""
    from .synth import frcnn_weight_shapes
    need = frcnn_weight_shapes(config)
    got = {}
    for k, v in weights.items():
        name = k[:-2] if (len(k) >= 3 and k[-2] == ":") else k
        if name.split("/")[-1] in _SLOT_NAMES or name not in need:
            continue
        got[name] = np.ascontiguousarray(v, dtype=np.float32)
    missing = sorted(set(need) - set(got))
    bad = sorted("%s: %s, expected %s" % (n, got[n].shape, need[n]) for n in got if tuple(got[n].shape) != tuple(need[n]))
    if missing or bad:
        raise ValueError("checkpoint does not fit the configured graph (num_class=%d, blocks=%s): %d missing %s%s; %d "
                         "mis-shaped %s" % (config.num_class, tuple(config.resnet_num_block), len(missing), missing[:8],
                                            " ..." if len(missing) > 8 else "", len(bad), bad[:8]))
    return got


class TensorHandle:
    """Stands in for a tf.Tensor / placeholder: only identity and a name matter to the drivers."""

    def __init__(self, model, name):
        self.model = model
        self.name = name

    def __repr__(self):
        return "<b200det tensor %s>" % self.name


class Mask_RCNN_FPN:
    """Single-image model object (reference: models.py:266-1813, inference surface only).  With use_partial_classes the
    checkpoint (or frozen graph) is the 81-class COCO model; the engine keeps the box-head columns of
    config.partial_class_ids and final_labels are 1..len(partial_classes), as the driver's partial targetid2class reads
    them (obj_detect_tracking.py:287-291).  final_masks keep the reference's channel choice (DESIGN.md section 4)."""

    is_multi = False

    def __init__(self, config, gpuid=0, precision="split", input_dtype="float32", feat_mode=0):
        self.config = normalize_config(config)
        if self.config.use_small_object_head and (self.is_multi or getattr(self.config, "is_load_from_pb", False)):
            # the batch graph has no small-object branch (models.py:1969-3487) and pack() exports the main outputs only
            # (models.py:134-147): such a model runs without it
            cfg = copy.copy(self.config)
            cfg.use_small_object_head = False
            self.config = normalize_config(cfg)
        self.gpuid = gpuid
        self.precision = precision
        self.input_dtype = input_dtype
        # what `fpn_box_feat` returns: 0 = the reference's [R,256,7,7]; 1 / 2 / 3 = the drivers' emb_agg_method avg / max /
        # spatial computed on the GPU ([R,256] / [R,256] / [R,49], obj_detect_tracking_multi_queuer.py:482-495): 49x fewer
        # bytes over PCIe, and create_obj_infos / preprocess_detections take the pooled form as it is
        self.feat_mode = int(feat_mode)
        self.num_class = self.config.num_class
        self.image = TensorHandle(self, "image:0")
        self.final_boxes = TensorHandle(self, "final_boxes:0")          # exported names: models.py:138-146
        self.final_labels = TensorHandle(self, "final_labels:0")
        self.final_probs = TensorHandle(self, "final_probs:0")
        self.fpn_box_feat = TensorHandle(self, "fpn_box_feat:0")
        self.final_valid_indices = TensorHandle(self, "final_valid_indices:0")
        self.final_masks = TensorHandle(self, "final_masks:0")          # with config.add_mask (models.py:143-146,958-961)
        # with config.use_small_object_head (models.py:893-897); single-image graph only
        self.so_final_boxes = TensorHandle(self, "so_final_boxes:0")
        self.so_final_labels = TensorHandle(self, "so_final_labels:0")
        self.so_final_probs = TensorHandle(self, "so_final_probs:0")
        self._weights = None
        self._detectors = {}

    # -- weights (reference: initialize(), obj_detect_tracking.py:392-448) ----------------------------
    def set_weights(self, weights: dict):
        self._weights = check_weights(self.config, weights)
        for d in self._detectors.values():
            d.load_weights(self._weights)

    def load_npz(self, path: str):
        """Tensorpack-style .npz: names with or without the ':0' suffix (obj_detect_tracking.py:417-443)."""
        with np.load(path) as z:
            self.set_weights({k: z[k] for k in z.files})

    def load_pb(self, path: str):
        """Frozen graph written by the reference's pack() (models.py:134-191): the variables are Const nodes under their
        checkpoint names; read without TensorFlow (pbreader.py), then the same manifest check as load_npz."""
        from .pbreader import read_frozen_graph
        consts = read_frozen_graph(path)
        prefix = "model_%s/" % self.gpuid           # graphs re-exported after import_graph_def carry it (models.py:211)
        self.set_weights({(k[len(prefix):] if k.startswith(prefix) else k): v for k, v in consts.items()})

    # -- feed dicts -----------------------------------------------------------------------------------
    def get_feed_dict_forward(self, imgdata):
        """models.py:1629-1636: {image placeholder: float32 HWC BGR frame}."""
        return {self.image: imgdata}

    def get_feed_dict_forward_multi(self, imgdatas):
        """models.py:3301-3310: list of equally sized frames -> [B,H,W,3]."""
        return {self.image: np.stack(imgdatas, axis=0)}

    # -- execution --------------------------------------------------------------------------------------
    def _detector(self, B, H, W) -> Detector:
        key = (B, H, W)
        det = self._detectors.get(key)
        if det is None:
            if self._weights is None:
                raise RuntimeError("model has no weights: call set_weights()/load_npz() first")
            det = Detector(self.config, B, H, W, device=self.gpuid, input_dtype=self.input_dtype,
                           precision=self.precision, multi_semantics=self.is_multi)
            det.load_weights(self._weights)
            self._detectors[key] = det
        return det

    def detector(self, batch, height, width) -> Detector:
        """The engine context behind this model object for a (batch, H, W) plan: queue-fed drivers use its two-slot
        streaming pair submit_host / wait (INTEGRATION.md 1a) instead of one synchronous sess.run per batch."""
        return self._detector(int(batch), int(height), int(width))

    def _run(self, fetches, feed_dict):
        img = feed_dict[self.image]
        img = np.asarray(img)
        single = img.ndim == 3
        frames = img[None] if single else img
        B, H, W, _ = frames.shape
        det = self._detector(B, H, W)
        self._last_det = det
        want_feat = any(f is self.fpn_box_feat for f in fetches)
        out = det.detect_host(frames, feat_mode=self.feat_mode, want_feat=want_feat)
        valid = out["valid"]
        so = None
        so_handles = (self.so_final_boxes, self.so_final_labels, self.so_final_probs)
        if any(f is h for f in fetches for h in so_handles):
            if not self.config.use_small_object_head:
                raise KeyError("so_final_boxes / so_final_labels / so_final_probs need config.use_small_object_head in the "
                               "single-image graph (models.py:590)")
            so = det.get_small_objects()
            if so["status"]:
                raise RuntimeError("small-object head: the classes %s kept %s boxes in their NMS; the reference's tf.map_fn "
                                   "needs equal counts and fails here (models.py:618-621)"
                                   % (list(self.config.small_objects), so["class_counts"].tolist()))
        res = []
        for f in fetches:
            if so is not None and any(f is h for h in so_handles):
                if f is self.so_final_boxes:
                    res.append(so["boxes"])
                elif f is self.so_final_labels:
                    res.append(so["labels"].astype(np.int64))                 # models.py:887-888: int64, 1..C
                else:
                    res.append(so["probs"])                                   # logits (models.py:884)
            elif single:
                r = int(valid[0])
                if f is self.final_boxes:
                    res.append(out["boxes"][0, :r].copy())
                elif f is self.final_labels:
                    res.append(out["labels"][0, :r].astype(np.int64))          # models.py:932: int64, class+1 (partial: 1..C)
                elif f is self.final_probs:
                    res.append(out["probs"][0, :r].copy())
                elif f is self.fpn_box_feat:
                    res.append(out["feat"][:r].copy())
                elif f is self.final_valid_indices:
                    res.append(valid.copy())
                elif f is self.final_masks:
                    if not getattr(self.config, "add_mask", False):
                        raise KeyError("final_masks needs config.add_mask (models.py:934)")
                    res.append(det.get_masks()[0, :r].copy())                  # [R,28,28] float32
                else:
                    raise KeyError("unknown fetch %r" % (f,))
            else:
                if f is self.final_boxes:
                    res.append(out["boxes"].copy())
                elif f is self.final_labels:
                    res.append(out["labels"].astype(np.float32))              # models.py:2973: float32 in batch mode
                elif f is self.final_probs:
                    res.append(out["probs"].copy())
                elif f is self.final_valid_indices:
                    res.append(valid.copy())
                elif f is self.fpn_box_feat:
                    R = det.R
                    res.append(np.concatenate([out["feat"][b * R:b * R + int(valid[b])] for b in range(B)], axis=0))
                elif f is self.final_masks:                                    # models.py:2379-2407: [sum R, 28, 28]
                    if not getattr(self.config, "add_mask", False):
                        raise KeyError("final_masks needs config.add_mask (models.py:2379)")
                    m = det.get_masks()
                    res.append(np.concatenate([m[b, :int(valid[b])] for b in range(B)], axis=0))
                else:
                    raise KeyError("unknown fetch %r" % (f,))
        return res


    def encode_masks(self, boxes_scaled, im_shape, image=0):
        """The drivers' RLE dicts ({"size": [H, W], "counts": str}, obj_detect_tracking.py:716-739) of the final_masks of
        image `image` of the last run, computed on the GPU where the masks are: boxes_scaled are that image's final_boxes
        divided by the resize scale (float32), im_shape the source frame's (H, W)."""
        if not getattr(self.config, "add_mask", False):
            raise KeyError("encode_masks needs config.add_mask (models.py:934)")
        det = getattr(self, "_last_det", None)
        if det is None:
            raise RuntimeError("encode_masks needs a run of the model first")
        return det.encode_masks(boxes_scaled, im_shape, image)


class RCNN_FPN_givenbox(Mask_RCNN_FPN):
    """Feature extractor for given boxes (reference: models.py:1816-1967): `model.image`, `model.boxes`,
    `model.final_box_features`, `model.get_feed_dict(im, boxes)`; run with Session.run([model.final_box_features], fd)."""

    def __init__(self, config, gpuid=0, precision="split", input_dtype="float32"):
        super().__init__(config, gpuid, precision, input_dtype)
        self.boxes = TensorHandle(self, "boxes:0")
        self.final_box_features = TensorHandle(self, "final_box_features:0")

    def get_feed_dict(self, im, boxes, is_train=False):          # models.py:1953-1967
        return {self.image: im, self.boxes: boxes}

    def _run(self, fetches, feed_dict):
        img = np.asarray(feed_dict[self.image])
        det = self._detector(1, img.shape[0], img.shape[1])
        feats = det.box_features(img, feed_dict[self.boxes])
        res = []
        for f in fetches:
            if f is not self.final_box_features:
                raise KeyError("the given-box model has one output: final_box_features")
            res.append(feats.copy())
        return res


def get_model_feat(config, gpuid=0, task=0, controller="/cpu:0", **kw):
    """models.get_model_feat (models.py:121-131)."""
    return RCNN_FPN_givenbox(config, gpuid=gpuid, **kw)


class Mask_RCNN_FPN_multi(Mask_RCNN_FPN):
    """Fixed-batch model object (reference: models.py:1969-3487): post-processing follows the batch graph
    (combined_non_max_suppression semantics, `multi_semantics` in the C ABI)."""

    is_multi = True


class EfficientDet:
    """EfficientDet model object (reference: efficientdet_wrapper.py:12-111 `EfficientDet`): same five attributes and
    `get_feed_dict_forward` as Mask_RCNN_FPN; the whole graph -- build_preprocess (uint8 BGR frame -> RGB, /255,
    mean/std, bilinear fit to (short_edge_size, max_size), zero pad), EfficientNet backbone, BiFPN, class/box nets,
    top-k + class-agnostic NMS, own-level ROIAlign feature -- runs in libb200det (b2_effdet_*).
    Outputs: boxes x1,y1,x2,y2 in the pixels of the frame that was fed (the graph multiplies by
    image_scale_to_original itself, wrapper :350-353), labels int32 in 1..num_classes (1..len(partial_classes) with
    use_partial_classes), probs float32, fpn_box_feat [R, fpn_num_filters]."""

    is_multi = False

    def __init__(self, config, gpuid=0, precision="split"):
        from .effdet_config import BACKBONE_OF, make_effdet_config
        self.config = config
        self.gpuid = gpuid
        self.precision = precision
        name = getattr(config, "efficientdet_modelname", "efficientdet-d0")
        over = dict(min_level=int(getattr(config, "efficientdet_min_level", 3)),
                    max_level=int(getattr(config, "efficientdet_max_level", 7)),
                    max_detection_topk=int(getattr(config, "efficientdet_max_detection_topk", 5000)),
                    result_score_thres=float(getattr(config, "result_score_thres", 1e-4)),
                    result_per_im=int(getattr(config, "result_per_im", 100)))
        # get_efficientdet_config (wrapper :160-252): image_size = (short_edge_size, max_size)
        self.eff_config = make_effdet_config(name, int(config.short_edge_size), int(config.max_size), **over)
        self.backbone_name = BACKBONE_OF[name]
        self.partial_class_idxs = []
        if getattr(config, "use_partial_classes", False):
            from .class_ids import coco_id_mapping_reverse
            self.partial_class_idxs = [coco_id_mapping_reverse[c] - 1 for c in config.partial_classes]
            self.eff_config.num_classes = len(self.partial_class_idxs)
        self.image = TensorHandle(self, "image:0")
        self.final_boxes = TensorHandle(self, "final_boxes:0")          # wrapper :31-35
        self.final_labels = TensorHandle(self, "final_labels:0")
        self.final_probs = TensorHandle(self, "final_probs:0")
        self.fpn_box_feat = TensorHandle(self, "fpn_box_feat:0")
        self._engine = None
        self._weights = None

    def set_weights(self, weights: dict):
        """TF checkpoint variables (efficientdet_arch.py / efficientnet_model.py names, kernels HWIO).  With
        use_partial_classes the class-predict columns are gathered here, which is what the graph's tf.gather on the
        class logits (wrapper :398-404) computes."""
        w = {k: np.asarray(v, dtype=np.float32) for k, v in weights.items()}
        if self.partial_class_idxs:
            na = self.eff_config.num_scales * len(self.eff_config.aspect_ratios)
            full = w["class_net/class-predict/bias"].shape[0] // na
            cols = np.concatenate([a * full + np.asarray(self.partial_class_idxs) for a in range(na)])
            w["class_net/class-predict/pointwise_kernel"] = w["class_net/class-predict/pointwise_kernel"][..., cols]
            w["class_net/class-predict/bias"] = w["class_net/class-predict/bias"][cols]
        self._weights = w
        if self._engine is not None:
            self._engine.load_weights(w)

    def load_npz(self, path: str):
        with np.load(path) as z:
            self.set_weights({k: z[k] for k in z.files})

    def load_pb(self, path: str):
        """Frozen EfficientDet graph (EfficientDet_frozen, models.py:103-104): Const nodes under the checkpoint variable
        names, read without TensorFlow (pbreader.py)."""
        from .pbreader import read_frozen_graph
        prefix = "model_%s/" % self.gpuid
        self.set_weights({(k[len(prefix):] if k.startswith(prefix) else k): v for k, v in read_frozen_graph(path).items()})

    def get_feed_dict_forward(self, imgdata):
        """wrapper :105-111: {image placeholder (uint8 [h,w,3] BGR): frame}."""
        return {self.image: imgdata}

    def _run(self, fetches, feed_dict):
        from .effdet import EffdetEngine
        if self._engine is None:
            if self._weights is None:
                raise RuntimeError("model has no weights: call set_weights()/load_npz() first")
            self._engine = EffdetEngine(self.eff_config, self._weights, device=self.gpuid, precision=self.precision,
                                        backbone=self.backbone_name)
        frame = np.asarray(feed_dict[self.image])
        if frame.dtype != np.uint8:
            frame = frame.astype(np.uint8)          # the placeholder is uint8 (wrapper :19-21)
        out = self._engine.detect(frame)
        table = {id(self.final_boxes): out["final_boxes"], id(self.final_labels): out["final_labels"],
                 id(self.final_probs): out["final_probs"], id(self.fpn_box_feat): out["fpn_box_feat"]}
        res = []
        for f in fetches:
            if id(f) not in table:
                raise KeyError("unknown fetch %r" % (f,))
            res.append(table[id(f)].copy())
        return res


class EfficientDet_multi(EfficientDet):
    """Batch-mode EfficientDet model object for the reference's batch drivers (obj_detect_tracking_multi_queuer.py:472-515
    with --is_efficientdet): `get_feed_dict_forward_multi(imgs)` and the `final_valid_indices` fetch.  The frames of a
    batch may differ in size; each runs with the single-image semantics of `EfficientDet` (bit-identical outputs) in one
    pass of a batch context, one context per batch size.  Outputs in the batch graph's layout: boxes [B, result_per_im, 4]
    and probs [B, result_per_im] zero-padded, labels [B, result_per_im] float32 (1-based, 0 in the padding), valid [B]
    int32, fpn_box_feat [sum(valid), fpn_num_filters] image by image."""

    is_multi = True

    def __init__(self, config, gpuid=0, precision="split"):
        super().__init__(config, gpuid=gpuid, precision=precision)
        self.final_valid_indices = TensorHandle(self, "final_valid_indices:0")
        self._engines = {}

    def set_weights(self, weights: dict):
        super().set_weights(weights)
        for e in self._engines.values():
            e.load_weights(self._weights)

    def get_feed_dict_forward_multi(self, imgdatas):
        """models.py:3301-3310: the batch's frames, each [h, w, 3]."""
        return {self.image: [np.asarray(im) for im in imgdatas]}

    def _engine_for(self, batch: int):
        from .effdet import EffdetEngine
        eng = self._engines.get(batch)
        if eng is None:
            if self._weights is None:
                raise RuntimeError("model has no weights: call set_weights()/load_npz() first")
            eng = EffdetEngine(self.eff_config, self._weights, device=self.gpuid, precision=self.precision,
                               backbone=self.backbone_name, batch=batch)
            self._engines[batch] = eng
        return eng

    def _run(self, fetches, feed_dict):
        imgs = feed_dict[self.image]
        frames = [np.asarray(f) for f in (imgs if isinstance(imgs, (list, tuple)) else np.asarray(imgs))]
        frames = [f if f.dtype == np.uint8 else f.astype(np.uint8) for f in frames]     # the placeholder is uint8
        B, m = len(frames), int(self.eff_config.result_per_im)
        outs = self._engine_for(B).detect_batch(frames)
        boxes = np.zeros((B, m, 4), np.float32)
        labels = np.zeros((B, m), np.float32)
        probs = np.zeros((B, m), np.float32)
        valid = np.zeros(B, np.int32)
        for b, o in enumerate(outs):
            r = len(o["final_probs"])
            boxes[b, :r], labels[b, :r], probs[b, :r], valid[b] = o["final_boxes"], o["final_labels"], o["final_probs"], r
        feat = np.concatenate([o["fpn_box_feat"] for o in outs], axis=0)
        table = {id(self.final_boxes): boxes, id(self.final_labels): labels, id(self.final_probs): probs,
                 id(self.final_valid_indices): valid, id(self.fpn_box_feat): feat}
        res = []
        for f in fetches:
            if id(f) not in table:
                raise KeyError("unknown fetch %r" % (f,))
            res.append(table[id(f)].copy())
        return res


class Session:
    """`sess.run(fetches, feed_dict=...)` for fetches that all belong to one model object."""

    def run(self, fetches, feed_dict=None):
        single = not isinstance(fetches, (list, tuple))
        flist = [fetches] if single else list(fetches)
        model = flist[0].model
        out = model._run(flist, feed_dict or {})
        return out[0] if single else out

    def close(self):
        pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()


def get_model(config, gpuid=0, task=0, controller="/cpu:0", is_multi=False, **kw):
    """models.get_model (models.py:97-119).  `controller`/`task` are TF device-placement arguments with
    no meaning here; kept for signature compatibility."""
    if getattr(config, "is_efficientdet", False):
        cls = EfficientDet_multi if is_multi else EfficientDet
        model = cls(config, gpuid=gpuid, **kw)                          # models.py:112-113
        if getattr(config, "is_load_from_pb", False):                   # EfficientDet_frozen (models.py:103-104)
            model.load_pb(config.load_from)
        return model
    cls = Mask_RCNN_FPN_multi if is_multi else Mask_RCNN_FPN
    model = cls(config, gpuid=gpuid, **kw)
    if getattr(config, "is_load_from_pb", False):                       # models.py:102-109 Mask_RCNN_FPN_frozen(config.load_from)
        model.load_pb(config.load_from)
    return model
