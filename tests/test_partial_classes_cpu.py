"""--use_partial_classes without a GPU: the configuration, the C ABI's refusals, the importer, the oracle's partial
post-processing against a plain numpy restatement of models.py:807-843, the mask channel quirk, and the driver glue
(obj_detect_tracking.py:287-291 + tracking.create_obj_infos)."""
import ctypes

import numpy as np
import pytest

import partial_oracle
import test_abi
from object_detection_tracking_b200 import _lib
from object_detection_tracking_b200.backend import check_weights
from object_detection_tracking_b200.class_ids import coco_obj_class_to_id, coco_obj_to_actev_obj
from object_detection_tracking_b200.config import make_config, normalize_config
from object_detection_tracking_b200.synth import synth_frame, synth_weights
from oracle import frcnn

COCO = dict(num_class=81, use_dilations=False, version=2)
PARTIAL = ["person", "car", "bus", "truck", "bicycle"]
# the driver's partial tables (obj_detect_tracking.py:287-291)
PARTIAL_ID2CLASS = {i: n for i, n in enumerate(["BG"] + PARTIAL)}


# ---- configuration --------------------------------------------------------------------------------------------------
def test_default_selection_is_the_actev_table_in_order():
    assert list(coco_obj_to_actev_obj) == PARTIAL
    cfg = make_config(use_partial_classes=True, **COCO)
    assert cfg.partial_classes == PARTIAL
    assert cfg.partial_class_ids == (1, 3, 6, 8, 2)
    assert cfg.partial_class_ids == tuple(coco_obj_class_to_id[n] for n in PARTIAL)
    assert make_config(**COCO).partial_class_ids == ()
    # the checkpoint driver's classname2id (the partial table) is not consulted: ids stay the COCO ids
    cfg = make_config(use_partial_classes=True, classname2id={n: i for i, n in PARTIAL_ID2CLASS.items()}, **COCO)
    assert cfg.partial_class_ids == (1, 3, 6, 8, 2)
    cfg = make_config(use_partial_classes=True, partial_classes=["truck", "person"], **COCO)
    assert cfg.partial_class_ids == (8, 1) and normalize_config(cfg).partial_class_ids == (8, 1)


@pytest.mark.parametrize("over, words", [
    (dict(partial_classes=["person", "motorbike"]), "'motorbike'"),
    (dict(partial_classes=["BG", "person"]), "'BG'"),
    (dict(partial_classes=["person", "car", "person"]), "'person'"),
    (dict(partial_classes=[]), "empty"),
    (dict(num_class=15), "num_class must be 81"),
])
def test_refusals_name_the_problem(over, words):
    kw = dict(COCO, use_partial_classes=True)
    kw.update(over)
    with pytest.raises(ValueError) as e:
        make_config(**kw)
    assert words in str(e.value)


def test_effdet_configs_keep_their_own_selection():
    cfg = make_config(is_efficientdet=True, use_partial_classes=True, partial_classes=PARTIAL)   # num_class 15 is fine
    assert cfg.partial_class_ids == ()


def test_config_ext2_carries_the_ids():
    assert ctypes.sizeof(_lib.B2ConfigExt2) == 4 * test_abi._header_struct_words("b2_config_ext2")
    e = _lib.make_config_ext2(make_config(use_partial_classes=True, **COCO))
    assert e.num_partial_classes == 5 and list(e.partial_class_ids[:5]) == [1, 3, 6, 8, 2]
    assert all(v == 0 for v in e.partial_class_ids[5:])
    assert _lib.make_config_ext2(make_config(**COCO)).num_partial_classes == 0
    every = make_config(use_partial_classes=True, partial_classes=[frcnn_name(i) for i in range(1, 81)], **COCO)
    e = _lib.make_config_ext2(every)
    assert e.num_partial_classes == 80 and list(e.partial_class_ids) == list(range(1, 81))


def frcnn_name(i):
    from object_detection_tracking_b200.class_ids import coco_obj_id_to_class
    return coco_obj_id_to_class[i]


@pytest.mark.parametrize("ids, words", [
    ([1, 0, 3], "partial_class_ids[1] = 0"),
    ([1, 81], "partial_class_ids[1] = 81"),
    ([3, 6, 3], "class id 3 appears twice"),
])
def test_create_refuses_bad_ids_before_touching_a_device(ids, words):
    lib = _lib.load()
    cfg = make_config(use_partial_classes=True, **COCO)
    c = _lib.make_config(cfg, 1, 256, 384)
    ext = _lib.make_config_ext(cfg)
    e = _lib.make_config_ext2(cfg)
    e.num_partial_classes = len(ids)
    for i, v in enumerate(ids):
        e.partial_class_ids[i] = v
    ctx = ctypes.c_void_p(0)
    assert lib.b2_create_ex2(ctypes.byref(ctx), 0, ctypes.byref(c), ctypes.byref(ext), ctypes.byref(e)) != 0
    assert words in lib.b2_last_error().decode() and not ctx.value
    e.num_partial_classes = 81
    assert lib.b2_create_ex2(ctypes.byref(ctx), 0, ctypes.byref(c), ctypes.byref(ext), ctypes.byref(e)) != 0
    assert "num_partial_classes" in lib.b2_last_error().decode()


def test_importer_still_wants_the_81_class_head():
    cfg = make_config(resnet_num_block=(1, 1, 1, 1), use_partial_classes=True, **COCO)
    W = synth_weights(cfg, 3)
    assert W["fastrcnn/outputs/class/W"].shape == (1024, 81) and W["fastrcnn/outputs/box/W"].shape == (1024, 324)
    check_weights(cfg, W)
    bad = dict(W)
    bad["fastrcnn/outputs/class/W"] = W["fastrcnn/outputs/class/W"][:, [0, 1, 3, 6, 8, 2]]    # an already-gathered head
    bad["fastrcnn/outputs/box/W"] = W["fastrcnn/outputs/box/W"][:, :24]
    with pytest.raises(ValueError) as e:
        check_weights(cfg, bad)
    assert "fastrcnn/outputs/class/W" in str(e.value) and "fastrcnn/outputs/box/W" in str(e.value)


# ---- post-processing: oracle vs a plain restatement of models.py:807-843 ------------------------------------------------
def _restate(cls_full, box_full, rois, ids, agnostic, hw, cfg, multi):
    """models.py:798-843 (single image) / :2256-2303 (batch graph), written out with numpy: tile, transposes, the two
    gathers, decode_bbox_target + clip_boxes (nn.py:1518-1538, 1339-1346), softmax, per-class greedy NMS, top-k.
    Returns (decoded [K,C,4], probs [K,C+1], [(roi, class0)] selection, final probs)."""
    f32 = np.float32
    K = cls_full.shape[0]
    box = box_full.reshape(K, -1, 4)
    box = np.tile(box, (1, 80, 1)) if agnostic else box[:, 1:]
    label_t = cls_full.transpose(1, 0)
    box_t = box.transpose(1, 0, 2)
    cls = label_t[[0] + list(ids)].transpose(1, 0)
    bl = box_t[[i - 1 for i in ids]].transpose(1, 0, 2)
    C = len(ids)
    t = (bl / np.asarray(cfg.fastrcnn_bbox_reg_weights, f32)).astype(f32)
    a = np.repeat(rois[:, None, :], C, 1)
    wa, ha = a[..., 2] - a[..., 0], a[..., 3] - a[..., 1]
    xa, ya = (a[..., 2] + a[..., 0]) * f32(0.5), (a[..., 3] + a[..., 1]) * f32(0.5)
    clip = f32(np.log(1333 / 16.0))
    wb, hb = np.exp(np.minimum(t[..., 2], clip)) * wa, np.exp(np.minimum(t[..., 3], clip)) * ha
    xb, yb = t[..., 0] * wa + xa, t[..., 1] * ha + ya
    dec = np.stack([xb - wb * f32(0.5), yb - hb * f32(0.5), xb + wb * f32(0.5), yb + hb * f32(0.5)], -1).astype(f32)
    dec = np.minimum(np.maximum(dec, f32(0)), np.array([hw[1], hw[0], hw[1], hw[0]], f32))
    e = np.exp(cls - cls.max(1, keepdims=True))
    probs = (e / e.sum(1, keepdims=True)).astype(f32)

    def iou(p, q):
        iw = max(min(p[2], q[2]) - max(p[0], q[0]), 0.0)
        ih = max(min(p[3], q[3]) - max(p[1], q[1]), 0.0)
        inter = iw * ih
        return inter / ((p[2] - p[0]) * (p[3] - p[1]) + (q[2] - q[0]) * (q[3] - q[1]) - inter)

    cand = []
    for c in range(C):
        pc = probs[:, c + 1]
        ok = [k for k in np.argsort(-pc, kind="stable") if multi or pc[k] > cfg.result_score_thres]
        kept = []
        for k in ok:
            if len(kept) < cfg.result_per_im and all(iou(dec[k, c], dec[j, c]) <= cfg.fastrcnn_nms_iou_thres for j in kept):
                kept.append(k)
        cand += [(int(k), c) for k in kept]
    cand.sort(key=lambda kc: -float(probs[kc[0], kc[1] + 1]))
    sel = cand[:cfg.result_per_im]
    return dec, probs, sel, np.array([probs[k, c + 1] for k, c in sel], f32)


def _random_head(seed, K=300, hw=(200, 300), agnostic=False):
    rng = np.random.default_rng(seed)
    xy = rng.uniform(0, [hw[1] - 40, hw[0] - 40], (K, 2))
    wh = rng.uniform(8, 60, (K, 2))
    rois = np.concatenate([xy, xy + wh], 1).astype(np.float32)
    cls = (rng.standard_normal((K, 81)) * 2.0).astype(np.float32)
    box = (rng.standard_normal((K, 4 if agnostic else 324)) * 0.5).astype(np.float32)
    return rois, cls, box


@pytest.mark.parametrize("agnostic", [False, True])
@pytest.mark.parametrize("multi", [False, True])
@pytest.mark.parametrize("ids", [(1, 3, 6, 8, 2), (8,), (80, 1, 40)])
def test_oracle_partial_postprocess_matches_restatement(agnostic, multi, ids):
    cfg = make_config(use_partial_classes=True, use_frcnn_class_agnostic=agnostic, **COCO)
    hw = (200, 300)
    rois, cls, box = _random_head(len(ids) * 7 + agnostic + 2 * multi, hw=hw, agnostic=agnostic)
    # the oracle's full head layout: box [K, 80, 4] (class 0 dropped, or the agnostic column tiled), fastrcnn_head :276-280
    full_box = np.tile(box.reshape(-1, 1, 4), (1, 80, 1)) if agnostic else box.reshape(-1, 81, 4)[:, 1:]
    pc, pb = partial_oracle.gather(cls, np.ascontiguousarray(full_box), ids)
    dec, probs, pred, fprobs = frcnn.head_postprocess(pc, pb, rois, hw, cfg, multi=multi)
    rdec, rprobs, rsel, rfprobs = _restate(cls, box, rois, ids, agnostic, hw, cfg, multi)
    assert dec.shape == (300, len(ids), 4) and probs.shape == (300, len(ids) + 1)
    np.testing.assert_allclose(dec, rdec, rtol=0, atol=1e-4)
    np.testing.assert_allclose(probs, rprobs, rtol=1e-6, atol=1e-7)
    assert len(pred) == len(rsel) > 0
    assert [tuple(map(int, r)) for r in pred] == rsel
    np.testing.assert_allclose(fprobs, rfprobs, rtol=1e-6, atol=1e-7)
    labels = pred[:, 1] + 1
    assert labels.min() >= 1 and labels.max() <= len(ids)


# ---- mask quirk and driver glue on a whole oracle pass ------------------------------------------------------------------
@pytest.fixture(scope="module")
def masked_pass():
    H, W = 128, 192
    cfg = make_config(resnet_num_block=(1, 1, 1, 1), max_size=W, short_edge_size=H, add_mask=True,
                      use_partial_classes=True, **COCO)
    Wt = synth_weights(cfg, 11)
    frame = synth_frame(H, W, seed=3).astype(np.float32)
    with partial_oracle.partial_classes(cfg.partial_class_ids):
        out = frcnn.forward(cfg, Wt, frame, stages=True)
    return cfg, out


def test_mask_of_label_l_is_full_channel_l_minus_1(masked_pass):
    cfg, out = masked_pass
    labels = out["final_labels"]
    assert out["cls_logits"].shape[1] == 6 and out["mask_logits"].shape[1] == 80
    assert len(labels) and labels.min() >= 1 and labels.max() <= 5
    sel = out["mask_logits"][np.arange(len(labels)), labels - 1]
    np.testing.assert_array_equal(out["final_masks"], (1.0 / (1.0 + np.exp(-sel))).astype(np.float32))
    # the reference quirk is visible: for a label whose COCO id is not the label itself, the class's own channel differs
    ids = np.asarray(cfg.partial_class_ids)
    j = np.nonzero(ids[labels - 1] != labels)[0]
    assert len(j)
    own = out["mask_logits"][j, ids[labels[j] - 1] - 1]
    assert not np.array_equal(own, sel[j])


def test_driver_glue_yields_the_actev_sets(masked_pass):
    from object_detection_tracking_b200 import tracking
    _, out = masked_pass
    boxes, probs, labels = out["final_boxes"], out["final_probs"], out["final_labels"]
    feats = out["fpn_box_feat"]
    assert len(labels) and set(labels.tolist()) - {1, 2, 3, 4, 5} == set()
    min_conf = float(np.median(probs))
    for obj in ("Person", "Vehicle", "Bike"):
        dets = tracking.create_obj_infos(0, boxes, probs, labels, feats, PARTIAL_ID2CLASS, [obj], min_conf, 0, 1.0,
                                         is_coco_model=True, coco_to_actev_mapping=coco_obj_to_actev_obj)
        want = [j for j in range(len(labels))
                if coco_obj_to_actev_obj[PARTIAL[labels[j] - 1]] == obj and round(float(probs[j]), 7) >= min_conf]
        got = np.array([np.r_[d.tlwh, d.confidence] for d in dets]).reshape(-1, 5)
        exp = np.array([np.r_[boxes[j, :2], boxes[j, 2:] - boxes[j, :2], round(float(probs[j]), 7)] for j in want])
        np.testing.assert_allclose(got, exp.reshape(-1, 5), rtol=1e-6, atol=1e-4)
        for d, j in zip(dets, want):
            np.testing.assert_allclose(d.feature, feats[j].mean(axis=(1, 2)), rtol=1e-6)
