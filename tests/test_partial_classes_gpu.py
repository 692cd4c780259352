"""--use_partial_classes on the GPU: the COCO-81 detector whose box head keeps only the selected classes (models.py:807-843,
batch graph :2256-2303, masks :934-962).

* The stages up to fc7 do not depend on the selection, and the partial head's logits are the full head's columns.
* Selecting all 80 classes in id order is the full model, byte for byte.
* Parity with the oracle's partial graph (tests/partial_oracle.py) at the headline geometry (R50 COCO-81, 720x1280,
  batch 1 and the batch-8 graph) under the bars of tests/test_baseline_configs_gpu.py, and at small geometries with the
  mask head, the class-agnostic head and a single class.
* The drop-in path: a frozen graph of the 81-class checkpoint through backend.get_model, Session.run and
  tracking.create_obj_infos with the driver's partial class table."""
import numpy as np
import pytest

import partial_oracle
from test_baseline_configs_gpu import assert_final, exact_margins, final_margins, log_margins, run_single

pytestmark = pytest.mark.gpu

COCO = dict(num_class=81, use_dilations=False, version=2)
R50 = dict(resnet_num_block=(3, 4, 6, 3), **COCO)
SMALL = dict(resnet_num_block=(1, 1, 2, 1), max_size=384, short_edge_size=256, **COCO)
PARTIAL = ["person", "car", "bus", "truck", "bicycle"]
PARTIAL_ID2CLASS = {i: n for i, n in enumerate(["BG"] + PARTIAL)}


def _cfg(**kw):
    from object_detection_tracking_b200.config import make_config
    return make_config(**kw)


def _names(ids):
    from object_detection_tracking_b200.class_ids import coco_obj_id_to_class
    return [coco_obj_id_to_class[i] for i in ids]


# every stage before the box head's output layer
UPSTREAM_STAGES = (["c1", "pool", "c2", "c3", "c4", "c5", "p2", "p3", "p4", "p5", "p6"] + ["rpn_l%d" % i for i in range(5)]
                   + ["lvl_boxes", "lvl_scores", "lvl_count", "proposal_boxes", "proposal_scores", "proposal_count",
                      "roi_feat", "fc6", "fc7"])


def _full_columns(ids, agnostic):
    """The columns of the full (81-class) fused head output that the partial one holds, in its order: class [0] + ids,
    then per kept class (class 0's slot first) its 4 box columns -- or the 4 class-agnostic box columns."""
    cls = [0] + list(ids)
    box = [81 + k for k in range(4)] if agnostic else [81 + c * 4 + k for c in cls for k in range(4)]
    return cls + box


@pytest.mark.parametrize("agnostic", [False, True])
@pytest.mark.parametrize("ids", [(1, 3, 6, 8, 2), (80, 40, 7)])
def test_upstream_unchanged_and_head_columns_bit_identical(ids, agnostic):
    from object_detection_tracking_b200.engine import Detector
    from object_detection_tracking_b200.synth import synth_frame, synth_weights
    H, W = 256, 384
    full_cfg = _cfg(use_frcnn_class_agnostic=agnostic, **R50)
    part_cfg = _cfg(use_frcnn_class_agnostic=agnostic, use_partial_classes=True, partial_classes=_names(ids), **R50)
    assert part_cfg.partial_class_ids == ids
    Wt = synth_weights(full_cfg, 4321)
    frame = synth_frame(H, W, seed=11).astype(np.float32)
    dets = []
    try:
        for cfg in (full_cfg, part_cfg):
            d = Detector(cfg, 1, H, W, precision="split", use_cuda_graph=False)
            dets.append(d)
            d.load_weights(Wt)
            d.set_stage("image", frame[None])
            d.run_phases(255)
        full, part = dets
        for name in UPSTREAM_STAGES:
            a, b = full.get_stage(name), part.get_stage(name)
            assert a.shape == b.shape and a.tobytes() == b.tobytes(), name
        fl, pl = full.get_stage("head_logits"), part.get_stage("head_logits")
        cols = _full_columns(ids, agnostic)
        assert pl.shape[2] >= len(cols) and pl.shape[2] < fl.shape[2]
        want, got = fl[:, :, cols], pl[:, :, :len(cols)]
        rec = {"config": "partial-columns", "ids": list(ids), "agnostic": agnostic, "cols": len(cols),
               "ld_full": int(fl.shape[2]), "ld_partial": int(pl.shape[2]),
               "head_logits_maxabs": float(np.abs(got.astype(np.float64) - want).max())}
        log_margins(rec)
        assert got.tobytes() == want.tobytes(), rec
        assert part.get_stage("probs").shape[2] == len(ids) + 1
        assert part.get_stage("dec_boxes").shape[2] == len(ids)
    finally:
        for d in dets:
            d.close()


def test_all_80_classes_in_id_order_reproduce_the_full_model():
    from object_detection_tracking_b200.engine import Detector
    from object_detection_tracking_b200.synth import synth_frame, synth_weights
    H, W, B = 256, 384, 2
    full_cfg = _cfg(**R50)
    every = _cfg(use_partial_classes=True, partial_classes=_names(range(1, 81)), **R50)
    assert every.partial_class_ids == tuple(range(1, 81))
    Wt = synth_weights(full_cfg, 4321)
    frames = np.stack([synth_frame(H, W, seed=30 + b) for b in range(B)]).astype(np.float32)
    outs, dets = [], []
    try:
        for cfg in (full_cfg, every):
            d = Detector(cfg, B, H, W, precision="split", use_cuda_graph=True)
            dets.append(d)
            d.load_weights(Wt)
            o = d.detect_host(frames)
            outs.append({**o, **{s: d.get_stage(s) for s in ("head_logits", "probs", "dec_boxes", "fpn_box_feat")}})
        for k in outs[0]:
            assert outs[0][k].tobytes() == outs[1][k].tobytes(), k
        assert int(outs[0]["valid"].sum()) > 0
    finally:
        for d in dets:
            d.close()


def test_headline_r50_coco81_partial_720x1280():
    """The reference's headline model (--is_coco_model --use_partial_classes --resnet50, version 2, rpn300) on two
    full-size frames, batch 1, against the oracle's partial graph: the bars of test_c4_r50_coco81_720x1280."""
    cfg = _cfg(use_partial_classes=True, **R50)
    assert cfg.partial_class_ids == (1, 3, 6, 8, 2) and cfg.rpn_test_post_nms_topk == 300
    with partial_oracle.partial_classes(cfg.partial_class_ids):
        recs = run_single(cfg, (11, 12), 720, 1280, "C4-partial", weight_seed=4321)
    assert all(r["final"] > 0 for r in recs)


def test_headline_batch8_multi_semantics():
    """The batch graph (Mask_RCNN_FPN_multi, models.py:2256-2303): the same gather, then the combined NMS over the 5
    classes, against oracle.frcnn.forward_multi with the partial gather."""
    from object_detection_tracking_b200.engine import Detector
    from object_detection_tracking_b200.synth import synth_frame, synth_weights
    from oracle import frcnn
    H, W, B = 720, 1280, 8
    cfg = _cfg(use_partial_classes=True, im_batch_size=B, **R50)
    Wt = synth_weights(cfg, 4321)
    frames = np.stack([synth_frame(H, W, seed=40 + s) for s in range(B)]).astype(np.float32)
    det = Detector(cfg, B, H, W, precision="split", use_cuda_graph=True, multi_semantics=True)
    det.load_weights(Wt)
    try:
        out = det.detect_host(frames)
        with partial_oracle.partial_classes(cfg.partial_class_ids):
            ref = frcnn.forward_multi(cfg, Wt, list(frames), stages=True)
            with frcnn.exact():
                ref64 = frcnn.forward_multi(cfg, Wt, list(frames), stages=False)
    finally:
        det.close()
    recs = []
    for b in range(B):
        rec = {"config": "C2-partial-r50", "image": b}
        r, rr, r64 = int(out["valid"][b]), int(ref["final_valid_indices"][b]), int(ref64["final_valid_indices"][b])
        got = (out["labels"][b, :r], out["boxes"][b, :r], out["probs"][b, :r])
        o32 = (ref["final_labels"][b, :rr], ref["final_boxes"][b, :rr], ref["final_probs"][b, :rr])
        final_margins(*got, *o32, rec)
        exact_margins(*got, o32, (ref64["final_labels"][b, :r64], ref64["final_boxes"][b, :r64],
                                  ref64["final_probs"][b, :r64]), rec)
        log_margins(rec)
        recs.append(rec)
    for rec in recs:
        assert_final(rec)
    assert all(set(out["labels"][b, :int(out["valid"][b])].tolist()) <= {1, 2, 3, 4, 5} for b in range(B))


@pytest.mark.parametrize("agnostic", [False, True])
def test_small_partial_parity(agnostic):
    cfg = _cfg(use_partial_classes=True, use_frcnn_class_agnostic=agnostic, **SMALL)
    with partial_oracle.partial_classes(cfg.partial_class_ids):
        run_single(cfg, (5, 6), 256, 384, "small-partial" + ("-agnostic" if agnostic else ""), weight_seed=77)


@pytest.mark.parametrize("result_per_im", [100, 1])
def test_one_class_selection(result_per_im):
    """partial_classes = ["person"]: one class-NMS block per image, and with result_per_im 1 a final top-k over one key."""
    cfg = _cfg(use_partial_classes=True, partial_classes=["person"], result_per_im=result_per_im, **SMALL)
    assert cfg.partial_class_ids == (1,)
    with partial_oracle.partial_classes(cfg.partial_class_ids):
        recs = run_single(cfg, (5, 7), 256, 384, "one-class-R%d" % result_per_im, weight_seed=77)
    assert all(r["final"] > 0 for r in recs)


def test_masks_follow_the_reference_channel_choice():
    """add_mask + partial: final_masks against the oracle, whose mask for partial label l is channel l - 1 of the 80
    COCO channels (models.py:954-958), and the engine's mask logits keep all 80 channels."""
    from object_detection_tracking_b200.engine import Detector
    from object_detection_tracking_b200.synth import synth_frame, synth_weights
    from oracle import frcnn
    H, W = 256, 384
    cfg = _cfg(use_partial_classes=True, add_mask=True, **SMALL)
    Wt = synth_weights(cfg, 77)
    frame = synth_frame(H, W, seed=5).astype(np.float32)
    det = Detector(cfg, 1, H, W, precision="split", use_cuda_graph=True)
    det.load_weights(Wt)
    try:
        out = det.detect_host(frame[None])
        masks = det.get_masks()[0]
        ml = det.get_stage("mask_logits")
    finally:
        det.close()
    with partial_oracle.partial_classes(cfg.partial_class_ids):
        ref = frcnn.forward(cfg, Wt, frame, stages=True)
    r = int(out["valid"][0])
    assert r == len(ref["final_labels"]) > 0
    labels = out["labels"][0, :r]
    assert labels.min() >= 1 and labels.max() <= 5
    d = (np.abs(out["boxes"][0, :r, None, :] - ref["final_boxes"][None, :, :]).max(-1)
         + 10.0 * (labels[:, None] != ref["final_labels"][None, :]))
    match = d.argmin(1)
    rec = {"config": "mask-partial", "final": r, "box_match": float(d.min(1).max()),
           "mask_maxabs": float(np.abs(masks[:r] - ref["final_masks"][match]).max())}
    log_margins(rec)
    assert rec["box_match"] < 2e-3 and rec["mask_maxabs"] < 2e-4
    assert (masks[r:] == 0).all()
    ld = ml.shape[2]
    assert ld >= 80
    got = ml.reshape(-1, 14, 14, 2, 2, ld)[:r, ..., :80].transpose(0, 5, 1, 3, 2, 4).reshape(r, 80, 28, 28)
    own = got[np.arange(r), labels - 1]
    np.testing.assert_allclose(masks[:r], 1.0 / (1.0 + np.exp(-own.astype(np.float64))), rtol=0, atol=1e-6)
    assert (np.asarray(cfg.partial_class_ids)[labels - 1] != labels).any()      # the quirk is exercised


def _write_frozen_graph(W, path):
    import test_importer_cpu as pb
    graph = pb._node("image", "Placeholder")
    for k, v in sorted(W.items()):
        graph += pb._node(k, "Const", pb._tensor_proto(v, "content"))
    with open(path, "wb") as f:
        f.write(graph)


def test_frozen_partial_model_through_get_model_and_the_tracker(tmp_path):
    """The headline command's path: --is_load_from_pb --use_partial_classes with the 81-class frozen graph ->
    get_model -> Session.run -> create_obj_infos with the driver's partial targetid2class (no KeyError, ActEV names)."""
    from object_detection_tracking_b200 import tracking
    from object_detection_tracking_b200.backend import Session, get_model
    from object_detection_tracking_b200.class_ids import coco_obj_to_actev_obj
    from object_detection_tracking_b200.synth import synth_frame, synth_weights
    H, W = 256, 384
    base = _cfg(**SMALL)
    path = str(tmp_path / "coco_partial.pb")
    _write_frozen_graph(synth_weights(base, 77), path)
    frames = [synth_frame(H, W, seed=5 + i).astype(np.float32) for i in range(2)]
    sess = Session()

    cfg = _cfg(use_partial_classes=True, is_load_from_pb=True, load_from=path, **SMALL)
    model = get_model(cfg, gpuid=0)
    fetches = [model.final_boxes, model.final_labels, model.final_probs, model.fpn_box_feat]
    boxes, labels, probs, feat = sess.run(fetches, feed_dict=model.get_feed_dict_forward(frames[0]))
    assert labels.dtype == np.int64 and len(labels) > 0 and labels.min() >= 1 and labels.max() <= 5
    assert len(feat) == len(boxes) == len(probs) == len(labels)
    assert model.detector(1, H, W).get_stage("probs").shape[2] == 6         # the 6-way softmax
    for obj in ("Person", "Vehicle", "Bike"):
        dets = tracking.create_obj_infos(0, boxes, probs, labels, feat, PARTIAL_ID2CLASS, [obj], 0.0, 0, 1.0,
                                         is_coco_model=True, coco_to_actev_mapping=coco_obj_to_actev_obj)
        assert len(dets) == sum(coco_obj_to_actev_obj[PARTIAL[l - 1]] == obj for l in labels)

    mcfg = _cfg(use_partial_classes=True, is_load_from_pb=True, load_from=path, im_batch_size=2, **SMALL)
    multi = get_model(mcfg, gpuid=0, is_multi=True)
    fetches = [multi.final_boxes, multi.final_labels, multi.final_probs, multi.final_valid_indices, multi.fpn_box_feat]
    mb, ml, mp, mv, mf = sess.run(fetches, feed_dict=multi.get_feed_dict_forward_multi(frames))
    assert ml.dtype == np.float32 and ml.shape == (2, cfg.result_per_im)
    for b in range(2):
        v = int(mv[b])
        assert v > 0 and set(ml[b, :v].tolist()) <= {1.0, 2.0, 3.0, 4.0, 5.0} and (ml[b, v:] == 0).all()
    assert len(mf) == int(mv.sum())
