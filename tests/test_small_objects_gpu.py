"""Small-object branch (`use_small_object_head`) on the GPU.

person_object_relation against float64 (split and fp16 planes, R = 1 / 2 / 10 key rows, up to 400 query rows, a
zero-width query box); every step of the branch at 192x256 against so_oracle's arithmetic fed with the engine's own inputs (so
that the selections can be compared bit for bit): the selection NMS, the gathered rows, ROIAlign of unclipped boxes,
fc6 / fc7, the association, the classification and the final NMS + top-k over logits, on the 2fc, relation and attention
heads with masks, with and without association and the score filter; the main outputs byte-identical to the model
without the branch; unequal class counts; determinism and graph replay; the full-size R101 merge-prop detector; and
get_model end to end."""
import numpy as np
import pytest
import torch

import so_oracle

pytestmark = pytest.mark.gpu

SMALL = dict(num_class=17, resnet_num_block=(1, 1, 2, 2), max_size=256, short_edge_size=192)
REL = so_oracle.REL


def _cfg(**kw):
    from object_detection_tracking_b200.config import make_config
    return make_config(**dict(SMALL, use_small_object_head=True, **kw))


def _rel_weights(rng, D):
    f = np.float32
    return {REL + "/geo_emb/W": (rng.standard_normal((4, 64)) * 0.3).astype(f),
            REL + "/geo_emb/b": (rng.standard_normal(64) * 0.1).astype(f),
            REL + "/geo_conv/W": (rng.standard_normal((1, 1, 64, 16)) / 8).astype(f),
            REL + "/geo_conv/b": (rng.standard_normal(16) * 0.05).astype(f),
            REL + "/query_linear/W": (rng.standard_normal((D, D)) * np.sqrt(2.0 / D)).astype(f),
            REL + "/key_linear/W": (rng.standard_normal((D, D)) * np.sqrt(2.0 / D)).astype(f),
            REL + "/output_linear/W": (rng.standard_normal((16 * D, D)) * np.sqrt(1.0 / (16 * D))).astype(f)}


def _boxes(rng, n, W=1280, H=720):
    xy = rng.uniform(-50, [W, H], (n, 2))
    wh = rng.uniform(4, 300, (n, 2))
    return np.concatenate([xy, xy + wh], 1).astype(np.float32)


@pytest.mark.parametrize("split", [True, False])
@pytest.mark.parametrize("K,R", [(1, 1), (37, 2), (400, 10), (5, 10)])
def test_so_attend_vs_fp64(K, R, split):
    from object_detection_tracking_b200.engine import op_so_attend
    from oracle import frcnn
    D = 1024
    rng = np.random.default_rng(K * 7 + R + split)
    h = np.maximum(rng.standard_normal((K, D)), 0).astype(np.float32)
    ref = np.maximum(rng.standard_normal((R, D)), 0).astype(np.float32)
    if not split:
        h, ref = (a.astype(np.float16).astype(np.float32) for a in (h, ref))
    boxes, ref_boxes = _boxes(rng, K), _boxes(rng, R)
    boxes[0, 2] = boxes[0, 0]                    # a zero-width query box: dw = -inf, tanh saturates
    W = _rel_weights(rng, D)
    got = op_so_attend(h, boxes, ref, ref_boxes, W, split=split)
    with frcnn.exact():
        want = frcnn._np(frcnn._t(h) + so_oracle.person_object_relation(h, boxes, ref_boxes, ref, W)).astype(np.float64)
    assert np.isfinite(got).all()
    err = np.abs(got - want).max() / np.abs(want).max()
    assert err < (2e-3 if split else 1e-2), err
    if R == 1:                                   # one key row: weight 1, so every query row gets the same output_linear
        delta = got - h
        assert np.abs(delta - delta[:1]).max() <= (1e-5 if split else 1e-2) * np.abs(delta).max()


STAGES = ("head_logits", "proposal_boxes", "proposal_count", "probs", "so_sel_probs", "so_sel_boxes", "so_sel_count",
          "so_keep", "so_person_keep", "so_status", "so_k", "so_boxes", "so_roi_feat", "so_fc6", "so_fc7",
          "so_cls_logits", "so_logits")


def _run(cfg, Wt, seed, H=192, W=256, graph=True, precision="split", det=None):
    from object_detection_tracking_b200.engine import Detector
    from object_detection_tracking_b200.synth import synth_frame
    frame = synth_frame(H, W, seed=seed).astype(np.float32)
    own = det is None
    if own:
        det = Detector(cfg, 1, H, W, precision=precision, use_cuda_graph=graph)
        det.load_weights(Wt)
    try:
        out = {k: v.copy() for k, v in det.detect_host(frame[None]).items()}
        if cfg.add_mask:
            out["masks"] = det.get_masks()
        if cfg.use_small_object_head:
            out["so"] = det.get_small_objects()
            out["st"] = {s: det.get_stage(s) for s in STAGES + (("so_asso",) if cfg.use_so_association else ())}
            out["st"].update({"p%d" % (i + 2): det.get_stage("p%d" % (i + 2)) for i in range(4)})
    finally:
        if own:
            det.close()
    return out


def _levels(cfg, st, H, W):
    from object_detection_tracking_b200.config import backbone_geometry
    g = backbone_geometry(H, W, cfg)
    return [np.ascontiguousarray(st["p%d" % (i + 2)][0][:g["p"][i][0], :g["p"][i][1]].transpose(2, 0, 1))
            for i in range(4)]


def _rel_err(got, want):
    return float(np.abs(got - want).max() / max(np.abs(want).max(), 1e-30))


def check_branch(cfg, Wt, o, H, W, tol=2e-3):
    """Every step of the branch against so_oracle's arithmetic on the engine's own inputs."""
    from oracle import frcnn, tf_ops
    st, so = o["st"], o["so"]
    C, R = len(cfg.small_object_class_ids), cfg.result_per_im
    Tp = cfg.so_person_topk if cfg.use_so_association else 0
    n = int(st["proposal_count"].reshape(-1)[0])
    ncls = cfg.num_class
    lg = st["head_logits"].reshape(-1, st["head_logits"].shape[2])[:n]
    pb = st["proposal_boxes"].reshape(-1, 4)[:n]
    probs = st["probs"].reshape(-1, ncls)[:n]
    ids = list(cfg.small_object_class_ids) + ([cfg.so_person_class_id] if Tp else [])
    sel_p = st["so_sel_probs"].reshape(-1, C + 2)[:n]
    sel_b = st["so_sel_boxes"].reshape(-1, C + 1, 4)[:n]
    # select: the gathered probabilities are the head's; the unclipped decode is decode_bbox_target's
    rw = np.asarray(cfg.fastrcnn_bbox_reg_weights, np.float32)
    for s, cid in enumerate(ids):
        np.testing.assert_array_equal(sel_p[:, s + 1], probs[:, cid])
        t = (lg[:, ncls + 4 * cid: ncls + 4 * cid + 4] / rw).astype(np.float32)
        np.testing.assert_allclose(sel_b[:, s], frcnn.decode_bbox_target(t, pb), rtol=1e-6, atol=1e-3)
    # per-class NMS without a score threshold, selection order, bit-exact
    counts = st["so_sel_count"].reshape(-1)
    keep = st["so_keep"].reshape(C, R)
    for s in range(C):
        want = tf_ops.non_max_suppression(sel_b[:, s], sel_p[:, s + 1], R, cfg.fastrcnn_nms_iou_thres)
        np.testing.assert_array_equal(keep[s, :counts[s]], want)
    rows = st["so_boxes"].reshape(-1, 4)
    K = int(st["so_k"].reshape(-1)[0])
    assert int(st["so_status"].reshape(-1)[0]) == (0 if len(set(counts[:C].tolist())) == 1 else 1)
    for s in range(C):
        np.testing.assert_array_equal(rows[s * R:s * R + K], sel_b[keep[s, :K], s])
        assert not rows[s * R + K:(s + 1) * R].any()
    if Tp:
        pk = st["so_person_keep"].reshape(-1)[:counts[C]]
        np.testing.assert_array_equal(pk, tf_ops.non_max_suppression(sel_b[:, C], sel_p[:, C + 1], Tp,
                                                                      cfg.fastrcnn_nms_iou_thres))
        np.testing.assert_array_equal(rows[C * R:C * R + len(pk)], sel_b[pk, C])
    # ROIAlign of the rows on the engine's levels (unclipped boxes; outside samples read 0)
    parts = [np.arange(s * R, s * R + K) for s in range(C)]
    if Tp:
        parts.append(np.arange(C * R, C * R + int(counts[C])))
    live = np.concatenate(parts).astype(np.int64)
    roi = st["so_roi_feat"].reshape(-1, 49 * 256)[:C * R + Tp]
    if len(live):
        want, _ = frcnn.multilevel_roi_align(_levels(cfg, st, H, W), rows[live], 7, cfg.anchor_strides)
        want = want.transpose(0, 2, 3, 1).reshape(len(live), -1)
        assert _rel_err(roi[live], want) < (1e-5 if tol <= 2e-3 else 1e-3)   # split / fp16 planes
    dead = np.setdiff1d(np.arange(C * R + Tp), live)
    assert not roi[dead].any()
    # fc6 / fc7: the head's layers over the rows (float64 of the engine's ROIAlign rows)
    with frcnn.exact():
        t = frcnn._t
        x = t(roi[live].reshape(len(live), 7, 7, 256).transpose(0, 3, 1, 2).reshape(len(live), -1))
        h6 = torch.relu(x @ t(Wt["fastrcnn/fc6/W"]) + t(Wt["fastrcnn/fc6/b"]))
        fc7 = st["so_fc7"].reshape(-1, cfg.fpn_frcnn_fc_head_dim)
        h7 = torch.relu(t(st["so_fc6"].reshape(-1, cfg.fpn_frcnn_fc_head_dim)[live]) @ t(Wt["fastrcnn/fc7/W"])
                        + t(Wt["fastrcnn/fc7/b"]))
        assert _rel_err(st["so_fc6"].reshape(-1, h6.shape[1])[live], frcnn._np(h6)) < tol
        assert _rel_err(fc7[live], frcnn._np(h7)) < tol
        hidden = fc7[:C * R]
        if Tp and K:
            asso = st["so_asso"].reshape(-1, fc7.shape[1])
            pr = np.arange(C * R, C * R + int(counts[C]))
            for s in range(C):
                q = np.arange(s * R, s * R + K)
                want = frcnn._np(t(fc7[q]) + so_oracle.person_object_relation(fc7[q], rows[q], rows[pr], fc7[pr], Wt))
                assert _rel_err(asso[q], want) < tol
            hidden = asso[:C * R]
        cls = st["so_cls_logits"].reshape(C * R, -1)
        for s in range(C):
            q = np.arange(s * R, s * R + K)
            nm = "fastrcnn/small_objects/small_object_classification_c%d/" % (s + 1)
            want = frcnn._np(t(hidden[q]) @ t(Wt[nm + "W"]) + t(Wt[nm + "b"]))
            if K:
                assert np.abs(cls[q, 2 * s:2 * s + 2] - want).max() <= tol * max(np.abs(want).max(), 1.0)
    # the rebuilt logits, exactly, and the final selection over them, bit-exact
    fl = st["so_logits"].reshape(R, C + 1)[:K]
    col = np.stack([cls[s * R:s * R + K, 2 * s + 1] for s in range(C)], 1) if K else np.zeros((0, C), np.float32)
    np.testing.assert_array_equal(fl[:, 1:], col)
    bg = np.zeros(K, np.float32)
    for s in range(C):
        bg = (bg + cls[s * R:s * R + K, 2 * s]).astype(np.float32)
    np.testing.assert_array_equal(fl[:, 0], (bg / np.float32(C)).astype(np.float32))
    boxes = frcnn.clip_boxes(np.stack([rows[s * R:s * R + K] for s in range(C)], 1), (H, W)) if K else \
        np.zeros((0, C, 4), np.float32)
    import copy
    fcfg = copy.copy(cfg)
    if not cfg.use_so_score_thres:
        fcfg.result_score_thres = -np.inf
    pred, fprobs = frcnn.fastrcnn_predictions(boxes, fl, fcfg)
    np.testing.assert_array_equal(so["labels"], pred[:, 1] + 1)
    np.testing.assert_array_equal(so["probs"], fprobs)
    np.testing.assert_array_equal(so["boxes"], boxes[pred[:, 0], pred[:, 1]] if len(pred) else np.zeros((0, 4)))
    return dict(K=K, n=len(so["probs"]), neg=int((so["probs"] < 0).sum()), counts=counts.tolist(),
                outside=int(((rows[live] < 0) | (rows[live, 2:3] > W) | (rows[live, 3:4] > H)).any(1).sum()))


PARITY = {
    "2fc": dict(),
    "2fc_assoc": dict(use_so_association=True),
    "2fc_assoc_thres": dict(use_so_association=True, use_so_score_thres=True),
    "relation_assoc": dict(add_relation_nn=True, use_so_association=True),
    "att_assoc_mask": dict(use_att_frcnn_head=True, use_so_association=True, add_mask=True),
    "gn_thres": dict(use_gn=True, use_so_score_thres=True),
}


@pytest.mark.parametrize("name", sorted(PARITY))
def test_stage_parity_small(name):
    """Each step at 192x256 on the engine's own inputs; the main outputs byte-identical to the model without the branch.
    result_per_im 20 keeps every small class saturated on these frames (the synthetic head keeps hundreds of boxes per
    class without a score threshold)."""
    from object_detection_tracking_b200.synth import synth_weights
    cfg = _cfg(result_per_im=20, **PARITY[name])
    Wt = synth_weights(cfg, 5)
    off = _cfg(result_per_im=20, **PARITY[name])
    off.use_small_object_head = False
    for seed in (1, 2):
        o = _run(cfg, Wt, seed)
        rec = check_branch(cfg, Wt, o, 192, 256)
        print(name, seed, rec)
        assert rec["K"] == 20 and (rec["n"] > 0 or cfg.use_so_score_thres)
        o_off = _run(off, Wt, seed)
        for k in ("boxes", "probs", "labels", "valid", "feat") + (("masks",) if cfg.add_mask else ()):
            np.testing.assert_array_equal(o[k], o_off[k], err_msg=k)


def test_logits_not_probs_and_filter():
    """The final scores are the rebuilt logits: negative ones are selected without the filter and dropped with it."""
    from object_detection_tracking_b200.synth import synth_weights
    cfg = _cfg(result_per_im=20)
    Wt = synth_weights(cfg, 5)
    o = _run(cfg, Wt, 1)
    rec = check_branch(cfg, Wt, o, 192, 256)
    assert rec["neg"] > 0, rec
    cfg_t = _cfg(result_per_im=20, use_so_score_thres=True)
    o_t = _run(cfg_t, Wt, 1)
    check_branch(cfg_t, Wt, o_t, 192, 256)
    assert (o_t["so"]["probs"] > cfg_t.result_score_thres).all()
    assert len(o_t["so"]["probs"]) < len(o["so"]["probs"])


def test_unequal_counts_then_next_frame():
    """Counts forced apart through the head logits and a re-run of the post phases: status 1, K = 0, no output, the main
    outputs still there; the next frame is right again."""
    from object_detection_tracking_b200.engine import Detector
    from object_detection_tracking_b200.synth import synth_frame, synth_weights
    cfg = _cfg(result_per_im=20, use_so_association=True)
    Wt = synth_weights(cfg, 5)
    det = Detector(cfg, 1, 192, 256)
    try:
        det.load_weights(Wt)
        first = _run(cfg, Wt, 1, det=det)
        lg = det.get_stage("head_logits").copy()
        n = int(det.get_stage("proposal_count").reshape(-1)[0])
        cid = cfg.small_object_class_ids[1]
        # class 2's boxes of proposals 3.. all decode to (about) proposal 0's box: its NMS keeps at most 3 of them
        pb = det.get_stage("proposal_boxes").reshape(-1, 4)[:n].astype(np.float64)
        w, h = pb[:, 2] - pb[:, 0], pb[:, 3] - pb[:, 1]
        cx, cy = pb[:, 0] + w / 2, pb[:, 1] + h / 2
        rw = cfg.fastrcnn_bbox_reg_weights
        t = np.stack([(cx[0] - cx) / w * rw[0], (cy[0] - cy) / h * rw[1], np.log(w[0] / w) * rw[2],
                      np.log(h[0] / h) * rw[3]], 1)
        lg[0, 3:n, 17 + 4 * cid:17 + 4 * cid + 4] = t[3:].reshape(n - 3, 4, 1)
        det.set_stage("head_logits", lg)
        det.run_phases((1 << 6) | (1 << 7))
        so = det.get_small_objects()
        assert so["status"] == 1 and len(so["probs"]) == 0, so
        assert int(det.get_stage("so_k").reshape(-1)[0]) == 0
        assert int(det.get_stage("final_count").reshape(-1)[0]) > 0
        again = _run(cfg, Wt, 1, det=det)
        assert again["so"]["status"] == 0
        for k in ("boxes", "probs", "labels"):
            np.testing.assert_array_equal(again["so"][k], first["so"][k])
    finally:
        det.close()


def test_determinism_and_graph_equals_eager():
    from object_detection_tracking_b200.synth import synth_weights
    cfg = _cfg(result_per_im=20, use_so_association=True)
    Wt = synth_weights(cfg, 5)
    a, b, c = _run(cfg, Wt, 3), _run(cfg, Wt, 3), _run(cfg, Wt, 3, graph=False)
    for o in (b, c):
        for k in ("boxes", "probs", "labels"):
            np.testing.assert_array_equal(o["so"][k], a["so"][k])
        np.testing.assert_array_equal(o["st"]["so_asso"], a["st"]["so_asso"])


def test_fp16_precision():
    from object_detection_tracking_b200.synth import synth_weights
    cfg = _cfg(result_per_im=20, use_so_association=True)
    Wt = synth_weights(cfg, 5)
    o = _run(cfg, Wt, 1, precision="fp16")
    rec = check_branch(cfg, Wt, o, 192, 256, tol=2e-2)
    assert rec["K"] == 20


def test_full_size_r101_merge_prop():
    """R101 merge-prop (num_class 17) at 720x1280, batch 1, rpn 1000, result_per_im 100, with association: every step
    against the oracle's arithmetic on the engine's inputs.  Every small class keeps 100 boxes on this frame."""
    from object_detection_tracking_b200.config import make_config
    from object_detection_tracking_b200.synth import synth_weights
    cfg = make_config(num_class=17, use_small_object_head=True, use_so_association=True, rpn_test_post_nms_topk=1000)
    Wt = synth_weights(cfg, 5)
    o = _run(cfg, Wt, 1, H=720, W=1280)
    rec = check_branch(cfg, Wt, o, 720, 1280)
    print(rec)
    assert rec["K"] == 100 and rec["n"] == 100


def test_get_model_session_run():
    from object_detection_tracking_b200.backend import Session, get_model
    from object_detection_tracking_b200.synth import synth_frame, synth_weights
    cfg = _cfg(result_per_im=20, use_so_association=True)
    Wt = synth_weights(cfg, 5)
    model = get_model(cfg)
    model.set_weights(Wt)
    frame = synth_frame(192, 256, seed=1).astype(np.float32)
    sess = Session()
    fb, fl, fp, sb, sl, sp = sess.run([model.final_boxes, model.final_labels, model.final_probs, model.so_final_boxes,
                                       model.so_final_labels, model.so_final_probs], model.get_feed_dict_forward(frame))
    assert sb.dtype == np.float32 and sl.dtype == np.int64 and sp.dtype == np.float32
    assert len(sb) == len(sl) == len(sp) > 0 and sl.min() >= 1 and sl.max() <= 4
    o = _run(cfg, Wt, 1)
    np.testing.assert_array_equal(sp, o["so"]["probs"])
    np.testing.assert_array_equal(fp, o["probs"][0, :len(fp)])
    off = _cfg(result_per_im=20)
    off.use_small_object_head = False
    m2 = get_model(off)
    m2.set_weights(Wt)
    with pytest.raises(KeyError, match="use_small_object_head"):
        sess.run([m2.so_final_boxes], m2.get_feed_dict_forward(frame))
