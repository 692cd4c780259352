"""Relation-network box head (`add_relation_nn`) on the GPU.

One relation module against float64 torch (split and fp16 planes, padded rows, an image alone and in a batch), stage
parity with the oracle at a small geometry (class-specific and class-agnostic heads, GroupNorm, the conv head taking
precedence), the full-size R101 detector against the oracle and its exact() evaluation (DESIGN 2.1), that the relation
path changes the detections, determinism (two passes, graph replay, batch parts, an image alone) and get_model."""
import numpy as np
import pytest

import relation_oracle

pytestmark = pytest.mark.gpu

REL = dict(add_relation_nn=True)
SMALL = dict(resnet_num_block=(1, 1, 2, 2), max_size=256, short_edge_size=192)


def _cfg(**kw):
    from object_detection_tracking_b200.config import make_config
    return make_config(**kw)


def module_weights(D, seed):
    from object_detection_tracking_b200.synth import synth_weights
    w = synth_weights(_cfg(fpn_frcnn_fc_head_dim=D, resnet_num_block=(1, 1, 1, 1), **REL), seed)
    return {k[len("fastrcnn/RM_r1/"):]: v for k, v in w.items() if k.startswith("fastrcnn/RM_r1/")}


def ref_relation(h, boxes, count, w):
    """float64 torch: h + relation_network(h[:n], boxes[:n]) per image, rows >= n unchanged."""
    out = h.astype(np.float64).copy()
    W = {"m/" + k: v for k, v in w.items()}
    from oracle import frcnn
    with frcnn.exact():
        for b in range(h.shape[0]):
            n = int(count[b])
            if n:
                out[b, :n] += relation_oracle.relation(frcnn._t(h[b, :n]), boxes[b, :n], W, "m").numpy()
    return out


def quantize(a, split):
    return a.astype(np.float32) if split else a.astype(np.float16).astype(np.float32)


@pytest.mark.parametrize("K,split", [(1, True), (7, False), (7, True), (300, True), (300, False), (1000, True)])
def test_relation_module_vs_fp64(K, split):
    from object_detection_tracking_b200.engine import op_relation
    D, B = 1024, 3
    rng = np.random.default_rng(K * 10 + split)
    w = module_weights(D, 40 + K)
    h = quantize(np.maximum(rng.standard_normal((B, K, D)) * 0.7, 0) + rng.uniform(0, 0.1, (B, 1, D)), split)
    xy = rng.uniform(0, 1000, (B, K, 2))
    wh = rng.uniform(8, 300, (B, K, 2))
    boxes = np.concatenate([xy, xy + wh], -1).astype(np.float32)
    if K >= 3:
        boxes[:, 1] = boxes[:, 0]                                          # a duplicate box: equal centres and sizes
    count = np.array([K, max(1, K - K // 3), 0 if K > 1 else 1], np.int32)
    got = op_relation(h, boxes, count, w, split=split)
    ref = ref_relation(h, boxes, count, w)
    assert np.isfinite(got).all()
    err = np.abs(got - ref).max() / np.abs(ref).max()
    # three split-precision GEMMs in a row (query|key, P.V, output_linear) and P in the planes: ~1e-5 of the largest output
    # at K = 1000 in split precision, fp16 planes everywhere in fp16
    assert err < (1e-4 if split else 4e-3), err
    for b in range(B):                     # padded rows: h itself, as the planes hold it (exact in fp16, ~2^-22 in split)
        pad_err = np.abs(got[b, count[b]:] - h[b, count[b]:])
        assert (pad_err <= (2.0 ** -19 if split else 0.0) * np.abs(h[b, count[b]:])).all(), pad_err.max()
    assert np.abs(got[0] - h[0]).max() > 0.05                              # the module is not a no-op
    # an image alone is bit-identical to the same image in the batch
    one = op_relation(h[1:2], boxes[1:2], count[1:2], w, split=split)
    np.testing.assert_array_equal(one, got[1:2])


def _run_small(cfg, seed, weight_seed=99, H=192, W=256):
    """Batch-1 context at the small geometry; returns the engine's and the oracle's (float32) head rows and detections."""
    from object_detection_tracking_b200.engine import Detector
    from object_detection_tracking_b200.synth import synth_frame, synth_weights
    Wt = synth_weights(cfg, weight_seed)
    frame = synth_frame(H, W, seed=seed).astype(np.float32)
    det = Detector(cfg, 1, H, W, precision="split")
    try:
        det.load_weights(Wt)
        out = det.detect_host(frame[None], want_feat=False)
        pc = int(det.get_stage("proposal_count").reshape(-1)[0])
        stages = {s: det.get_stage(s).reshape(-1, cfg.fpn_frcnn_fc_head_dim)[:pc] for s in ("rm_r1", "rm_r2")} \
            if relation_oracle.use_relation(cfg) else {}
    finally:
        det.close()
    ref = relation_oracle.forward(cfg, Wt, frame, stages=True)
    return out, stages, ref, dict(relation_oracle.LAST)


def _stage_parity(cfg, seeds, tag, weight_seed=99):
    from test_baseline_configs_gpu import run_single
    with relation_oracle.graph(cfg):
        return run_single(cfg, seeds, 192, 256, tag, weight_seed=weight_seed)


@pytest.mark.parametrize("agnostic", [False, True])
def test_stage_parity_small_relation(agnostic):
    """Backbone to detections against relation_oracle at 192x256 (DESIGN 2.1 bars), and both module sums row by row."""
    cfg = _cfg(use_frcnn_class_agnostic=agnostic, **dict(SMALL, **REL))
    recs = _stage_parity(cfg, (3, 4), "relation_small_agn%d" % agnostic)
    assert recs[0]["final"] > 0
    _, st, ref, last = _run_small(cfg, 3)
    for s in ("rm_r1", "rm_r2"):
        assert st[s].shape == last[s].shape
        err = np.abs(st[s] - last[s]).max() / np.abs(last[s]).max()
        assert err < 1e-4, (s, err)


def test_stage_parity_small_gn_relation():
    cfg = _cfg(use_gn=True, **dict(SMALL, **REL))
    _stage_parity(cfg, (5,), "gn_relation_small", weight_seed=17)


def test_conv_head_takes_precedence():
    """add_relation_nn with use_conv_frcnn_head is the conv-head model: same detections, bit for bit."""
    base = dict(SMALL, use_gn=True, use_conv_frcnn_head=True)
    a, _, _, _ = _run_small(_cfg(**base), 6, weight_seed=17)
    b, _, _, _ = _run_small(_cfg(**dict(base, **REL)), 6, weight_seed=17)
    for k in ("boxes", "probs", "labels", "valid"):
        np.testing.assert_array_equal(a[k], b[k])


FULL = dict(resnet_num_block=(3, 4, 23, 3), num_class=15, use_frcnn_class_agnostic=True, use_dilations=True, **REL)


def test_relation_r101_720x1280_batch1():
    """R101 dilated, class-agnostic + relation head, 720x1280, single-image semantics: counts and labels exact, boxes by
    the rule of DESIGN 2.1."""
    recs = _stage_parity(_cfg(**FULL), (11,), "relation-R101", weight_seed=1234)
    assert recs[0]["final"] > 0


def test_relation_r101_720x1280_batch8_multi():
    from test_baseline_configs_gpu import exact_margins, final_margins, log_margins
    from object_detection_tracking_b200.engine import Detector
    from object_detection_tracking_b200.synth import synth_frame, synth_weights
    from oracle import frcnn
    H, W, B = 720, 1280, 8
    cfg = _cfg(im_batch_size=B, **FULL)
    Wt = synth_weights(cfg, 1234)
    frames = np.stack([synth_frame(H, W, seed=40 + s) for s in range(B)]).astype(np.float32)
    det = Detector(cfg, B, H, W, precision="split", use_cuda_graph=True, multi_semantics=True)
    try:
        det.load_weights(Wt)
        out = det.detect_host(frames)
    finally:
        det.close()
    ref = relation_oracle.forward_multi(cfg, Wt, list(frames), stages=False)
    with frcnn.exact():
        ref64 = relation_oracle.forward_multi(cfg, Wt, list(frames), stages=False)
    for b in range(B):
        rec = {"config": "relation-R101-multi8", "image": b}
        r, rr, r64 = int(out["valid"][b]), int(ref["final_valid_indices"][b]), int(ref64["final_valid_indices"][b])
        got = (out["labels"][b, :r], out["boxes"][b, :r], out["probs"][b, :r])
        final_margins(*got, ref["final_labels"][b, :rr], ref["final_boxes"][b, :rr], ref["final_probs"][b, :rr], rec)
        exact_margins(*got, (ref["final_labels"][b, :rr], ref["final_boxes"][b, :rr], ref["final_probs"][b, :rr]),
                      (ref64["final_labels"][b, :r64], ref64["final_boxes"][b, :r64], ref64["final_probs"][b, :r64]),
                      rec)
        log_margins(rec)
        assert rec["final"] == rec["final_ref"] and rec["labels_sorted_equal"], rec
        assert rec["gpu_to_exact"] < 1e-3, rec
        assert rec["final"] > 0


def test_detections_depend_on_the_relation_head():
    """The same weights with add_relation_nn off (the RM arrays then ignored) give other detections."""
    cfg = _cfg(**dict(SMALL, use_frcnn_class_agnostic=True, **REL))
    a, _, _, _ = _run_small(cfg, 7)
    b, _, _, _ = _run_small(_cfg(**dict(SMALL, use_frcnn_class_agnostic=True)), 7)
    n = min(int(a["valid"][0]), int(b["valid"][0]))
    assert int(a["valid"][0]) != int(b["valid"][0]) or np.abs(a["probs"][0, :n] - b["probs"][0, :n]).max() > 1e-3


HEAD = ["rm_r1", "rm_r2", "head_logits", "proposal_boxes", "proposal_count"]


def _outputs(cfg, Wt, frames, **kw):
    from object_detection_tracking_b200.engine import Detector
    det = Detector(cfg, len(frames), frames.shape[1], frames.shape[2], precision="split", multi_semantics=True, **kw)
    try:
        det.load_weights(Wt)
        a = {k: v.copy() for k, v in det.detect_host(frames).items()}
        b = det.detect_host(frames)
        for k in a:
            np.testing.assert_array_equal(a[k], b[k], err_msg="second pass differs: " + k)
        K = cfg.rpn_test_post_nms_topk
        for s in HEAD:
            v = det.get_stage(s)
            a[s] = v.reshape(len(frames), K, -1) if s.startswith("rm") else v
        return a
    finally:
        det.close()


def test_determinism_graph_batch_parts_and_single_images(monkeypatch):
    """Two passes are bit-identical, graph replay equals eager, B2_SPLIT=1 / 2 / 4 agree bit for bit, and every image of
    the batch of 8 gets the module sums and head logits it gets alone."""
    from object_detection_tracking_b200.synth import synth_frame, synth_weights
    cfg = _cfg(im_batch_size=8, use_frcnn_class_agnostic=True, **dict(SMALL, **REL))
    Wt = synth_weights(cfg, 99)
    frames = np.stack([synth_frame(192, 256, seed=60 + s) for s in range(8)]).astype(np.float32)
    dual = _outputs(cfg, Wt, frames, use_cuda_graph=True)
    eager = _outputs(cfg, Wt, frames, use_cuda_graph=False)
    monkeypatch.setenv("B2_SPLIT", "1")
    single = _outputs(cfg, Wt, frames, use_cuda_graph=True)
    monkeypatch.setenv("B2_SPLIT", "4")
    quarter = _outputs(cfg, Wt, frames, use_cuda_graph=True)
    for other in (eager, single, quarter):
        for k in dual:
            np.testing.assert_array_equal(dual[k], other[k], err_msg=k)
    assert int(dual["valid"].sum()) > 0
    monkeypatch.delenv("B2_SPLIT")
    K = cfg.rpn_test_post_nms_topk
    for k in range(8):
        alone = _outputs(cfg, Wt, frames[k:k + 1], use_cuda_graph=False)
        for s in ("rm_r1", "rm_r2"):
            np.testing.assert_array_equal(dual[s][k:k + 1], alone[s], err_msg="image %d, %s" % (k, s))
        np.testing.assert_array_equal(dual["head_logits"][k:k + 1], alone["head_logits"], err_msg="image %d" % k)
        for o in ("boxes", "probs", "labels", "valid"):
            np.testing.assert_array_equal(dual[o][k:k + 1], alone[o], err_msg="image %d, %s" % (k, o))


@pytest.mark.parametrize("is_multi", [False, True])
def test_get_model_relation(is_multi):
    from object_detection_tracking_b200.backend import Session, get_model
    from object_detection_tracking_b200.synth import synth_frame, synth_weights
    cfg = _cfg(**dict(SMALL, **REL))
    Wt = synth_weights(cfg, 99)
    frames = [synth_frame(192, 256, seed=70 + s).astype(np.float32) for s in range(2 if is_multi else 1)]
    model = get_model(cfg, is_multi=is_multi)
    model.set_weights(Wt)
    fetches = [model.final_boxes, model.final_labels, model.final_probs, model.final_valid_indices]
    if is_multi:
        boxes, labels, probs, valid = Session().run(fetches, feed_dict=model.get_feed_dict_forward_multi(frames))
        ref = relation_oracle.forward_multi(cfg, Wt, frames)
        per = [(boxes[b, :valid[b]], labels[b, :valid[b]], probs[b, :valid[b]], ref["final_boxes"][b],
                ref["final_labels"][b], ref["final_probs"][b], int(ref["final_valid_indices"][b])) for b in range(2)]
    else:
        boxes, labels, probs, valid = Session().run(fetches, feed_dict=model.get_feed_dict_forward(frames[0]))
        ref = relation_oracle.forward(cfg, Wt, frames[0], stages=False)
        per = [(boxes, labels, probs, ref["final_boxes"], ref["final_labels"], ref["final_probs"], len(ref["final_boxes"]))]
    for bx, lb, pr, rbx, rlb, rpr, n in per:
        assert len(bx) == n > 0
        got = np.concatenate([np.asarray(lb, np.float64)[:, None] * 10.0, bx, pr[:, None]], 1)
        exp = np.concatenate([np.asarray(rlb[:n], np.float64)[:, None] * 10.0, rbx[:n], rpr[:n, None]], 1)
        d = np.abs(got[:, None, :] - exp[None, :, :]).max(-1)
        assert d.min(1).max() < 2e-3 and d.min(0).max() < 2e-3, (d.min(1).max(), d.min(0).max())
