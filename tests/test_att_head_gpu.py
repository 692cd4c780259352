"""Attention box head (`use_att_frcnn_head`) on the GPU.

The pool kernel against float64 (split and fp16 planes, non-finite ROIs, an ROI alone and in a batch), stage parity with
att_oracle at a small geometry (2fc, GroupNorm + conv head, relation, COCO-81 partial classes, mask), the cases where the
flag must not change anything (class-agnostic heads, the attention conv's own weights), the load-time refusals, the
full-size R101 detector against the oracle and its exact() evaluation (DESIGN 2.1), determinism (two passes, graph
replay, batch parts, an image alone) and get_model."""
import contextlib

import numpy as np
import pytest

import att_oracle

pytestmark = pytest.mark.gpu

ATT = dict(use_att_frcnn_head=True)
SMALL = dict(resnet_num_block=(1, 1, 2, 2), max_size=256, short_edge_size=192)
NAMES = ("fastrcnn/attention/W", "fastrcnn/attention/b", "fastrcnn/att_trans/W", "fastrcnn/att_trans/b")


def _cfg(**kw):
    from object_detection_tracking_b200.config import make_config
    return make_config(**kw)


def _pool_bound(x, ref, split):
    """|got - ref| bound of the pool: 49 fp32 additions (each within 2^-24 of the running sum, which is below sum|x|), the
    split planes' input error (2^-23 |x|), and the output planes' rounding (2^-21 |s| split, 2^-11 |s| fp16)."""
    ax = np.abs(x.astype(np.float64)).sum(axis=1)
    return ax * (49 * 2.0 ** -24 + (2.0 ** -23 if split else 0.0)) + np.abs(ref) * (2.0 ** -21 if split else 2.0 ** -11)


def _pool_input(rng, M, split, C=256):
    x = rng.standard_normal((M, 49, C)) * rng.uniform(0.01, 300.0, (M, 1, 1)) + rng.uniform(-1, 3, (M, 1, C))
    x[: M // 3] = np.maximum(x[: M // 3], 0)                                   # post-ReLU-like rows
    if M > 1:
        x[-1, :, :8] = 60000.0 * (1 - 2 * (np.arange(49) % 2))[:, None]       # +-60000 by bin: near the fp16 limit, the
                                                                              # sum 60000 after 48 cancellations
    x = x.astype(np.float32)
    return x if split else x.astype(np.float16).astype(np.float32)


@pytest.mark.parametrize("split", [True, False])
@pytest.mark.parametrize("M", [1, 7, 300, 2400])
def test_att_pool_vs_fp64(M, split):
    from object_detection_tracking_b200.engine import op_att_pool
    rng = np.random.default_rng(M * 2 + split)
    x = _pool_input(rng, M, split)
    got = op_att_pool(x, split=split)
    ref = x.astype(np.float64).sum(axis=1)
    assert np.isfinite(got).all()
    err = np.abs(got - ref)
    assert (err <= _pool_bound(x, ref, split)).all(), float((err / np.maximum(_pool_bound(x, ref, split), 1e-30)).max())
    # an ROI alone is bit-identical to the same ROI in the batch
    k = M // 2
    np.testing.assert_array_equal(op_att_pool(x[k:k + 1], split=split), got[k:k + 1])


@pytest.mark.parametrize("split", [True, False])
@pytest.mark.parametrize("bad", [np.inf, -np.inf, np.nan])
def test_att_pool_non_finite_roi_is_nan_alone(bad, split):
    from object_detection_tracking_b200.engine import op_att_pool
    rng = np.random.default_rng(11)
    x = _pool_input(rng, 300, split)
    clean = op_att_pool(x, split=split)
    x[123, 48, 255] = bad
    x[200, 0, 0] = bad
    got = op_att_pool(x, split=split)
    assert np.isnan(got[[123, 200]]).all()
    keep = np.setdiff1d(np.arange(300), [123, 200])
    np.testing.assert_array_equal(got[keep], clean[keep])


def _run_small(cfg, seed, weight_seed=99, H=192, W=256, Wt=None):
    """Batch-1 context at the small geometry: the detections and the branch's rows of the proposals."""
    from object_detection_tracking_b200.engine import Detector
    from object_detection_tracking_b200.synth import synth_frame, synth_weights
    Wt = synth_weights(cfg, weight_seed) if Wt is None else Wt
    frame = synth_frame(H, W, seed=seed).astype(np.float32)
    det = Detector(cfg, 1, H, W, precision="split")
    try:
        det.load_weights(Wt)
        out = {k: v.copy() for k, v in det.detect_host(frame[None], want_feat=False).items()}
        pc = int(det.get_stage("proposal_count").reshape(-1)[0])
        st = {}
        if att_oracle.use_att(cfg):
            st["roi_feat"] = det.get_stage("roi_feat").reshape(-1, 49, 256)[:pc]
            st["att_pool"] = det.get_stage("att_pool").reshape(-1, 256)[:pc]
            for s in ("att_trans", "att_sum"):
                st[s] = det.get_stage(s).reshape(-1, cfg.fpn_frcnn_fc_head_dim)[:pc]
        out["head_logits"] = det.get_stage("head_logits").copy()
    finally:
        det.close()
    return out, st, frame, Wt


def _stage_parity(cfg, seeds, tag, weight_seed=99, H=192, W=256):
    import partial_oracle
    from test_baseline_configs_gpu import run_single
    ids = tuple(getattr(cfg, "partial_class_ids", ()))
    with att_oracle.graph(cfg), partial_oracle.partial_classes(ids) if ids else contextlib.nullcontext():
        return run_single(cfg, seeds, H, W, tag, weight_seed=weight_seed)


PARITY = {
    "2fc": (dict(), 99),
    "gn_conv_head": (dict(use_gn=True, use_conv_frcnn_head=True), 17),
    "relation": (dict(add_relation_nn=True), 99),
    "coco81_partial": (dict(num_class=81, use_partial_classes=True), 77),
    "mask": (dict(add_mask=True), 99),
}


@pytest.mark.parametrize("name", sorted(PARITY))
def test_stage_parity_small(name):
    """Backbone to detections against att_oracle at 192x256 (DESIGN 2.1 bars); att_pool row by row against the engine's
    own ROIAlign rows in float64, att_trans / att_sum against the oracle's rows."""
    import partial_oracle
    from oracle import frcnn
    kw, ws = PARITY[name]
    cfg = _cfg(**dict(SMALL, **dict(kw, **ATT)))
    recs = _stage_parity(cfg, (3, 4), "att_small_" + name, weight_seed=ws)
    assert recs[0]["final"] > 0
    _, st, frame, Wt = _run_small(cfg, 3, weight_seed=ws)
    roi = st["roi_feat"].astype(np.float64)
    ref = roi.sum(axis=1)
    err = np.abs(st["att_pool"] - ref)
    assert (err <= _pool_bound(st["roi_feat"], ref, True)).all()
    ids = tuple(getattr(cfg, "partial_class_ids", ()))
    with att_oracle.graph(cfg), partial_oracle.partial_classes(ids) if ids else contextlib.nullcontext():
        frcnn.forward(cfg, Wt, frame, stages=False)
    last = dict(att_oracle.LAST)
    for s in ("att_pool", "att_trans", "att_sum"):
        assert st[s].shape == last[s].shape, (s, st[s].shape, last[s].shape)
        e = np.abs(st[s] - last[s]).max() / np.abs(last[s]).max()
        assert e < 1e-4, (s, e)


def _same_detections(a, b):
    for k in ("boxes", "probs", "labels", "valid", "head_logits"):
        np.testing.assert_array_equal(a[k], b[k], err_msg=k)


def test_class_agnostic_ignores_the_flag():
    for kw in (dict(), dict(add_relation_nn=True)):
        base = dict(SMALL, use_frcnn_class_agnostic=True, **kw)
        a, _, _, _ = _run_small(_cfg(**base), 6)
        b, _, _, _ = _run_small(_cfg(**dict(base, **ATT)), 6)
        _same_detections(a, b)


def test_attention_conv_weights_do_not_change_the_detections():
    """Fact 1 on the device: two different fastrcnn/attention/{W,b} that pass the load check give the same detections,
    bit for bit; the same weights with the flag off give other detections."""
    from object_detection_tracking_b200.synth import synth_weights
    cfg = _cfg(**dict(SMALL, **ATT))
    Wt = synth_weights(cfg, 99)
    rng = np.random.default_rng(1)
    W2 = dict(Wt)
    W2["fastrcnn/attention/W"] = (rng.standard_normal(Wt["fastrcnn/attention/W"].shape) * 3.0).astype(np.float32)
    W2["fastrcnn/attention/b"] = np.array([-1e6], np.float32)
    a, _, _, _ = _run_small(cfg, 7, Wt=Wt)
    b, _, _, _ = _run_small(cfg, 7, Wt=W2)
    _same_detections(a, b)
    c, _, _, _ = _run_small(_cfg(**SMALL), 7, Wt=Wt)
    n = min(int(a["valid"][0]), int(c["valid"][0]))
    assert int(a["valid"][0]) != int(c["valid"][0]) or np.abs(a["probs"][0, :n] - c["probs"][0, :n]).max() > 1e-3


@pytest.mark.parametrize("name,value", [("fastrcnn/attention/W", np.nan), ("fastrcnn/attention/W", np.inf),
                                        ("fastrcnn/attention/b", -np.inf), ("fastrcnn/attention/W", 1e32)])
def test_load_refuses_attention_weights_that_could_make_a_logit_non_finite(name, value):
    """Non-finite attention weights, or weights with 65536 * sum|W| + |b| >= FLT_MAX (1e32 in every tap: 65536 * 2304 *
    1e32 > 3.4e38), are refused by name."""
    from object_detection_tracking_b200.engine import Detector
    from object_detection_tracking_b200.synth import synth_weights
    cfg = _cfg(**dict(SMALL, **ATT))
    Wt = synth_weights(cfg, 99)
    if value == 1e32:
        Wt[name] = np.full_like(Wt[name], value)
    else:
        Wt[name] = Wt[name].copy()
        Wt[name].reshape(-1)[-1] = value
    det = Detector(cfg, 1, 192, 256, precision="split")
    try:
        with pytest.raises(RuntimeError) as e:
            det.load_weights(Wt)
        assert name in str(e.value)
    finally:
        det.close()


FULL = dict(resnet_num_block=(3, 4, 23, 3), num_class=15, use_frcnn_class_agnostic=False, use_dilations=True, **ATT)


def test_att_r101_720x1280_batch1():
    """R101 dilated (--version 3), 15 classes, class-specific + attention head, 720x1280, single-image semantics: counts and
    labels exact, boxes by the rule of DESIGN 2.1."""
    recs = _stage_parity(_cfg(**FULL), (11,), "att-R101", weight_seed=1234, H=720, W=1280)
    assert recs[0]["final"] > 0


def test_att_r101_720x1280_batch8_multi():
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
    ref = att_oracle.forward_multi(cfg, Wt, list(frames), stages=False)
    with frcnn.exact():
        ref64 = att_oracle.forward_multi(cfg, Wt, list(frames), stages=False)
    for b in range(B):
        rec = {"config": "att-R101-multi8", "image": b}
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


HEAD = ["att_pool", "att_sum", "head_logits", "proposal_boxes", "proposal_count"]


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
            a[s] = v.reshape(len(frames), K, -1) if s.startswith("att") else v
        return a
    finally:
        det.close()


def test_determinism_graph_batch_parts_and_single_images(monkeypatch):
    """Two passes are bit-identical, graph replay equals eager, B2_SPLIT=1 / 2 / 4 agree bit for bit, and every image of
    the batch of 8 gets the branch rows, head logits and detections it gets alone."""
    from object_detection_tracking_b200.synth import synth_frame, synth_weights
    cfg = _cfg(im_batch_size=8, **dict(SMALL, **ATT))
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
    for k in range(8):
        alone = _outputs(cfg, Wt, frames[k:k + 1], use_cuda_graph=False)
        for s in ("att_pool", "att_sum"):
            np.testing.assert_array_equal(dual[s][k:k + 1], alone[s], err_msg="image %d, %s" % (k, s))
        np.testing.assert_array_equal(dual["head_logits"][k:k + 1], alone["head_logits"], err_msg="image %d" % k)
        for o in ("boxes", "probs", "labels", "valid"):
            np.testing.assert_array_equal(dual[o][k:k + 1], alone[o], err_msg="image %d, %s" % (k, o))


@pytest.mark.parametrize("is_multi", [False, True])
def test_get_model_att(is_multi):
    from object_detection_tracking_b200.backend import Session, get_model
    from object_detection_tracking_b200.synth import synth_frame, synth_weights
    cfg = _cfg(**dict(SMALL, **ATT))
    Wt = synth_weights(cfg, 99)
    frames = [synth_frame(192, 256, seed=70 + s).astype(np.float32) for s in range(2 if is_multi else 1)]
    model = get_model(cfg, is_multi=is_multi)
    model.set_weights(Wt)
    fetches = [model.final_boxes, model.final_labels, model.final_probs, model.final_valid_indices]
    if is_multi:
        boxes, labels, probs, valid = Session().run(fetches, feed_dict=model.get_feed_dict_forward_multi(frames))
        ref = att_oracle.forward_multi(cfg, Wt, frames)
        per = [(boxes[b, :valid[b]], labels[b, :valid[b]], probs[b, :valid[b]], ref["final_boxes"][b],
                ref["final_labels"][b], ref["final_probs"][b], int(ref["final_valid_indices"][b])) for b in range(2)]
    else:
        boxes, labels, probs, valid = Session().run(fetches, feed_dict=model.get_feed_dict_forward(frames[0]))
        ref = att_oracle.forward(cfg, Wt, frames[0], stages=False)
        per = [(boxes, labels, probs, ref["final_boxes"], ref["final_labels"], ref["final_probs"], len(ref["final_boxes"]))]
    for bx, lb, pr, rbx, rlb, rpr, n in per:
        assert len(bx) == n > 0
        got = np.concatenate([np.asarray(lb, np.float64)[:, None] * 10.0, bx, pr[:, None]], 1)
        exp = np.concatenate([np.asarray(rlb[:n], np.float64)[:, None] * 10.0, rbx[:n], rpr[:n, None]], 1)
        d = np.abs(got[:, None, :] - exp[None, :, :]).max(-1)
        assert d.min(1).max() < 2e-3 and d.min(0).max() < 2e-3, (d.min(1).max(), d.min(0).max())
