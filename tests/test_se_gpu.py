"""SE-ResNet detector (`use_se`, `--version 6`) on the GPU.

The squeeze-excite kernels against float64 torch, stage parity with the oracle at a small geometry (with and without the
dilated res5, and with GroupNorm), the full-size v6 detector against the oracle and its exact() evaluation (DESIGN 2.1),
that the SE path changes the detections, determinism (two passes, graph replay, batch parts, an image alone) and the
given-box features."""
import numpy as np
import pytest
import torch

import se_oracle

pytestmark = pytest.mark.gpu

V6 = dict(use_se=True, use_frcnn_class_agnostic=True, use_dilations=False, version=6)


def ref_se(x, w1, b1, w2, b2, res=None):
    """float64 nn.py:506-521 on NHWC x [B,H,W,C]: relu(x * sigmoid(relu(mean_hw(x) @ w1 + b1) @ w2 + b2) + res)."""
    t = torch.from_numpy(x.astype(np.float64))
    d = lambda a: torch.from_numpy(np.asarray(a, np.float64))
    s = torch.relu(t.mean(dim=(1, 2)) @ d(w1) + d(b1))
    g = torch.sigmoid(s @ d(w2) + d(b2))
    y = t * g[:, None, None, :]
    if res is not None:
        y = y + d(res)
    return torch.relu(y).numpy(), g.numpy()


def quantize(a, split):
    """What the engine's planes hold: ~fp32 in split precision, fp16 otherwise."""
    return a.astype(np.float32) if split else a.astype(np.float16).astype(np.float32)


# (B, H, W, C, residual, split): fc1 width C / 16 (16 for C = 256, 128 for C = 2048)
KERNEL_CASES = [
    (3, 184, 320, 256, True, True),
    (3, 184, 320, 256, False, False),
    (3, 23, 40, 2048, True, False),
    (3, 23, 40, 2048, False, True),
    (3, 46, 80, 1024, True, True),
]


@pytest.mark.parametrize("B,H,W,C,res,split", KERNEL_CASES)
def test_squeeze_excite_kernel_vs_fp64(B, H, W, C, res, split):
    from object_detection_tracking_b200.engine import op_squeeze_excite
    rng = np.random.default_rng(B * 1000 + C + H)
    nr = C // 16
    # per-image, per-channel offsets: a squeeze or a gate that mixes images would be visibly wrong
    x = rng.standard_normal((B, H, W, C)) * rng.uniform(0.5, 2, (B, 1, 1, C)) + rng.uniform(-0.5, 0.5, (B, 1, 1, C))
    x = quantize(x, split)
    w1 = (rng.standard_normal((C, nr)) * np.sqrt(8.0 / C)).astype(np.float32)
    b1 = rng.uniform(0.0, 0.1, nr).astype(np.float32)
    w2 = (rng.standard_normal((nr, C)) * np.sqrt(2.0 / nr)).astype(np.float32)
    b2 = (rng.standard_normal(C) * 0.4).astype(np.float32)
    r = quantize(rng.standard_normal((B, H, W, C)), split) if res else None
    got, gate = op_squeeze_excite(x, w1, b1, w2, b2, res=r, split=split)
    ref, gref = ref_se(x, w1, b1, w2, b2, r)
    assert np.abs(gate - gref).max() < 2e-6, np.abs(gate - gref).max()
    assert 0.02 < gref.min() and gref.max() < 0.98 and np.abs(gref[0] - gref[1]).max() > 0.05   # not saturated, per image
    err = np.abs(got - ref).max() / (np.abs(ref).max() + 1e-12)
    assert err < (2e-6 if split else 1.5e-3), err
    # an image's result does not depend on the batch it is in
    one, g1 = op_squeeze_excite(x[1:2], w1, b1, w2, b2, res=None if r is None else r[1:2], split=split)
    np.testing.assert_array_equal(one, got[1:2])
    np.testing.assert_array_equal(g1, gate[1:2])


def _cfg(**kw):
    from object_detection_tracking_b200.config import make_config
    return make_config(**kw)


def _stage_parity(cfg, H, W, seeds, tag, weight_seed):
    """test_baseline_configs_gpu.run_single (stage-wise + final parity, DESIGN 2.1 bars) with the oracle evaluating the
    squeeze-excite graph of `cfg`."""
    from test_baseline_configs_gpu import run_single
    with se_oracle.graph(cfg):
        return run_single(cfg, seeds, H, W, tag, weight_seed=weight_seed)


SMALL = dict(resnet_num_block=(1, 1, 2, 2), max_size=256, short_edge_size=192)


@pytest.mark.parametrize("dil", [False, True])
def test_stage_parity_small_se(dil):
    """c2..c5, p2..p6, RPN logits, proposals, final detections and box features against se_oracle at 192x256; with
    dilations, res5's stride-2 block writes an offset view that conv3 reads before the gate."""
    cfg = _cfg(**dict(SMALL, **dict(V6, use_dilations=dil)))
    _stage_parity(cfg, 192, 256, (3, 4), "se_small_dil%d" % dil, 99)


def test_stage_parity_small_gn_se():
    """use_gn + use_se: conv3's GroupNorm step carries no residual and no ReLU; the SE apply adds both."""
    cfg = _cfg(**dict(SMALL, **V6, use_gn=True, use_conv_frcnn_head=True))
    _stage_parity(cfg, 192, 256, (5,), "gn_se_small", 17)


FULL = dict(resnet_num_block=(3, 4, 23, 3), num_class=15, **V6)


def test_v6_r101_720x1280_batch1():
    """The "Object v6" model of the reference README (README.md:350-352): R101, squeeze-excite, class-agnostic, no dilation, 15 classes, 720x1280,
    single-image semantics: integer outputs bit-exact, boxes by the rule of DESIGN 2.1."""
    recs = _stage_parity(_cfg(**FULL), 720, 1280, (11,), "v6-R101", 1234)
    assert recs[0]["final"] > 0


def test_v6_r101_720x1280_batch8_multi():
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
    ref = se_oracle.forward_multi(cfg, Wt, list(frames), stages=False)
    with frcnn.exact():
        ref64 = se_oracle.forward_multi(cfg, Wt, list(frames), stages=False)
    for b in range(B):
        rec = {"config": "v6-R101-multi8", "image": b}
        r, rr, r64 = int(out["valid"][b]), int(ref["final_valid_indices"][b]), int(ref64["final_valid_indices"][b])
        got = (out["labels"][b, :r], out["boxes"][b, :r], out["probs"][b, :r])
        final_margins(*got, ref["final_labels"][b, :rr], ref["final_boxes"][b, :rr], ref["final_probs"][b, :rr], rec)
        exact_margins(*got, (ref["final_labels"][b, :rr], ref["final_boxes"][b, :rr], ref["final_probs"][b, :rr]),
                      (ref64["final_labels"][b, :r64], ref64["final_boxes"][b, :r64], ref64["final_probs"][b, :r64]),
                      rec)
        log_margins(rec)
        # DESIGN 2.1: counts and class ids bit-exact, boxes within 1e-3 px of the exact evaluation and within 1.5e-3 px
        # of the float32 port
        assert rec["final"] == rec["final_ref"] and rec["labels_sorted_equal"], rec
        assert rec["gpu_to_exact"] < 1e-3, rec
        assert rec["final_set_dist"] < 1.5e-3, rec
        assert rec["final"] > 0


def test_v6_detections_depend_on_the_se_path():
    """The same weights with use_se off (the SE arrays then ignored) give other detections: the gate is exercised."""
    from object_detection_tracking_b200.engine import Detector
    from object_detection_tracking_b200.synth import synth_frame, synth_weights
    cfg = _cfg(**FULL)
    Wt = synth_weights(cfg, 1234)
    frame = synth_frame(720, 1280, seed=11).astype(np.float32)[None]
    outs = []
    for use_se in (True, False):
        det = Detector(_cfg(**dict(FULL, use_se=use_se)), 1, 720, 1280, precision="split")
        try:
            det.load_weights(Wt)
            outs.append({k: v.copy() for k, v in det.detect_host(frame, want_feat=False).items()})
            outs[-1]["c5"] = det.get_stage("c5")
        finally:
            det.close()
    a, b = outs
    assert np.abs(a["c5"] - b["c5"]).max() > 1e-2
    n = min(int(a["valid"][0]), int(b["valid"][0]))
    assert int(a["valid"][0]) != int(b["valid"][0]) or np.abs(a["boxes"][0, :n] - b["boxes"][0, :n]).max() > 1e-2


STAGES = ["c2", "c3", "c4", "c5", "p2", "p3", "p4", "p5", "p6"] + ["rpn_l%d" % i for i in range(5)]


def _outputs(cfg, Wt, frames, **kw):
    from object_detection_tracking_b200.engine import Detector
    det = Detector(cfg, len(frames), frames.shape[1], frames.shape[2], precision="split", **kw)
    try:
        det.load_weights(Wt)
        a = det.detect_host(frames)
        a = {k: v.copy() for k, v in a.items()}
        b = det.detect_host(frames)
        for k in a:
            np.testing.assert_array_equal(a[k], b[k], err_msg="second pass differs: " + k)
        for s in STAGES:
            a[s] = det.get_stage(s)
        return a
    finally:
        det.close()


def test_determinism_graph_batch_parts_and_single_images(monkeypatch):
    """Two passes are bit-identical, graph replay equals eager, B2_SPLIT=1 / 2 (default) / 4 agree bit for bit, and every
    image's backbone, FPN and RPN-head outputs in the batch of 8 equal those of the image run alone (the squeeze, the gate
    and their scratch are per image)."""
    from object_detection_tracking_b200.synth import synth_frame, synth_weights
    cfg = _cfg(im_batch_size=8, **dict(SMALL, **V6))
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
        for s in STAGES:
            np.testing.assert_array_equal(dual[s][k:k + 1], alone[s], err_msg="image %d, %s" % (k, s))


def test_given_box_features_se():
    from object_detection_tracking_b200.backend import Session, get_model_feat
    from object_detection_tracking_b200.synth import synth_frame, synth_weights
    cfg = _cfg(**dict(SMALL, **V6))
    Wt = synth_weights(cfg, 99)
    frame = synth_frame(192, 256, seed=8).astype(np.float32)
    boxes = np.array([[10, 12, 80, 90], [100, 20, 250, 180], [0, 0, 255, 191], [30.5, 40.25, 31.5, 41.0]], np.float32)
    model = get_model_feat(cfg)
    model.set_weights(Wt)
    got = Session().run(model.final_box_features, feed_dict=model.get_feed_dict(frame, boxes))
    ref = se_oracle.forward_givenbox(cfg, Wt, frame, boxes)
    assert got.shape == ref.shape == (4, 256)
    assert np.abs(got - ref).max() / np.abs(ref).max() < 1e-4


@pytest.mark.parametrize("is_multi", [False, True])
def test_get_model_v6(is_multi):
    """get_model(config) with use_se: the single-image graph (Mask_RCNN_FPN) and the batch graph (Mask_RCNN_FPN_multi) run
    the SE backbone and match se_oracle's detections."""
    from object_detection_tracking_b200.backend import Session, get_model
    from object_detection_tracking_b200.synth import synth_frame, synth_weights
    cfg = _cfg(**dict(SMALL, **V6))
    Wt = synth_weights(cfg, 99)
    frames = [synth_frame(192, 256, seed=70 + s).astype(np.float32) for s in range(2 if is_multi else 1)]
    model = get_model(cfg, is_multi=is_multi)
    assert type(model).__name__ == ("Mask_RCNN_FPN_multi" if is_multi else "Mask_RCNN_FPN")
    model.set_weights(Wt)
    fetches = [model.final_boxes, model.final_labels, model.final_probs, model.final_valid_indices]
    if is_multi:
        boxes, labels, probs, valid = Session().run(fetches, feed_dict=model.get_feed_dict_forward_multi(frames))
        ref = se_oracle.forward_multi(cfg, Wt, frames)
        per = [(boxes[b, :valid[b]], labels[b, :valid[b]], probs[b, :valid[b]], ref["final_boxes"][b],
                ref["final_labels"][b], ref["final_probs"][b], int(ref["final_valid_indices"][b])) for b in range(2)]
    else:
        boxes, labels, probs, valid = Session().run(fetches, feed_dict=model.get_feed_dict_forward(frames[0]))
        ref = se_oracle.forward(cfg, Wt, frames[0], stages=False)
        per = [(boxes, labels, probs, ref["final_boxes"], ref["final_labels"], ref["final_probs"], len(ref["final_boxes"]))]
    for bx, lb, pr, rbx, rlb, rpr, n in per:
        assert len(bx) == n > 0
        got = np.concatenate([np.asarray(lb, np.float64)[:, None] * 10.0, bx, pr[:, None]], 1)
        exp = np.concatenate([np.asarray(rlb[:n], np.float64)[:, None] * 10.0, rbx[:n], rpr[:n, None]], 1)
        d = np.abs(got[:, None, :] - exp[None, :, :]).max(-1)
        assert d.min(1).max() < 2e-3 and d.min(0).max() < 2e-3, (d.min(1).max(), d.min(0).max())
