"""ResNet-18 / ResNet-34 detectors (`use_basic_block`) on the GPU.

Stage parity at a small geometry on the tensor-core and CUDA-core paths, full-size ResNet-34 at batch 1 and ResNet-18 at
batch 8 with batch-graph semantics against the oracle and its exact() evaluation (DESIGN 2.1), ResNet-34 with GroupNorm,
an image alone / in a batch part / in the full batch, the flags the block ignores (same outputs and the same plan), the
given-box features, get_model on a reference-style namespace, and fp16 precision."""
import types

import numpy as np
import pytest

import basic_block_oracle

pytestmark = pytest.mark.gpu

F32 = np.float32
SMALL = dict(resnet_num_block=(1, 2, 1, 1), max_size=256, short_edge_size=192, use_basic_block=True)
FEATS = ["c2", "c3", "c4", "c5", "p2", "p3", "p4", "p5", "p6"]
STAGES = FEATS + ["rpn_l%d" % i for i in range(5)]


def _cfg(**kw):
    from object_detection_tracking_b200.config import make_config
    return make_config(**kw)


def _stage_parity(cfg, H, W, seeds, tag, weight_seed=1234):
    from test_baseline_configs_gpu import run_single
    with basic_block_oracle.graph(cfg):
        return run_single(cfg, seeds, H, W, tag, weight_seed=weight_seed)


@pytest.mark.parametrize("extra", [dict(), dict(use_gn=True, use_conv_frcnn_head=True)], ids=["bn", "gn"])
def test_stage_parity_small(extra):
    """c2..c5, p2..p6, RPN logits, proposals, final detections and box features against the oracle at 192x256."""
    cfg = _cfg(**dict(SMALL, **extra))
    _stage_parity(cfg, 192, 256, (3, 4), "basic_small_" + "_".join(sorted(extra)), 99)


def _run(cfg, Wt, frames, **kw):
    from object_detection_tracking_b200.engine import Detector
    det = Detector(cfg, len(frames), frames.shape[1], frames.shape[2], **kw)
    try:
        det.load_weights(Wt)
        a = {k: v.copy() for k, v in det.detect_host(frames).items()}
        for s in STAGES:
            a[s] = det.get_stage(s)
        a["steps"] = [(p["name"], p["kind"], p["flops"], p["bytes"]) for p in det.profile_steps(reps=1)]
        a["launches"] = det.kernel_launches()
        return a
    finally:
        det.close()


def test_cuda_core_path_matches_the_oracle_and_the_tensor_cores():
    from object_detection_tracking_b200.synth import synth_frame, synth_weights
    from test_baseline_configs_gpu import rel
    cfg = _cfg(**SMALL)
    Wt = synth_weights(cfg, 99)
    frame = synth_frame(192, 256, seed=5).astype(F32)
    tc = _run(cfg, Wt, frame[None], precision="split", use_cuda_graph=False)
    simt = _run(cfg, Wt, frame[None], precision="split", use_cuda_graph=False, conv_impl="simt")
    ref = basic_block_oracle.forward(cfg, Wt, frame)
    for i in range(4):
        c = "c%d" % (i + 2)
        assert simt[c].shape[-1] == (64, 128, 256, 512)[i]
        assert rel(simt[c][0].transpose(2, 0, 1), ref["c2345"][i]) < 5e-5, c
        assert rel(simt[c], tc[c]) < 5e-5, c
    for i in range(5):
        r = ref["p23456"][i]
        g = simt["p%d" % (i + 2)][0].transpose(2, 0, 1)[:, :r.shape[1], :r.shape[2]]
        assert rel(g, r) < 1e-4 and rel(simt["p%d" % (i + 2)], tc["p%d" % (i + 2)]) < 1e-4
    n = int(tc["valid"][0])
    assert n > 0 and int(simt["valid"][0]) == n
    np.testing.assert_array_equal(np.sort(simt["labels"][0, :n]), np.sort(tc["labels"][0, :n]))


def test_r34_720x1280_batch1():
    cfg = _cfg(resnet34=True, version=4, use_frcnn_class_agnostic=True)
    assert cfg.resnet_num_block == (3, 4, 6, 3) and cfg.use_basic_block and cfg.use_dilations and cfg.num_class == 15
    recs = _stage_parity(cfg, 720, 1280, (11,), "basic_r34")
    assert recs[0]["final"] > 0


def test_r18_720x1280_batch8_multi():
    from test_baseline_configs_gpu import exact_margins, final_margins, log_margins
    from object_detection_tracking_b200.engine import Detector
    from object_detection_tracking_b200.synth import synth_frame, synth_weights
    from oracle import frcnn
    H, W, B = 720, 1280, 8
    cfg = _cfg(resnet18=True, im_batch_size=B)
    assert cfg.resnet_num_block == (2, 2, 2, 2) and cfg.use_basic_block
    Wt = synth_weights(cfg, 1234)
    frames = np.stack([synth_frame(H, W, seed=40 + s) for s in range(B)]).astype(F32)
    det = Detector(cfg, B, H, W, precision="split", use_cuda_graph=True, multi_semantics=True)
    try:
        det.load_weights(Wt)
        out = det.detect_host(frames)
    finally:
        det.close()
    ref = basic_block_oracle.forward_multi(cfg, Wt, list(frames), stages=False)
    with frcnn.exact():
        ref64 = basic_block_oracle.forward_multi(cfg, Wt, list(frames), stages=False)
    for b in range(B):
        rec = {"config": "basic-r18-multi8", "image": b}
        r, rr, r64 = int(out["valid"][b]), int(ref["final_valid_indices"][b]), int(ref64["final_valid_indices"][b])
        got = (out["labels"][b, :r], out["boxes"][b, :r], out["probs"][b, :r])
        final_margins(*got, ref["final_labels"][b, :rr], ref["final_boxes"][b, :rr], ref["final_probs"][b, :rr], rec)
        exact_margins(*got, (ref["final_labels"][b, :rr], ref["final_boxes"][b, :rr], ref["final_probs"][b, :rr]),
                      (ref64["final_labels"][b, :r64], ref64["final_boxes"][b, :r64], ref64["final_probs"][b, :r64]),
                      rec)
        log_margins(rec)
        assert rec["final"] == rec["final_ref"] and rec["labels_sorted_equal"], rec
        assert rec["gpu_to_exact"] < 1e-3, rec
        assert rec["final_set_dist"] < 1.5e-3, rec
        assert rec["final"] > 0


def test_r34_groupnorm_stage_parity():
    cfg = _cfg(resnet34=True, use_gn=True, use_conv_frcnn_head=True, max_size=256, short_edge_size=192)
    _stage_parity(cfg, 192, 256, (6,), "basic_r34_gn", 7)


def test_an_image_is_bit_identical_alone_in_a_batch_part_and_in_the_full_batch(monkeypatch):
    """Graph replay equals eager; B2_SPLIT 1 / 2 / 4 give the same bits; every image's backbone, FPN and RPN-head outputs in
    the batch of 4 equal those of the image run alone."""
    from object_detection_tracking_b200.synth import synth_frame, synth_weights
    cfg = _cfg(im_batch_size=4, **SMALL)
    Wt = synth_weights(cfg, 99)
    frames = np.stack([synth_frame(192, 256, seed=60 + s) for s in range(4)]).astype(F32)
    dual = _run(cfg, Wt, frames, use_cuda_graph=True)
    others = [_run(cfg, Wt, frames, use_cuda_graph=False)]
    for n in ("1", "4"):
        monkeypatch.setenv("B2_SPLIT", n)
        others.append(_run(cfg, Wt, frames, use_cuda_graph=True))
    monkeypatch.delenv("B2_SPLIT")
    skip = ("steps", "launches")
    for other in others:
        for k in dual:
            if k not in skip:
                np.testing.assert_array_equal(dual[k], other[k], err_msg=k)
    assert int(dual["valid"].sum()) > 0
    for k in (0, 3):
        alone = _run(cfg, Wt, frames[k:k + 1], use_cuda_graph=False)
        for s in STAGES:
            np.testing.assert_array_equal(dual[s][k:k + 1], alone[s], err_msg="image %d, %s" % (k, s))


@pytest.mark.parametrize("extra", [dict(use_se=True), dict(use_deformable=True, use_dilations=True),
                                   dict(use_dilations=True)], ids=["se", "deformable_dilations", "dilations"])
def test_ignored_flags_give_the_same_outputs_and_plan(extra):
    """The basic block has no squeeze-excite, deformable or dilated branch: the outputs are bit-identical to the flag-off
    model and the step lists equal (names, kinds, FLOPs, bytes).  In particular b2_create does not refuse use_deformable
    with use_dilations, as the reference runs that combination."""
    from object_detection_tracking_b200.synth import synth_frame, synth_weights
    frames = np.stack([synth_frame(192, 256, seed=80 + s) for s in range(2)]).astype(F32)
    base = dict(SMALL, im_batch_size=2, use_dilations=False)
    off = _cfg(**base)
    on = _cfg(**dict(base, **extra))
    Wt = synth_weights(off, 99)
    a = _run(off, Wt, frames, use_cuda_graph=True)
    b = _run(on, synth_weights(on, 99), frames, use_cuda_graph=True)
    assert a["steps"] == b["steps"] and a["launches"] == b["launches"]
    for k in a:
        if k not in ("steps", "launches"):
            np.testing.assert_array_equal(a[k], b[k], err_msg=k)


def test_given_box_features_basic():
    from object_detection_tracking_b200.backend import Session, get_model_feat
    from object_detection_tracking_b200.synth import synth_frame, synth_weights
    cfg = _cfg(**SMALL)
    Wt = synth_weights(cfg, 99)
    frame = synth_frame(192, 256, seed=8).astype(F32)
    boxes = np.array([[10, 12, 80, 90], [100, 20, 250, 180], [0, 0, 255, 191], [30.5, 40.25, 31.5, 41.0]], F32)
    model = get_model_feat(cfg)
    model.set_weights(Wt)
    got = Session().run(model.final_box_features, feed_dict=model.get_feed_dict(frame, boxes))
    ref = basic_block_oracle.forward_givenbox(cfg, Wt, frame, boxes)
    assert got.shape == ref.shape == (4, 256)
    assert np.abs(got - ref).max() / np.abs(ref).max() < 1e-4


def test_get_model_on_a_reference_namespace():
    """The drivers' argparse namespace after obj_detect_tracking.py's derivations: --resnet34 --version 4."""
    from object_detection_tracking_b200.backend import Session, get_model
    from object_detection_tracking_b200.synth import synth_frame, synth_weights
    ns = types.SimpleNamespace(resnet152=False, resnet50=False, resnet34=True, resnet18=False, version=4,
                               use_frcnn_class_agnostic=True, use_dilations=True, num_class=15, max_size=256,
                               short_edge_size=192)
    model = get_model(ns)
    cfg = model.config
    assert cfg.resnet_num_block == (3, 4, 6, 3) and cfg.use_basic_block
    Wt = synth_weights(cfg, 99)
    model.set_weights(Wt)
    frame = synth_frame(192, 256, seed=70).astype(F32)
    fetches = [model.final_boxes, model.final_labels, model.final_probs]
    boxes, labels, probs = Session().run(fetches, feed_dict=model.get_feed_dict_forward(frame))
    ref = basic_block_oracle.forward(cfg, Wt, frame, stages=False)
    n = len(ref["final_boxes"])
    assert len(boxes) == n > 0
    got = np.concatenate([np.asarray(labels, np.float64)[:, None] * 10.0, boxes, probs[:, None]], 1)
    exp = np.concatenate([np.asarray(ref["final_labels"], np.float64)[:, None] * 10.0, ref["final_boxes"],
                          ref["final_probs"][:, None]], 1)
    d = np.abs(got[:, None, :] - exp[None, :, :]).max(-1)
    assert d.min(1).max() < 2e-3 and d.min(0).max() < 2e-3, (d.min(1).max(), d.min(0).max())


CONV2_SHAPES = {   # name: (B, H, W, C) -- a basic block's conv2 (3x3, C -> C, the shortcut in the epilogue) per group
    "res2_c64": (2, 46, 80, 64),
    "res3_c128": (2, 23, 40, 128),
    "res4_c256": (1, 24, 40, 256),
    "res5_c512": (2, 12, 20, 512),
}


@pytest.mark.parametrize("name", sorted(CONV2_SHAPES))
@pytest.mark.parametrize("split,tol", [(True, 2e-5), (False, 5e-3)], ids=["split", "fp16"])
def test_conv2_shapes_staged_equals_direct(name, split, tol):
    """The staged epilogue of a 3x3 residual layer (one residual slot per warpgroup, DESIGN 4) gives the direct path's
    bits, and both are right against float64 torch."""
    import torch
    import torch.nn.functional as F
    from object_detection_tracking_b200.engine import op_conv2d_view
    B, H, W, C = CONV2_SHAPES[name]
    rng = np.random.default_rng(H * W + C)
    x = np.maximum(rng.standard_normal((B, H, W, C)), 0).astype(F32)
    w = (rng.standard_normal((3, 3, C, C)) / np.sqrt(9 * C)).astype(F32)
    bias = (rng.standard_normal(C) * 0.1).astype(F32)
    res = rng.standard_normal((B, H, W, C)).astype(F32)
    kw = dict(pad=(1, 1, 1, 1), relu=1, split=split)
    _, dh, dl, _ = op_conv2d_view(x, w, bias, res, force_epi=0, **kw)
    out, sh, sl, _ = op_conv2d_view(x, w, bias, res, force_epi=1, **kw)
    assert (dh == sh).all()
    if split:
        assert (dl == sl).all()
    d = lambda a: torch.from_numpy(np.asarray(a, np.float64))
    ref = F.conv2d(d(x).permute(0, 3, 1, 2), d(w).permute(3, 2, 0, 1), d(bias), padding=1).permute(0, 2, 3, 1)
    ref = torch.relu(ref + d(res)).numpy()
    assert np.abs(out - ref).max() <= tol * np.abs(ref).max()


def test_fp16_precision_is_close():
    from object_detection_tracking_b200.synth import synth_frame, synth_weights
    from test_baseline_configs_gpu import rel
    cfg = _cfg(**SMALL)
    Wt = synth_weights(cfg, 99)
    frame = synth_frame(192, 256, seed=9).astype(F32)
    got = _run(cfg, Wt, frame[None], precision="fp16", use_cuda_graph=True)
    ref = basic_block_oracle.forward(cfg, Wt, frame)
    for i in range(4):
        assert rel(got["c%d" % (i + 2)][0].transpose(2, 0, 1), ref["c2345"][i]) < 2e-2   # fp16 operands: ~1e-3 per layer
    assert int(got["valid"][0]) > 0
