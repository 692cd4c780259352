"""ResNeXt detector (`use_resnext`) on the GPU.

The grouped conv kernel against float64 torch and against the CUDA-core kernel, stage parity with the oracle at a small
geometry (with and without the dilated res5, and with GroupNorm), the full-size ResNeXt-101 32x4d detector against the
oracle and its exact() evaluation (DESIGN 2.1), determinism (graph replay, batch parts, an image alone), that use_se does
not change a ResNeXt model, the given-box features and get_model."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import resnext_oracle

pytestmark = pytest.mark.gpu

RX = dict(use_resnext=True)


def ref_group_conv(x, w, bias, res, stride, dil, pad, relu):
    """float64 F.conv2d(groups=C/Cg) on NHWC x with the HWIO kernel w [R, S, Cg, C] and explicit pads."""
    d = lambda a: torch.from_numpy(np.asarray(a, np.float64))
    xt = F.pad(d(x).permute(0, 3, 1, 2), (pad[2], pad[3], pad[0], pad[1]))
    groups = x.shape[3] // w.shape[2]
    y = F.conv2d(xt, d(w).permute(3, 2, 0, 1), None if bias is None else d(bias), stride=stride, dilation=dil,
                 groups=groups).permute(0, 2, 3, 1)
    if res is not None:
        y = y + d(res)
    return (torch.relu(y) if relu else y).numpy()


# name: (B, H, W, C, stride, dil, residual): C = 32 * Cg, SAME pads; M = B * Ho * Wo not a multiple of 128
KERNEL_CASES = {
    "cg4_s1_b2_res":  (2, 23, 30, 128, 1, 1, True),
    "cg8_s2_same":    (1, 46, 80, 256, 2, 1, False),     # pads 0 / 1: bottom / right
    "cg16_s1_d2":     (1, 23, 40, 512, 1, 2, True),
    "cg32_s2_d2":     (2, 12, 18, 1024, 2, 2, False),    # res5 block 0 with dilation: pads 1 / 2
    "cg32_s1_ragged": (1, 5, 7, 1024, 1, 1, True),       # M = 35 < one tile
}


def _case(name):
    B, H, W, C, stride, dil, res = KERNEL_CASES[name]
    rng = np.random.default_rng(len(name) * 7 + C)
    cg = C // 32
    x = rng.standard_normal((B, H, W, C)).astype(np.float32)
    w = (rng.standard_normal((3, 3, cg, C)) / np.sqrt(9 * cg)).astype(np.float32)
    bias = rng.standard_normal(C).astype(np.float32)
    pad = resnext_oracle.same_pads(H, 3, stride, dil) + resnext_oracle.same_pads(W, 3, stride, dil)
    Ho, Wo = -(-H // stride), -(-W // stride)
    r = rng.standard_normal((B, Ho, Wo, C)).astype(np.float32) if res else None
    return x, w, bias, r, dict(stride=stride, dil=dil, pad=pad, relu=True)


@pytest.mark.parametrize("name", sorted(KERNEL_CASES))
@pytest.mark.parametrize("split,tol", [(True, 2e-5), (False, 3e-3)])
def test_group_conv_tc_matches_torch_fp64(name, split, tol):
    from object_detection_tracking_b200.engine import op_group_conv2d
    x, w, bias, r, kw = _case(name)
    ref = ref_group_conv(x, w, bias, r, kw["stride"], kw["dil"], kw["pad"], kw["relu"])
    out = op_group_conv2d(x, w, bias, r, impl="tcgen05", split=split, **kw)
    assert out.shape == ref.shape and np.isfinite(out).all()
    assert np.abs(out - ref).max() <= tol * np.abs(ref).max()     # tolerance of test_conv_gpu: split ~fp32, fp16 ~2^-11


@pytest.mark.parametrize("name", ["cg4_s1_b2_res", "cg32_s2_d2"])
@pytest.mark.parametrize("split,tol", [(True, 1e-5), (False, 2e-3)])
def test_group_conv_tc_matches_cuda_cores(name, split, tol):
    """The tensor-core windows and the CUDA-core kernel on the dense block-diagonal expansion, same operands."""
    from object_detection_tracking_b200.engine import op_group_conv2d
    x, w, bias, r, kw = _case(name)
    tc = op_group_conv2d(x, w, bias, r, impl="tcgen05", split=split, **kw)
    simt = op_group_conv2d(x, w, bias, r, impl="simt", split=split, **kw)
    assert np.abs(tc - simt).max() <= tol * np.abs(simt).max()


def test_group_conv_refuses_what_the_windows_cannot_map():
    from object_detection_tracking_b200.engine import op_group_conv2d
    rng = np.random.default_rng(0)
    x = rng.standard_normal((1, 8, 8, 256)).astype(np.float32)
    with pytest.raises(RuntimeError, match="windows need"):      # Cg = 128 does not divide 64
        op_group_conv2d(x, rng.standard_normal((3, 3, 128, 256)).astype(np.float32), pad=(1, 1, 1, 1))
    with pytest.raises(RuntimeError, match="windows need"):      # C = 96: groups of 3 straddle the 64-channel windows
        op_group_conv2d(x[..., :96], rng.standard_normal((3, 3, 3, 96)).astype(np.float32), pad=(1, 1, 1, 1))


def _cfg(**kw):
    from object_detection_tracking_b200.config import make_config
    return make_config(**kw)


def _stage_parity(cfg, H, W, seeds, tag, weight_seed):
    """test_baseline_configs_gpu.run_single (stage-wise + final parity, DESIGN 2.1 bars) with the oracle evaluating the
    ResNeXt graph of `cfg`."""
    from test_baseline_configs_gpu import run_single
    with resnext_oracle.graph(cfg):
        return run_single(cfg, seeds, H, W, tag, weight_seed=weight_seed)


SMALL = dict(resnet_num_block=(1, 1, 2, 2), max_size=256, short_edge_size=192, **RX)


@pytest.mark.parametrize("dil", [False, True])
def test_stage_parity_small_resnext(dil):
    """c2..c5, p2..p6, RPN logits, proposals, final detections and box features against resnext_oracle at 192x256; with
    dilations, res5's stride-2 block pads 1 / 2 and writes no offset."""
    cfg = _cfg(**dict(SMALL, use_dilations=dil))
    _stage_parity(cfg, 192, 256, (3, 4), "resnext_small_dil%d" % dil, 99)


def test_stage_parity_small_gn_resnext():
    cfg = _cfg(**dict(SMALL, use_gn=True, use_conv_frcnn_head=True))
    _stage_parity(cfg, 192, 256, (5,), "gn_resnext_small", 17)


FULL = dict(resnet_num_block=(3, 4, 23, 3), **RX)      # --version 3: 15 classes, dilated res5


def test_resnext101_720x1280_batch1():
    """ResNeXt-101 32x4d, --version 3 flags, 720x1280, single-image semantics: integer outputs bit-exact, boxes by the
    rule of DESIGN 2.1."""
    cfg = _cfg(**FULL)
    assert cfg.use_dilations and cfg.num_class == 15
    recs = _stage_parity(cfg, 720, 1280, (11,), "resnext101", 1234)
    assert recs[0]["final"] > 0


def test_resnext101_720x1280_batch8_multi():
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
    ref = resnext_oracle.forward_multi(cfg, Wt, list(frames), stages=False)
    with frcnn.exact():
        ref64 = resnext_oracle.forward_multi(cfg, Wt, list(frames), stages=False)
    for b in range(B):
        rec = {"config": "resnext101-multi8", "image": b}
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


STAGES = ["c2", "c3", "c4", "c5", "p2", "p3", "p4", "p5", "p6"] + ["rpn_l%d" % i for i in range(5)]


def _outputs(cfg, Wt, frames, **kw):
    from object_detection_tracking_b200.engine import Detector
    det = Detector(cfg, len(frames), frames.shape[1], frames.shape[2], precision="split", **kw)
    try:
        det.load_weights(Wt)
        a = {k: v.copy() for k, v in det.detect_host(frames).items()}
        for s in STAGES:
            a[s] = det.get_stage(s)
        return a
    finally:
        det.close()


def test_determinism_graph_batch_parts_and_single_images(monkeypatch):
    """Graph replay equals eager, one stream equals the default two half-batch streams bit for bit, and every image's
    backbone, FPN and RPN-head outputs in the batch of 4 equal those of the image run alone."""
    from object_detection_tracking_b200.synth import synth_frame, synth_weights
    cfg = _cfg(im_batch_size=4, **dict(SMALL, use_dilations=True))
    Wt = synth_weights(cfg, 99)
    frames = np.stack([synth_frame(192, 256, seed=60 + s) for s in range(4)]).astype(np.float32)
    dual = _outputs(cfg, Wt, frames, use_cuda_graph=True)
    eager = _outputs(cfg, Wt, frames, use_cuda_graph=False)
    monkeypatch.setenv("B2_SPLIT", "1")
    single = _outputs(cfg, Wt, frames, use_cuda_graph=True)
    monkeypatch.delenv("B2_SPLIT")
    for other in (eager, single):
        for k in dual:
            np.testing.assert_array_equal(dual[k], other[k], err_msg=k)
    assert int(dual["valid"].sum()) > 0
    for k in (0, 3):
        alone = _outputs(cfg, Wt, frames[k:k + 1], use_cuda_graph=False)
        for s in STAGES:
            np.testing.assert_array_equal(dual[s][k:k + 1], alone[s], err_msg="image %d, %s" % (k, s))


def test_use_se_does_not_change_a_resnext_model():
    """The ResNeXt block has no squeeze-excite branch: use_se on or off gives the same bits."""
    from object_detection_tracking_b200.synth import synth_frame, synth_weights
    cfg = _cfg(**SMALL)
    Wt = synth_weights(cfg, 99)
    frames = synth_frame(192, 256, seed=8).astype(np.float32)[None]
    a = _outputs(cfg, Wt, frames)
    b = _outputs(_cfg(use_se=True, **SMALL), Wt, frames)
    for k in a:
        np.testing.assert_array_equal(a[k], b[k], err_msg=k)


def test_given_box_features_resnext():
    from object_detection_tracking_b200.backend import Session, get_model_feat
    from object_detection_tracking_b200.synth import synth_frame, synth_weights
    cfg = _cfg(**SMALL)
    Wt = synth_weights(cfg, 99)
    frame = synth_frame(192, 256, seed=8).astype(np.float32)
    boxes = np.array([[10, 12, 80, 90], [100, 20, 250, 180], [0, 0, 255, 191], [30.5, 40.25, 31.5, 41.0]], np.float32)
    model = get_model_feat(cfg)
    model.set_weights(Wt)
    got = Session().run(model.final_box_features, feed_dict=model.get_feed_dict(frame, boxes))
    ref = resnext_oracle.forward_givenbox(cfg, Wt, frame, boxes)
    assert got.shape == ref.shape == (4, 256)
    assert np.abs(got - ref).max() / np.abs(ref).max() < 1e-4


@pytest.mark.parametrize("is_multi", [False, True])
def test_get_model_resnext(is_multi):
    from object_detection_tracking_b200.backend import Session, get_model
    from object_detection_tracking_b200.synth import synth_frame, synth_weights
    cfg = _cfg(**SMALL)
    Wt = synth_weights(cfg, 99)
    frames = [synth_frame(192, 256, seed=70 + s).astype(np.float32) for s in range(2 if is_multi else 1)]
    model = get_model(cfg, is_multi=is_multi)
    assert type(model).__name__ == ("Mask_RCNN_FPN_multi" if is_multi else "Mask_RCNN_FPN")
    model.set_weights(Wt)
    fetches = [model.final_boxes, model.final_labels, model.final_probs, model.final_valid_indices]
    if is_multi:
        boxes, labels, probs, valid = Session().run(fetches, feed_dict=model.get_feed_dict_forward_multi(frames))
        ref = resnext_oracle.forward_multi(cfg, Wt, frames)
        per = [(boxes[b, :valid[b]], labels[b, :valid[b]], probs[b, :valid[b]], ref["final_boxes"][b],
                ref["final_labels"][b], ref["final_probs"][b], int(ref["final_valid_indices"][b])) for b in range(2)]
    else:
        boxes, labels, probs, valid = Session().run(fetches, feed_dict=model.get_feed_dict_forward(frames[0]))
        ref = resnext_oracle.forward(cfg, Wt, frames[0], stages=False)
        per = [(boxes, labels, probs, ref["final_boxes"], ref["final_labels"], ref["final_probs"], len(ref["final_boxes"]))]
    for bx, lb, pr, rbx, rlb, rpr, n in per:
        assert len(bx) == n > 0
        got = np.concatenate([np.asarray(lb, np.float64)[:, None] * 10.0, bx, pr[:, None]], 1)
        exp = np.concatenate([np.asarray(rlb[:n], np.float64)[:, None] * 10.0, rbx[:n], rpr[:n, None]], 1)
        d = np.abs(got[:, None, :] - exp[None, :, :]).max(-1)
        assert d.min(1).max() < 2e-3 and d.min(0).max() < 2e-3, (d.min(1).max(), d.min(0).max())
