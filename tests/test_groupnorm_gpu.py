"""GroupNorm detectors on the GPU (use_gn backbone + FPN, use_conv_frcnn_head box head).

Kernel cases of csrc/groupnorm.cu against float64 torch, stage parity with the oracle at a small geometry (with and
without the dilated res5, whose stride-2 block normalises an offset view), the full-size R50-GN conv-head detector against
the oracle and its exact() evaluation (DESIGN 2.1), the other flag combinations, determinism (two passes, graph replay,
half-batch streams) and the given-box features."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import gn_oracle

pytestmark = pytest.mark.gpu


def ref_gn(x, gamma, beta, res=None, res_shift=0, relu=False):
    """float64 GroupNorm of NHWC x [B,H,W,C] (+ residual at (y >> s, x >> s)) (ReLU)."""
    t = torch.from_numpy(x.astype(np.float64)).permute(0, 3, 1, 2)
    y = F.group_norm(t, 32, torch.from_numpy(gamma.astype(np.float64)), torch.from_numpy(beta.astype(np.float64)), eps=1e-5)
    y = y.permute(0, 2, 3, 1).numpy()
    if res is not None:
        r = res.astype(np.float64)
        if res_shift:
            r = r.repeat(2, axis=1).repeat(2, axis=2)
        y = y + r[:, :y.shape[1], :y.shape[2]]
    return np.maximum(y, 0.0) if relu else y


def quantize(a, split):
    """What the engine's planes hold: ~fp32 in split precision, fp16 otherwise."""
    return a.astype(np.float32) if split else a.astype(np.float16).astype(np.float32)


# (B, H, W, C, residual: None / "same" / "up", relu, split, per_roi)
KERNEL_CASES = [
    (3, 184, 320, 64, None, True, True, False),       # group size 2, per-image statistics over 3 images
    (1, 184, 320, 256, "same", True, True, False),
    (3, 23, 40, 2048, "same", True, False, False),    # group size 64, c5, fp16
    (2, 46, 80, 256, "up", False, True, False),       # FPN top-down sum
    (3, 23, 40, 2048, None, False, True, False),
    (5, 7, 7, 256, None, False, True, True),          # per-ROI head GN
    (4, 7, 7, 64, None, False, False, True),
    (3, 7, 7, 1024, None, True, True, True),
]


@pytest.mark.parametrize("B,H,W,C,res,relu,split,per_roi", KERNEL_CASES)
def test_group_norm_kernel_vs_fp64(B, H, W, C, res, relu, split, per_roi):
    from object_detection_tracking_b200.engine import op_group_norm
    rng = np.random.default_rng(B * 1000 + C + H)
    # per-image, per-channel offsets: statistics that mix images or groups would be visibly wrong
    x = (rng.standard_normal((B, H, W, C)) * rng.uniform(0.5, 3, (B, 1, 1, C)) + rng.uniform(-2, 2, (B, 1, 1, C)))
    x = quantize(x, split)
    gamma = rng.uniform(0.5, 1.5, C).astype(np.float32)
    beta = (rng.standard_normal(C) * 0.2).astype(np.float32)
    r, shift = None, 0
    if res == "same":
        r = quantize(rng.standard_normal((B, H, W, C)), split)
    elif res == "up":
        r, shift = quantize(rng.standard_normal((B, (H + 1) // 2, (W + 1) // 2, C)), split), 1
    got = op_group_norm(x, gamma, beta, res=r, res_shift=shift, relu=relu, per_roi=per_roi, split=split)
    ref = ref_gn(x, gamma, beta, r, shift, relu)
    err = np.abs(got - ref).max() / (np.abs(ref).max() + 1e-12)
    assert err < (2e-6 if split else 1.5e-3), err


@pytest.mark.parametrize("split", [True, False])
@pytest.mark.parametrize("in_place", [True, False])
def test_group_norm_offset_view_keeps_border(split, in_place):
    """The dilated stride-2 block: the conv output sits at (1, 1) of a buffer whose first row / column are the [1, 0] pad
    (nn.py:490-497).  Statistics cover the view only and the border stays exactly 0."""
    from object_detection_tracking_b200.engine import op_group_norm
    rng = np.random.default_rng(7)
    B, H, W, C = 2, 23, 40, 512
    buf = np.zeros((B, H + 1, W + 1, C), np.float32)
    buf[:, 1:, 1:] = quantize(rng.standard_normal((B, H, W, C)) * 3 + 1, split)
    gamma = rng.uniform(0.5, 1.5, C).astype(np.float32)
    beta = (rng.standard_normal(C) * 0.2).astype(np.float32)
    got = op_group_norm(buf, gamma, beta, view=(1, 1, H, W), relu=True, split=split, in_place=in_place)
    assert not got[:, 0].any() and not got[:, :, 0].any()
    ref = ref_gn(buf[:, 1:, 1:], gamma, beta, relu=True)
    err = np.abs(got[:, 1:, 1:] - ref).max() / np.abs(ref).max()
    assert err < (2e-6 if split else 1.5e-3), err


def _cfg(**kw):
    from object_detection_tracking_b200.config import make_config
    return make_config(**kw)


SMALL = dict(resnet_num_block=(1, 1, 2, 2), max_size=256, short_edge_size=192, num_class=81, use_gn=True,
             use_conv_frcnn_head=True)


def _stage_parity(cfg, H, W, seeds, tag, weight_seed):
    """test_baseline_configs_gpu.run_single (stage-wise + final parity, DESIGN 2.1 bars) with the oracle evaluating the
    GroupNorm / conv-head graph of `cfg`."""
    from test_baseline_configs_gpu import run_single
    with gn_oracle.graph(cfg):
        return run_single(cfg, seeds, H, W, tag, weight_seed=weight_seed)


@pytest.mark.parametrize("dil", [True, False])
def test_stage_parity_small_gn_conv_head(dil):
    """c2..c5, p2..p6, RPN logits, proposals, final detections and box features against the oracle (gn_oracle.forward) at 192x256
    with (1,1,2,2) blocks; with dilations, res5's stride-2 block is dilated and normalises an offset view.  The head
    logits are compared where the proposals agree."""
    from object_detection_tracking_b200.engine import Detector
    from object_detection_tracking_b200.synth import synth_frame, synth_weights
    cfg = _cfg(use_dilations=dil, version=3 if dil else 2, **SMALL)
    _stage_parity(cfg, 192, 256, (3, 4), "gn_small_dil%d" % dil, 99)
    Wt = synth_weights(cfg, 99)
    frame = synth_frame(192, 256, seed=3).astype(np.float32)
    det = Detector(cfg, 1, 192, 256, precision="split", use_cuda_graph=False)
    try:
        det.load_weights(Wt)
        det.set_stage("image", frame[None])
        det.run_phases(255)
        o = gn_oracle.forward(cfg, Wt, frame)
        pc = int(det.get_stage("proposal_count")[0].reshape(-1)[0])
        assert pc == len(o["proposal_boxes"])
        K = cfg.rpn_test_post_nms_topk
        pb = det.get_stage("proposal_boxes")[0].reshape(K, 4)[:pc]
        assert np.abs(pb - o["proposal_boxes"]).max() < 1.5e-3            # same order: head rows correspond
        logits = det.get_stage("head_logits")[0].reshape(K, -1)[:pc, :cfg.num_class]
        rel = np.abs(logits - o["cls_logits"]).max() / np.abs(o["cls_logits"]).max()
        assert rel < 2e-4, rel
    finally:
        det.close()


def test_r50_gn_conv_head_720x1280_batch1():
    """R50-GN-FPN with the GN conv head, COCO 81 classes (version 2: no dilation), 720x1280, batch 1, single-image
    semantics: integer outputs bit-exact, boxes by the rule of DESIGN 2.1."""
    cfg = _cfg(resnet_num_block=(3, 4, 6, 3), num_class=81, use_dilations=False, version=2, use_gn=True,
               use_conv_frcnn_head=True)
    recs = _stage_parity(cfg, 720, 1280, (11,), "R50-GN", 4321)
    assert recs[0]["final"] > 0


def test_r50_gn_conv_head_720x1280_batch2_multi():
    from test_baseline_configs_gpu import exact_margins, final_margins, log_margins, set_dist
    from object_detection_tracking_b200.engine import Detector
    from object_detection_tracking_b200.synth import synth_frame, synth_weights
    from oracle import frcnn
    H, W, B = 720, 1280, 2
    cfg = _cfg(resnet_num_block=(3, 4, 6, 3), num_class=81, use_dilations=False, version=2, use_gn=True,
               use_conv_frcnn_head=True, im_batch_size=B)
    Wt = synth_weights(cfg, 4321)
    frames = np.stack([synth_frame(H, W, seed=40 + s) for s in range(B)]).astype(np.float32)
    det = Detector(cfg, B, H, W, precision="split", use_cuda_graph=True, multi_semantics=True)
    try:
        det.load_weights(Wt)
        out = det.detect_host(frames)
        ref = gn_oracle.forward_multi(cfg, Wt, list(frames), stages=True)
        with frcnn.exact():
            ref64 = gn_oracle.forward_multi(cfg, Wt, list(frames), stages=False)
        K = cfg.rpn_test_post_nms_topk
        for b in range(B):
            rec = {"config": "R50-GN-multi", "image": b}
            pc = int(det.get_stage("proposal_count")[b].reshape(-1)[0])
            rb = ref["per_image"][b]["proposal_boxes"]
            assert pc == len(rb)
            pb = det.get_stage("proposal_boxes")[b].reshape(K, 4)[:pc]
            assert max(set_dist(pb, rb), set_dist(rb, pb)) < 1.5e-3
            r, rr, r64 = int(out["valid"][b]), int(ref["final_valid_indices"][b]), int(ref64["final_valid_indices"][b])
            got = (out["labels"][b, :r], out["boxes"][b, :r], out["probs"][b, :r])
            final_margins(*got, ref["final_labels"][b, :rr], ref["final_boxes"][b, :rr], ref["final_probs"][b, :rr], rec)
            exact_margins(*got, (ref["final_labels"][b, :rr], ref["final_boxes"][b, :rr], ref["final_probs"][b, :rr]),
                          (ref64["final_labels"][b, :r64], ref64["final_boxes"][b, :r64], ref64["final_probs"][b, :r64]),
                          rec)
            log_margins(rec)
            # DESIGN 2.1: counts and class ids bit-exact, boxes within 1e-3 px of the exact evaluation and, against the
            # float32 port, within 1e-3 px plus the port's own distance from the exact evaluation on this frame
            assert rec["final"] == rec["final_ref"] and rec["labels_sorted_equal"]
            assert rec["gpu_to_exact"] < 1e-3, rec
            assert rec["final_set_dist"] < 1e-3 + rec["oracle32_to_exact"], rec
            assert rec["final"] > 0
    finally:
        det.close()


@pytest.mark.parametrize("use_gn,conv_head", [(True, False), (False, True)])
def test_other_flag_combinations_small(use_gn, conv_head):
    cfg = _cfg(resnet_num_block=(1, 1, 2, 1), max_size=256, short_edge_size=192, use_gn=use_gn,
               use_conv_frcnn_head=conv_head)
    _stage_parity(cfg, 192, 256, (5,), "gn%d_convhead%d" % (use_gn, conv_head), 17)


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
        a["c5"] = det.get_stage("c5")
        a["p2"] = det.get_stage("p2")
        return a
    finally:
        det.close()


def test_determinism_graph_and_half_batch_streams(monkeypatch):
    """Two passes are bit-identical, graph replay equals eager, and the default dual-stream half-batch plan equals
    B2_SPLIT=1 (the GroupNorm statistics of an image do not depend on the batch it is in)."""
    from object_detection_tracking_b200.synth import synth_frame, synth_weights
    cfg = _cfg(resnet_num_block=(1, 1, 2, 2), max_size=256, short_edge_size=192, num_class=81, use_gn=True,
               use_conv_frcnn_head=True, im_batch_size=4)
    Wt = synth_weights(cfg, 99)
    frames = np.stack([synth_frame(192, 256, seed=60 + s) for s in range(4)]).astype(np.float32)
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


def test_given_box_features_gn():
    from object_detection_tracking_b200.backend import Session, get_model_feat
    from object_detection_tracking_b200.synth import synth_frame, synth_weights
    cfg = _cfg(**SMALL)
    Wt = synth_weights(cfg, 99)
    frame = synth_frame(192, 256, seed=8).astype(np.float32)
    boxes = np.array([[10, 12, 80, 90], [100, 20, 250, 180], [0, 0, 255, 191], [30.5, 40.25, 31.5, 41.0]], np.float32)
    model = get_model_feat(cfg)
    model.set_weights(Wt)
    got = Session().run(model.final_box_features, feed_dict=model.get_feed_dict(frame, boxes))
    ref = gn_oracle.forward_givenbox(cfg, Wt, frame, boxes)
    assert got.shape == ref.shape == (4, 256)
    assert np.abs(got - ref).max() / np.abs(ref).max() < 1e-4
