"""Deformable-conv detector (`use_deformable`) on the GPU.

The sampler bit for bit against the oracle's float32 sample on adversarial offsets, the whole deformable conv against
float64 torch with the tensor-core and CUDA-core paths agreeing, stage parity at a small geometry with deformable res3-res5
(also with GroupNorm and with squeeze-excite), the full-size ResNet-101 with --version 2 flags against the oracle and its
exact() evaluation (DESIGN 2.1), an image alone / in a batch part / in the full batch, that the offsets matter, the
use_dilations refusal, the given-box features and get_model."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import deform_oracle
from selection_inputs import planes_value, same_bits

pytestmark = pytest.mark.gpu

DF = dict(use_deformable=True, use_dilations=False)
F32 = np.float32


def stored(v, split):
    """What the engine's planes hold for float32 v: hi + lo / 2048 in split precision, the fp16 value otherwise."""
    return planes_value(v) if split else np.asarray(v, F32).astype(np.float16).astype(F32)


def adversarial_offsets(rng, B, H, W):
    """[B, ceil(H/2), ceil(W/2), 18]: each offset drawn from integers, halves, +-0.0, values that land exactly on 0, h - 1
    or w - 1, offsets beyond every border, huge values and ordinary fractions."""
    Ho, Wo = (H + 1) // 2, (W + 1) // 2
    base = np.zeros((B, Ho, Wo, 18), F32)
    i = np.arange(Ho)[None, :, None]
    j = np.arange(Wo)[None, None, :]
    for k, (by, bx) in enumerate(deform_oracle.TAP_BASE):
        base[..., 2 * k] = 2 * i - 1 + by
        base[..., 2 * k + 1] = 2 * j - 1 + bx
    last = np.zeros(18, F32)
    last[0::2], last[1::2] = H - 1, W - 1
    choices = [
        rng.integers(-3, 4, base.shape).astype(F32),                            # integers
        rng.integers(-3, 3, base.shape).astype(F32) + F32(0.5),                 # halves
        np.where(rng.random(base.shape) < 0.5, F32(0.0), F32(-0.0)),            # signed zeros
        (last - base).astype(F32),                                              # exactly h - 1 / w - 1
        (-base).astype(F32),                                                    # exactly 0
        rng.choice(np.array([-7.25, 9.75, -1e6, 1e6, -3e38, 3e38], F32), base.shape),   # beyond the borders, huge
        (rng.standard_normal(base.shape) * 1.5).astype(F32),                    # fractions
        (rng.standard_normal(base.shape) * 1e-3).astype(F32),                   # tiny fractions
    ]
    pick = rng.integers(0, len(choices), base.shape)
    return np.choose(pick, choices).astype(F32)


SAMPLE_CASES = {   # name: (B, H, W, C)
    "c128_b1_odd": (1, 23, 31, 128),
    "c256_b3_odd": (3, 13, 17, 256),
    "c512_b1_even": (1, 46, 80, 512),
    "c512_b3_odd": (3, 9, 11, 512),
}


@pytest.mark.parametrize("name", sorted(SAMPLE_CASES))
@pytest.mark.parametrize("split", [True, False])
def test_deform_sample_bit_exact(name, split):
    from object_detection_tracking_b200.engine import op_deform_sample
    B, H, W, C = SAMPLE_CASES[name]
    rng = np.random.default_rng(B * 1000 + H * 10 + C)
    x = (rng.standard_normal((B, H, W, C)) * 2).astype(F32)
    x[..., :8] = np.abs(x[..., :8])                                             # ReLU'd maps: +0.0 next to values
    x[:, ::3, :, 8:16] = 0.0
    off = adversarial_offsets(rng, B, H, W)
    got = op_deform_sample(x, off, split=split)
    xin = torch.from_numpy(stored(x, split).transpose(0, 3, 1, 2).copy())
    ref = deform_oracle.sample(xin, torch.from_numpy(off.transpose(0, 3, 1, 2).copy())).numpy()   # [B, 9, C, Ho, Wo]
    ref = stored(ref.transpose(0, 3, 4, 1, 2), split)
    assert got.shape == ref.shape == (B, (H + 1) // 2, (W + 1) // 2, 9, C)
    if not same_bits(got, ref):
        bad = np.argwhere(got.view(np.uint32) != ref.view(np.uint32))
        pytest.fail("%d of %d samples differ, first at %s: %r vs %r" % (len(bad), got.size, bad[0], got[tuple(bad[0])],
                                                                         ref[tuple(bad[0])]))


def ref_deform_conv64(x, ow, ob, w):
    """float64 torch: the reference's stride-1 offsets read at the centres, the sampler, the conv3d."""
    d = lambda a: torch.from_numpy(np.asarray(a, np.float64))
    xt = d(x).permute(0, 3, 1, 2)
    off = F.conv2d(F.pad(xt, (1, 1, 1, 1)), d(ow).permute(3, 2, 0, 1), d(ob))[:, :, ::2, ::2]
    s = deform_oracle.sample(xt, off)
    out = torch.einsum("nkchw,kco->nhwo", s, d(w).reshape(9, x.shape[3], w.shape[3]))
    return out.numpy(), off.permute(0, 2, 3, 1).numpy()


CONV_CASES = {   # name: (B, H, W, C, Cout)
    "c128_b2": (2, 24, 32, 128, 128),
    "c256_odd": (1, 13, 19, 256, 256),
    "c512_res5": (1, 46, 80, 512, 512),
}


@pytest.mark.parametrize("name", sorted(CONV_CASES))
@pytest.mark.parametrize("split,tol", [(True, 2e-5), (False, 5e-3)])
def test_deform_conv2d_matches_torch_fp64(name, split, tol):
    from object_detection_tracking_b200.engine import op_deform_conv2d
    B, H, W, C, Cout = CONV_CASES[name]
    rng = np.random.default_rng(H * W + C)
    x = np.maximum(rng.standard_normal((B, H, W, C)), 0).astype(F32)
    ow = (rng.standard_normal((3, 3, C, 18)) * np.sqrt(2.0 / (9 * C))).astype(F32)
    ob = (rng.standard_normal(18) * 0.5).astype(F32)
    w = (rng.standard_normal((3, 3, C, Cout)) / np.sqrt(9 * C)).astype(F32)
    ref, ref_off = ref_deform_conv64(stored(x, split), ow, ob, w)
    tc, off = op_deform_conv2d(x, ow, ob, w, impl="tcgen05", split=split, return_offsets=True)
    simt = op_deform_conv2d(x, ow, ob, w, impl="simt", split=split)
    assert tc.shape == ref.shape and np.isfinite(tc).all()
    assert np.abs(off - ref_off).max() <= tol * np.abs(ref_off).max()
    assert np.abs(tc - ref).max() <= tol * np.abs(ref).max()
    assert np.abs(tc - simt).max() <= tol * np.abs(simt).max()


def _cfg(**kw):
    from object_detection_tracking_b200.config import make_config
    return make_config(**kw)


def _stage_parity(cfg, H, W, seeds, tag, weight_seed):
    from test_baseline_configs_gpu import run_single
    with deform_oracle.graph(cfg):
        return run_single(cfg, seeds, H, W, tag, weight_seed=weight_seed)


SMALL = dict(resnet_num_block=(1, 1, 2, 1), max_size=256, short_edge_size=192, **DF)
BLOCKS = ("group1/block0", "group2/block0", "group3/block0")


@pytest.mark.parametrize("extra", [dict(), dict(use_gn=True, use_conv_frcnn_head=True), dict(use_se=True)],
                         ids=["bn", "gn", "se"])
def test_stage_parity_small_deformable(extra):
    """c2..c5, p2..p6, RPN logits, proposals, final detections and box features against deform_oracle at 192x256, with
    deformable res3, res4 and res5."""
    cfg = _cfg(**dict(SMALL, **extra))
    _stage_parity(cfg, 192, 256, (3, 4), "deform_small_" + "_".join(sorted(extra)), 99)


def test_offset_and_sample_stages_match_the_oracle():
    from object_detection_tracking_b200.engine import Detector
    from object_detection_tracking_b200.synth import synth_frame, synth_weights
    from oracle import frcnn
    from test_baseline_configs_gpu import rel
    cfg = _cfg(**SMALL)
    Wt = synth_weights(cfg, 99)
    frame = synth_frame(192, 256, seed=5).astype(F32)
    det = Detector(cfg, 1, 192, 256, precision="split", use_cuda_graph=False)
    try:
        det.load_weights(Wt)
        det.set_stage("image", frame[None])
        det.run_phases(1)
        got = {p: (det.get_stage(p + "/conv2_offset"), det.get_stage(p + "/conv2_sample")) for p in BLOCKS}
    finally:
        det.close()
    deform_oracle.forward(cfg, Wt, frame, stages=False)
    for p in BLOCKS:
        off, smp = got[p]
        roff, rsmp = deform_oracle.LAST[p + "/conv2_offset"], deform_oracle.LAST[p + "/conv2_sample"]
        assert off.shape[-1] == 32 and not off[..., 18:].any()                 # columns 18..31: the Cout_pad padding
        assert rel(off[..., :18], roff) < 1e-4, p
        assert rel(smp.reshape(rsmp.shape), rsmp) < 1e-4, p


FULL = dict(resnet_num_block=(3, 4, 23, 3), version=2, **DF)      # --version 2: no dilation; res5 block 0 deformable


def test_r101_deformable_720x1280_batch1():
    cfg = _cfg(**FULL)
    assert not cfg.use_dilations and cfg.num_class == 15
    recs = _stage_parity(cfg, 720, 1280, (11,), "deform_r101", 1234)
    assert recs[0]["final"] > 0


def test_r101_deformable_720x1280_batch8_multi():
    from test_baseline_configs_gpu import exact_margins, final_margins, log_margins
    from object_detection_tracking_b200.engine import Detector
    from object_detection_tracking_b200.synth import synth_frame, synth_weights
    from oracle import frcnn
    H, W, B = 720, 1280, 8
    cfg = _cfg(im_batch_size=B, **FULL)
    Wt = synth_weights(cfg, 1234)
    frames = np.stack([synth_frame(H, W, seed=40 + s) for s in range(B)]).astype(F32)
    det = Detector(cfg, B, H, W, precision="split", use_cuda_graph=True, multi_semantics=True)
    try:
        det.load_weights(Wt)
        out = det.detect_host(frames)
    finally:
        det.close()
    ref = deform_oracle.forward_multi(cfg, Wt, list(frames), stages=False)
    with frcnn.exact():
        ref64 = deform_oracle.forward_multi(cfg, Wt, list(frames), stages=False)
    for b in range(B):
        rec = {"config": "deform-r101-multi8", "image": b}
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


STAGES = (["c2", "c3", "c4", "c5", "p2", "p3", "p4", "p5", "p6"] + ["rpn_l%d" % i for i in range(5)] +
          [p + s for p in BLOCKS for s in ("/conv2_offset", "/conv2_sample")])


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


def test_an_image_is_bit_identical_alone_in_a_batch_part_and_in_the_full_batch(monkeypatch):
    """Graph replay equals eager; B2_SPLIT 1 / 2 / 4 give the same bits; every image's backbone, offsets, samples, FPN and
    RPN-head outputs in the batch of 4 equal those of the image run alone."""
    from object_detection_tracking_b200.synth import synth_frame, synth_weights
    cfg = _cfg(im_batch_size=4, **SMALL)
    Wt = synth_weights(cfg, 99)
    frames = np.stack([synth_frame(192, 256, seed=60 + s) for s in range(4)]).astype(F32)
    dual = _outputs(cfg, Wt, frames, use_cuda_graph=True)
    eager = _outputs(cfg, Wt, frames, use_cuda_graph=False)
    others = [eager]
    for n in ("1", "4"):
        monkeypatch.setenv("B2_SPLIT", n)
        others.append(_outputs(cfg, Wt, frames, use_cuda_graph=True))
    monkeypatch.delenv("B2_SPLIT")
    for other in others:
        for k in dual:
            np.testing.assert_array_equal(dual[k], other[k], err_msg=k)
    assert int(dual["valid"].sum()) > 0
    for k in (0, 3):
        alone = _outputs(cfg, Wt, frames[k:k + 1], use_cuda_graph=False)
        for s in STAGES:
            np.testing.assert_array_equal(dual[s][k:k + 1], alone[s], err_msg="image %d, %s" % (k, s))


def test_offsets_matter():
    """Zeroing conv2_offset changes c5, and the engine then matches the oracle's zero-offset model."""
    from object_detection_tracking_b200.synth import synth_frame, synth_weights
    from test_baseline_configs_gpu import rel
    cfg = _cfg(**SMALL)
    Wt = synth_weights(cfg, 99)
    frames = synth_frame(192, 256, seed=8).astype(F32)[None]
    Z = {k: (np.zeros_like(v) if "/conv2_offset/" in k else v) for k, v in Wt.items()}
    a = _outputs(cfg, Wt, frames)
    z = _outputs(cfg, Z, frames)
    assert rel(z["c5"], a["c5"]) > 0.05
    for p in BLOCKS:
        assert not z[p + "/conv2_offset"].any()
    ref = deform_oracle.forward(cfg, Z, frames[0])
    assert rel(z["c5"][0].transpose(2, 0, 1), ref["c2345"][3]) < 5e-5


def test_use_dilations_is_refused_by_b2_create_and_get_model():
    from object_detection_tracking_b200.backend import Session, get_model
    from object_detection_tracking_b200.engine import Detector
    from object_detection_tracking_b200.synth import synth_frame, synth_weights
    cfg = _cfg(resnet_num_block=(3, 4, 23, 3), use_deformable=True)
    assert cfg.use_dilations
    with pytest.raises(RuntimeError, match="use_deformable cannot be combined with use_dilations"):
        Detector(cfg, 1, 192, 256)
    model = get_model(cfg)
    model.set_weights(synth_weights(cfg, 1))
    with pytest.raises(RuntimeError, match="group3/block0 pads its deformable conv2 output"):
        Session().run(model.final_boxes, feed_dict=model.get_feed_dict_forward(synth_frame(192, 256, 1).astype(F32)))
    # the ResNeXt block has no deformable branch: the flag is ignored there, dilations or not
    Detector(_cfg(resnet_num_block=(1, 1, 2, 1), use_deformable=True, use_resnext=True), 1, 192, 256).close()


def test_given_box_features_deformable():
    from object_detection_tracking_b200.backend import Session, get_model_feat
    from object_detection_tracking_b200.synth import synth_frame, synth_weights
    cfg = _cfg(**SMALL)
    Wt = synth_weights(cfg, 99)
    frame = synth_frame(192, 256, seed=8).astype(F32)
    boxes = np.array([[10, 12, 80, 90], [100, 20, 250, 180], [0, 0, 255, 191], [30.5, 40.25, 31.5, 41.0]], F32)
    model = get_model_feat(cfg)
    model.set_weights(Wt)
    got = Session().run(model.final_box_features, feed_dict=model.get_feed_dict(frame, boxes))
    ref = deform_oracle.forward_givenbox(cfg, Wt, frame, boxes)
    assert got.shape == ref.shape == (4, 256)
    assert np.abs(got - ref).max() / np.abs(ref).max() < 1e-4


@pytest.mark.parametrize("is_multi", [False, True])
def test_get_model_deformable(is_multi):
    from object_detection_tracking_b200.backend import Session, get_model
    from object_detection_tracking_b200.synth import synth_frame, synth_weights
    cfg = _cfg(**SMALL)
    Wt = synth_weights(cfg, 99)
    frames = [synth_frame(192, 256, seed=70 + s).astype(F32) for s in range(2 if is_multi else 1)]
    model = get_model(cfg, is_multi=is_multi)
    model.set_weights(Wt)
    fetches = [model.final_boxes, model.final_labels, model.final_probs, model.final_valid_indices]
    if is_multi:
        boxes, labels, probs, valid = Session().run(fetches, feed_dict=model.get_feed_dict_forward_multi(frames))
        ref = deform_oracle.forward_multi(cfg, Wt, frames)
        per = [(boxes[b, :valid[b]], labels[b, :valid[b]], probs[b, :valid[b]], ref["final_boxes"][b],
                ref["final_labels"][b], ref["final_probs"][b], int(ref["final_valid_indices"][b])) for b in range(2)]
    else:
        boxes, labels, probs, valid = Session().run(fetches, feed_dict=model.get_feed_dict_forward(frames[0]))
        ref = deform_oracle.forward(cfg, Wt, frames[0], stages=False)
        per = [(boxes, labels, probs, ref["final_boxes"], ref["final_labels"], ref["final_probs"], len(ref["final_boxes"]))]
    for bx, lb, pr, rbx, rlb, rpr, n in per:
        assert len(bx) == n > 0
        got = np.concatenate([np.asarray(lb, np.float64)[:, None] * 10.0, bx, pr[:, None]], 1)
        exp = np.concatenate([np.asarray(rlb[:n], np.float64)[:, None] * 10.0, rbx[:n], rpr[:n, None]], 1)
        d = np.abs(got[:, None, :] - exp[None, :, :]).max(-1)
        assert d.min(1).max() < 2e-3 and d.min(0).max() < 2e-3, (d.min(1).max(), d.min(0).max())
