"""main.py --mode forward's fetches on the GPU (main.py:1540-1870).

The scene feature fpn_feature (models.py:517-518) bit for bit against the oracle's resize applied to the engine's own p5,
in split and fp16 precision, batch 1 and 2, at 192x256 (a 6x8 p5, upsampled), 720x1280 and 1088x1920; the backbone-only
pass (--just_feat) against a full pass, with and without the CUDA graph; the proposals (--get_rpn_out) bit for bit against
the engine's stage, in the single-image and the batch layout; the use_cpu_nms outputs (--no_nms / --save_all_box) as a
bit-exact re-layout of the engine's decoded boxes, probabilities and proposals, on the class-specific head with the
small-object branch and on the class-agnostic head; the full-size R101 720x1280 detector's feature, proposals and use_cpu_nms
outputs against the oracle within the baseline tests' bounds; and main.py's --gpu N loop restated with two models on one
device."""
import numpy as np
import pytest

import forward_oracle

pytestmark = pytest.mark.gpu

SMALL = dict(resnet_num_block=(1, 1, 2, 1), max_size=256, short_edge_size=192)


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


def _frames(B, H, W, seed=0):
    from object_detection_tracking_b200.synth import synth_frame
    return np.stack([synth_frame(H, W, seed + b) for b in range(B)]).astype(np.float32)


def _cfg(**kw):
    from object_detection_tracking_b200.config import make_config
    return make_config(**dict(SMALL, **kw))


def set_dist(a, b):
    if len(a) == 0:
        return 0.0
    d = np.abs(a[:, None, :].astype(np.float64) - b[None, :, :].astype(np.float64)).max(-1)
    return float(d.min(1).max())


@pytest.mark.parametrize("precision", ["split", "fp16"])
@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("H,W", [(192, 256), (720, 1280), (1088, 1920)])
def test_fpn_feature_kernel_bit_exact(H, W, B, precision):
    from object_detection_tracking_b200.config import backbone_geometry
    from object_detection_tracking_b200.engine import Detector
    from object_detection_tracking_b200.synth import synth_weights
    cfg = _cfg(max_size=max(H, W), short_edge_size=min(H, W))
    h, w = backbone_geometry(H, W, cfg)["p_full"][3]
    assert (h, w) == {192: (6, 8), 720: (23, 40), 1088: (34, 60)}[H]
    det = Detector(cfg, B, H, W, precision=precision)
    try:
        det.load_weights(synth_weights(cfg, 1234))
        det.detect_host(_frames(B, H, W, seed=3 * B))
        got = det.fpn_feature()
        p5 = det.get_stage("p5")
        assert p5.shape[1] >= h and p5.shape[2] >= w
        assert got.shape == (B, 7, 7, 256)
        for b in range(B):
            want = forward_oracle.fpn_feature(p5[b, :h, :w].transpose(2, 0, 1))[0]
            assert np.array_equal(_bits(got[b]), _bits(want)), (b, np.abs(got[b] - want).max())
    finally:
        det.close()


@pytest.mark.parametrize("graph", [True, False])
def test_backbone_only_pass(graph):
    """Batch 2 (the forked two-stream backbone): the feature-only pass equals a full pass + the resize of its p5, launches
    fewer kernels, and a later full pass is byte-identical to one before it."""
    from object_detection_tracking_b200.engine import Detector
    from object_detection_tracking_b200.synth import synth_weights
    cfg = _cfg()
    B, H, W = 2, 192, 256
    det = Detector(cfg, B, H, W, use_cuda_graph=graph)
    try:
        det.load_weights(synth_weights(cfg, 1234))
        f1, f2 = _frames(B, H, W, 0), _frames(B, H, W, 10)
        out1 = {k: v.copy() for k, v in det.detect_host(f1).items()}
        props1 = det.get_proposals()
        full = det.fpn_feature()
        assert det.fpn_feature_launches() < det.kernel_launches()
        only = det.fpn_feature(f1)
        assert np.array_equal(_bits(only), _bits(full))
        other = det.fpn_feature(f2)
        assert not np.array_equal(_bits(other), _bits(full))
        assert np.array_equal(_bits(det.fpn_feature()), _bits(other))
        stale = det.get_proposals()                              # past the FPN nothing ran
        assert all(_same(stale[k], props1[k]) for k in props1)
        out2 = det.detect_host(f1)
        for k in out1:
            assert _same(out2[k], out1[k]), k
        assert np.array_equal(_bits(det.fpn_feature()), _bits(full))
    finally:
        det.close()


def test_proposals_single_image_match_stage():
    from object_detection_tracking_b200.backend import Mask_RCNN_FPN, Session
    from object_detection_tracking_b200.synth import synth_weights
    cfg = _cfg()
    m = Mask_RCNN_FPN(cfg)
    m.set_weights(synth_weights(cfg, 1234))
    frame = _frames(1, 192, 256, 4)[0]
    pb, ps, boxes = Session().run([m.proposal_boxes, m.proposal_scores, m.final_boxes], m.get_feed_dict_forward(frame))
    det = m._last_det
    K = cfg.rpn_test_post_nms_topk
    n = int(det.get_stage("proposal_count").reshape(-1)[0])
    assert n > 0 and pb.shape == (n, 4) and ps.shape == (n,)
    assert _same(pb, det.get_stage("proposal_boxes").reshape(K, 4)[:n])
    assert _same(ps, det.get_stage("proposal_scores").reshape(K)[:n])
    assert np.all(ps[:-1] >= ps[1:])                             # score descending
    assert len(boxes) > 0


def test_proposals_batch_layout_batch2():
    """Mask_RCNN_FPN_multi at batch 2: [M, 5] rows (image index, box) image by image, bit for bit the engine's stages, and
    each image's set within 1.5e-3 of the oracle's batch-graph proposals."""
    from object_detection_tracking_b200.backend import Mask_RCNN_FPN_multi, Session
    from object_detection_tracking_b200.synth import synth_weights
    from oracle import frcnn
    cfg = _cfg(im_batch_size=2)
    Wt = synth_weights(cfg, 1234)
    m = Mask_RCNN_FPN_multi(cfg)
    m.set_weights(Wt)
    frames = _frames(2, 192, 256, 7)
    pb, ps = Session().run([m.proposal_boxes, m.proposal_scores], m.get_feed_dict_forward_multi(list(frames)))
    det = m._last_det
    K = cfg.rpn_test_post_nms_topk
    count = det.get_stage("proposal_count").reshape(2)
    sb, ss = det.get_stage("proposal_boxes").reshape(2, K, 4), det.get_stage("proposal_scores").reshape(2, K)
    assert pb.shape == (int(count.sum()), 5) and ps.shape == (int(count.sum()),) and count.min() > 1
    ref = frcnn.forward_multi(cfg, Wt, list(frames), stages=True)
    off = 0
    for b in range(2):
        n = int(count[b])
        rows = pb[off:off + n]
        assert np.all(rows[:, 0] == b)
        assert _same(rows[:, 1:], sb[b, :n]) and _same(ps[off:off + n], ss[b, :n])
        rb = ref["per_image"][b]["proposal_boxes"]
        assert n == len(rb)
        assert max(set_dist(rows[:, 1:], rb), set_dist(rb, rows[:, 1:])) < 1.5e-3
        off += n


@pytest.mark.parametrize("head", ["class_specific_small_objects", "class_agnostic"])
def test_use_cpu_nms_is_a_relayout_of_the_engine(head):
    from object_detection_tracking_b200.backend import Mask_RCNN_FPN, Session
    from object_detection_tracking_b200.synth import synth_weights
    kw = (dict(num_class=17, use_small_object_head=True, small_objects=["Bike"]) if head != "class_agnostic"
          else dict(use_frcnn_class_agnostic=True, version=4))
    cfg = _cfg(use_cpu_nms=True, add_mask=True, **kw)
    Wt = synth_weights(cfg, 5)
    m = Mask_RCNN_FPN(cfg)
    assert m.use_cpu_nms and not m.config.add_mask
    m.set_weights(Wt)
    frame = _frames(1, 192, 256, 2)[0]
    fetch = [m.final_boxes, m.final_labels, m.final_probs]
    if m.config.use_small_object_head:
        fetch += [m.so_final_boxes, m.so_final_labels, m.so_final_probs]
    out = Session().run(fetch, m.get_feed_dict_forward(frame))
    det = m._last_det
    K, C = cfg.rpn_test_post_nms_topk, cfg.num_class
    n = int(det.get_stage("proposal_count").reshape(-1)[0])
    assert n > 0
    boxes, rois, probs = out[0], out[1], out[2]
    assert boxes.shape == (C - 1, n, 4) and probs.shape == (C - 1, n) and rois.shape == (n, 4)
    assert _same(boxes, np.ascontiguousarray(det.get_stage("dec_boxes").reshape(K, C - 1, 4)[:n].transpose(1, 0, 2)))
    assert _same(probs, np.ascontiguousarray(det.get_stage("probs").reshape(K, C)[:n, 1:].T))
    assert _same(rois, det.get_stage("proposal_boxes").reshape(K, 4)[:n])
    if head == "class_agnostic":
        assert _same(boxes, np.ascontiguousarray(np.broadcast_to(boxes[:1], boxes.shape)))   # main.py:1811-1814
    else:
        # the small-object branch is built before the early return: the same outputs as the NMS graph's
        plain = Mask_RCNN_FPN(_cfg(**kw))
        plain.set_weights(Wt)
        so = Session().run([plain.so_final_boxes, plain.so_final_labels, plain.so_final_probs],
                           plain.get_feed_dict_forward(frame))
        for a, b in zip(out[3:], so):
            assert _same(a, b)
        assert len(out[3]) == len(out[4]) == len(out[5])


def test_r101_720x1280_against_oracle():
    """The full-size R101 detector (make_config's defaults) through Session.run: fpn_feature within the p_rel bound that
    the baseline tests hold p5 to, the proposals within their set distance, and the use_cpu_nms outputs within the final
    boxes' and probabilities' bounds of the oracle's head_postprocess, row by row of matching proposals."""
    from object_detection_tracking_b200.backend import Mask_RCNN_FPN, Session
    from object_detection_tracking_b200.synth import synth_frame, synth_weights
    from oracle import frcnn
    from object_detection_tracking_b200.config import make_config
    cfg = make_config(use_cpu_nms=True)
    Wt = synth_weights(cfg, 1234)
    m = Mask_RCNN_FPN(cfg)
    m.set_weights(Wt)
    frame = synth_frame(720, 1280, seed=1).astype(np.float32)
    boxes, rois, probs, pb, ps, feat = Session().run(
        [m.final_boxes, m.final_labels, m.final_probs, m.proposal_boxes, m.proposal_scores, m.fpn_feature],
        m.get_feed_dict_forward(frame))
    o = frcnn.forward(cfg, Wt, frame)
    want = forward_oracle.fpn_feature(o["p23456"][3])
    assert feat.shape == want.shape == (1, 7, 7, 256)
    p_rel = float(np.abs(feat.astype(np.float64) - want).max() / np.abs(want).max())
    assert p_rel < 1e-4, p_rel
    n = len(o["proposal_scores"])
    assert pb.shape == (n, 4) and rois.shape == (n, 4) and _same(rois, pb)
    assert max(set_dist(pb, o["proposal_boxes"]), set_dist(o["proposal_boxes"], pb)) < 1.5e-3
    d = np.abs(pb[:, None, :].astype(np.float64) - o["proposal_boxes"][None].astype(np.float64)).max(-1)
    j = d.argmin(1)                                              # the oracle's row of each proposal
    dec, oprobs = o["decoded_boxes"], o["probs"]
    assert boxes.shape == (cfg.num_class - 1, n, 4) and probs.shape == (cfg.num_class - 1, n)
    box_err = float(np.abs(boxes - dec[j].transpose(1, 0, 2)).max())
    prob_err = float(np.abs(probs - oprobs[j, 1:].T).max())
    assert box_err < 1.5e-3 and prob_err < 1e-3, (box_err, prob_err)


def test_driver_loop_two_models_one_device():
    """main.py:1571-1583, 1667-1728 with --gpu 2 --im_batch_size 2, both models on device 0: one sess.run over both
    models' fetches gives each image what a run of its own gives; --just_feat's run gives the same features."""
    from object_detection_tracking_b200.backend import Session, get_model
    from object_detection_tracking_b200.synth import synth_weights
    cfg = _cfg()
    Wt = synth_weights(cfg, 1234)
    models = [get_model(cfg, 0) for _ in range(2)]
    for m in models:
        m.set_weights(Wt)
    images = list(_frames(2, 192, 256, 20))
    sess = Session()
    feed_dict = {}
    for i, m in enumerate(models):
        feed_dict.update(m.get_feed_dict_forward(images[i]))
    sess_input = []
    for m in models:
        sess_input += [m.final_boxes, m.final_labels, m.final_probs, m.fpn_feature]
    outputs = sess.run(sess_input, feed_dict=feed_dict)
    feats = sess.run([m.fpn_feature for m in models], feed_dict=feed_dict)
    solo = get_model(cfg, 0)
    solo.set_weights(Wt)
    for i in range(2):
        alone = sess.run([solo.final_boxes, solo.final_labels, solo.final_probs, solo.fpn_feature],
                         feed_dict=solo.get_feed_dict_forward(images[i]))
        assert len(alone[0]) > 0
        for a, b in zip(outputs[4 * i:4 * i + 4], alone):
            assert _same(a, b)
        assert _same(feats[i], alone[3])
