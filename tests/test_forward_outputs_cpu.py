"""main.py --mode forward's fetches on the host side: the scene feature's reference (fpn_feature, models.py:517-518)
against an independent float64 evaluation of TF's legacy bilinear at the p5 sizes of 720x1280 (23x40) and 1080x1920
(34x60), 7x7 (the identity) and 6x8 (upsampling, from a 192x256 frame through the oracle's own forward); the batch
graph's proposal assembly (models.py:2490-2521) at M = 0, 1 and more; the use_cpu_nms refusals and where the flag is
ignored (models.py:899-916); and Session.run over several model objects (main.py --gpu N)."""
import numpy as np
import pytest

import forward_oracle


def _close(got, exact):
    # five float32 roundings of values bounded by max|p5|
    return np.abs(got - exact).max() <= 6e-7 * np.abs(exact).max() + 1e-30


@pytest.mark.parametrize("h,w", [(23, 40), (34, 60), (7, 7), (6, 8)])
def test_fpn_feature_reference_matches_float64(h, w):
    rng = np.random.default_rng(h * 100 + w)
    p5 = (rng.standard_normal((256, h, w)) * rng.uniform(0.1, 30.0, (256, 1, 1))).astype(np.float32)
    got = forward_oracle.fpn_feature(p5)
    assert got.shape == (1, 7, 7, 256) and got.dtype == np.float32
    assert _close(got, forward_oracle.fpn_feature_exact(p5))
    if (h, w) == (7, 7):
        assert np.array_equal(got[0], p5.transpose(1, 2, 0))             # scale 1: every sample on a pixel
    if h < 7:
        # the last rows' upper tap ceil(y * 6/7) is clamped to h - 1 (TF's min(ceil(in), in_size - 1))
        assert any(hi == h - 1 and lo == h - 1 for lo, hi, _ in forward_oracle.taps(h))


def test_fpn_feature_of_oracle_forward_upsamples_p5():
    """A 192x256 frame has a 6x8 p5: the feature of the oracle's own forward pass, through the 7x7 upsampling."""
    from object_detection_tracking_b200.config import backbone_geometry, make_config
    from object_detection_tracking_b200.synth import synth_frame, synth_weights
    from oracle import frcnn
    cfg = make_config(resnet_num_block=(1, 1, 2, 1), max_size=256, short_edge_size=192)
    assert backbone_geometry(192, 256, cfg)["p_full"][3] == (6, 8)
    Wt = synth_weights(cfg, 1234)
    o = frcnn.forward(cfg, Wt, synth_frame(192, 256, 5).astype(np.float32))
    p5 = o["p23456"][3]
    assert p5.shape == (256, 6, 8)
    assert _close(forward_oracle.fpn_feature(p5), forward_oracle.fpn_feature_exact(p5))


def _props(counts, K=6, seed=0):
    rng = np.random.default_rng(seed)
    B = len(counts)
    boxes = rng.uniform(0, 100, (B, K, 4)).astype(np.float32)
    scores = rng.standard_normal((B, K)).astype(np.float32)
    return boxes, scores, np.asarray(counts, np.int32)


def test_batch_proposals_general():
    from object_detection_tracking_b200.backend import batch_proposals
    boxes, scores, count = _props([3, 0, 5])
    pb, ps = batch_proposals(boxes, scores, count)
    assert pb.shape == (8, 5) and ps.shape == (8,) and pb.dtype == np.float32 and ps.dtype == np.float32
    assert pb[:, 0].tolist() == [0, 0, 0, 2, 2, 2, 2, 2]                  # image index as float32, image by image
    assert np.array_equal(pb[:3, 1:], boxes[0, :3]) and np.array_equal(pb[3:, 1:], boxes[2, :5])
    assert np.array_equal(ps, np.concatenate([scores[0, :3], scores[2, :5]]))


def test_batch_proposals_none():
    from object_detection_tracking_b200.backend import batch_proposals
    pb, ps = batch_proposals(*_props([0, 0]))
    assert pb.shape == (0, 5) and ps.shape == (0,)


def test_batch_proposals_one_row_squeezes():
    """tf.squeeze(tf.where(area > 0)) of a single surviving row is a scalar index: shapes (5,) and ()."""
    from object_detection_tracking_b200.backend import batch_proposals
    boxes, scores, count = _props([0, 1])
    pb, ps = batch_proposals(boxes, scores, count)
    assert pb.shape == (5,) and ps.shape == ()
    assert pb[0] == 1.0 and np.array_equal(pb[1:], boxes[1, 0]) and float(ps) == float(scores[1, 0])


def _cfg(**kw):
    from object_detection_tracking_b200.config import make_config
    return make_config(**kw)


def test_use_cpu_nms_defaults_off():
    from object_detection_tracking_b200.backend import Mask_RCNN_FPN
    assert _cfg().use_cpu_nms is False
    assert Mask_RCNN_FPN(_cfg()).use_cpu_nms is False


def test_use_cpu_nms_refuses_a_class_subset():
    """models.py:902-903 asserts boxes.shape[1] == num_class - 1: with partial classes only all 80 pass."""
    from object_detection_tracking_b200.backend import Mask_RCNN_FPN
    cfg = _cfg(num_class=81, use_partial_classes=True, use_cpu_nms=True)
    assert len(cfg.partial_classes) < 80
    with pytest.raises(ValueError, match="models.py:902-903"):
        Mask_RCNN_FPN(cfg)
    from object_detection_tracking_b200.class_ids import coco_obj_class_to_id
    every = [n for n in coco_obj_class_to_id if n != "BG"]
    assert len(every) == 80
    assert Mask_RCNN_FPN(_cfg(num_class=81, use_partial_classes=True, partial_classes=every, use_cpu_nms=True)).use_cpu_nms


def test_use_cpu_nms_builds_without_the_mask_head():
    from object_detection_tracking_b200.backend import Mask_RCNN_FPN
    m = Mask_RCNN_FPN(_cfg(add_mask=True, use_cpu_nms=True))
    assert m.use_cpu_nms and not m.config.add_mask
    frame = np.zeros((64, 64, 3), np.float32)
    for f in (m.fpn_box_feat, m.final_masks):                 # refused before any device work
        with pytest.raises(KeyError, match="models.py:916"):
            m._run([m.final_boxes, f], m.get_feed_dict_forward(frame))


def test_use_cpu_nms_ignored_by_batch_and_frozen_models():
    from object_detection_tracking_b200.backend import Mask_RCNN_FPN, Mask_RCNN_FPN_multi
    partial = dict(num_class=81, use_partial_classes=True, add_mask=True, use_cpu_nms=True)
    m = Mask_RCNN_FPN_multi(_cfg(**partial))                  # no refusal either
    assert not m.use_cpu_nms and m.config.add_mask
    f = Mask_RCNN_FPN(_cfg(is_load_from_pb=True, **partial))
    assert not f.use_cpu_nms and f.config.add_mask


def test_batch_model_has_no_fpn_feature():
    from object_detection_tracking_b200.backend import Mask_RCNN_FPN_multi
    m = Mask_RCNN_FPN_multi(_cfg())
    with pytest.raises(KeyError, match="models.py:2085"):
        m._run([m.fpn_feature], m.get_feed_dict_forward_multi([np.zeros((64, 64, 3), np.float32)] * 2))


def test_session_run_over_two_models_keeps_fetch_order():
    """main.py --gpu 2: one sess.run over the fetches of two model objects, interleaved; each model runs once, on its own
    image of the shared feed_dict, with its own fetches only."""
    from object_detection_tracking_b200.backend import Mask_RCNN_FPN, Session
    models = [Mask_RCNN_FPN(_cfg(), gpuid=i) for i in range(2)]
    calls = []

    def stub(model):
        def run(fetches, feed_dict):
            calls.append((model, list(fetches)))
            img = feed_dict[model.image]
            return [(f.name, float(img[0, 0, 0])) for f in fetches]
        return run

    feed = {}
    for i, m in enumerate(models):
        m._run = stub(m)
        feed.update(m.get_feed_dict_forward(np.full((4, 4, 3), i + 1, np.float32)))
    a, b = models
    fetches = [a.final_boxes, a.final_labels, b.final_boxes, a.fpn_feature, b.proposal_scores, b.final_probs]
    out = Session().run(fetches, feed_dict=feed)
    assert out == [(f.name, 1.0 if f.model is a else 2.0) for f in fetches]
    assert [(m, [f.name for f in fs]) for m, fs in calls] == [
        (a, ["final_boxes:0", "final_labels:0", "fpn_feature:0"]),
        (b, ["final_boxes:0", "proposal_scores:0", "final_probs:0"])]
    calls.clear()
    assert Session().run(b.final_probs, feed_dict=feed) == ("final_probs:0", 2.0)
    assert calls == [(b, [b.final_probs])]
