"""Batched EfficientDet (b2_effdet_detect_batch): a context created with batch B runs up to B independent frames of any
sizes in one pass, and every output of image b -- count, boxes, scores, classes, levels, box_feat, image_scale -- is bit
for bit what b2_effdet_detect(frame_b) gives on a batch-1 context with the same configuration, weights and precision.
There is no tolerance anywhere in this file: a difference is a bug."""
import math

import numpy as np
import pytest

import effdet_post_inputs as ep

pytestmark = pytest.mark.gpu

F32 = np.float32
POST, BOX_FEAT = 4, 8                      # B2_EFFDET_PHASE_POST / _BOX_FEAT
OUT_KEYS = ("final_boxes", "final_probs", "final_labels", "levels", "fpn_box_feat")
NET_STAGES = ["image", "c3", "c4", "c5"] + ["%s%d" % (k, l) for k in ("fpn", "cls", "box") for l in range(3, 8)]


def textured(h, w, seed):
    rng = np.random.default_rng(seed)
    base = rng.integers(0, 256, (h // 8 + 1, w // 8 + 1, 3)).astype(np.float32)
    img = np.kron(base, np.ones((8, 8, 1), np.float32))[:h, :w]
    return np.clip(img + rng.standard_normal((h, w, 3)) * 12, 0, 255).astype(np.uint8)


# frames whose squeeze-excite gates differ sharply, in three different sizes
FRAMES = [textured(300, 500, 3), np.zeros((240, 320, 3), np.uint8), np.full((200, 190, 3), 255, np.uint8),
          textured(128, 256, 9)]


def same_bits(a, b):
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    if a.dtype == F32:
        return np.array_equal(a.view(np.int32), b.view(np.int32))
    return np.array_equal(a, b)


def assert_same_result(got, exp, what):
    for k in OUT_KEYS:
        assert same_bits(got[k], exp[k]), "%s: %s not bit-identical (%s vs %s rows)" % (what, k, len(got[k]), len(exp[k]))
    assert np.float32(got["image_scale"]).view(np.int32) == np.float32(exp["image_scale"]).view(np.int32), what


def weights(det, cfg, tweak=None):
    from object_detection_tracking_b200.effdet_config import BACKBONE_OF
    from object_detection_tracking_b200.synth import synth_effdet_weights, synth_efficientnet_weights
    Wt = dict(synth_effdet_weights(cfg))
    Wt.update(synth_efficientnet_weights(BACKBONE_OF[det]))
    if tweak is not None:
        tweak(Wt)
    return Wt


def mbconv_blocks(backbone):
    """Blocks of EfficientNet-b<i> (efficientnet_model.py: the seven stages' repeats times the depth coefficient)."""
    depth = (1.0, 1.1, 1.2, 1.4, 1.8, 2.2, 2.6, 3.1)[int(backbone[-1])]
    return sum(int(math.ceil(depth * r)) for r in (1, 2, 2, 3, 3, 4, 1))


class D0:
    """A batch-1 and a batch-3 context of one small D0 configuration, and the batch-1 reference of every frame."""

    def __init__(self, precision):
        from object_detection_tracking_b200.effdet import EffdetEngine
        from object_detection_tracking_b200.effdet_config import BACKBONE_OF, make_effdet_config
        self.cfg = make_effdet_config("efficientdet-d0", 128, 256, fpn_cell_repeats=2, box_class_repeats=2)
        self.bb = BACKBONE_OF["efficientdet-d0"]
        Wt = weights("efficientdet-d0", self.cfg)
        self.one = EffdetEngine(self.cfg, Wt, precision=precision, backbone=self.bb)
        self.ref, self.ref_stages = [], []
        for f in FRAMES:
            self.ref.append(self.one.detect(f))
            self.ref_stages.append({n: self.one.stage(n) for n in NET_STAGES})
        self.many = EffdetEngine(self.cfg, Wt, precision=precision, backbone=self.bb, batch=3)

    def close(self):
        self.one.close()
        self.many.close()


@pytest.fixture(scope="module", params=["split", "fp16"])
def d0(request):
    c = D0(request.param)
    yield c
    c.close()


# ---- 1. whole-frame detect, frames of three sizes --------------------------------------------------------------------
def test_each_image_equals_the_batch1_context(d0):
    outs = d0.many.detect_batch(FRAMES[:3])
    assert len(outs) == 3
    assert any(len(r["final_probs"]) for r in d0.ref[:3])
    for b in range(3):
        assert_same_result(outs[b], d0.ref[b], "image %d" % b)


# ---- 2. stages, so that a difference is localised --------------------------------------------------------------------
def test_stages_of_each_image_equal_the_batch1_stages(d0):
    d0.many.detect_batch(FRAMES[:3])
    for name in NET_STAGES:
        every = d0.many.stage(name)
        assert every.shape[0] == 3, (name, every.shape)
        for b in range(3):
            assert same_bits(d0.many.stage(name, image=b), d0.ref_stages[b][name]), "%s of image %d" % (name, b)
            assert same_bits(every[b], d0.ref_stages[b][name]), name


# ---- 3. isolation: order, short batches, no state carried between calls ---------------------------------------------
def test_permuting_the_frames_permutes_the_outputs(d0):
    for order in ((2, 0, 1), (1, 2, 0), (3, 1, 2)):
        outs = d0.many.detect_batch([FRAMES[i] for i in order])
        for b, i in enumerate(order):
            assert_same_result(outs[b], d0.ref[i], "order %s, image %d" % (order, b))


def test_short_batches_return_n_results(d0):
    for idx in ((1,), (3, 0)):
        outs = d0.many.detect_batch([FRAMES[i] for i in idx])
        assert len(outs) == len(idx)
        for b, i in enumerate(idx):
            assert_same_result(outs[b], d0.ref[i], "short batch %s, image %d" % (idx, b))
    with pytest.raises(ValueError):
        d0.many.detect_batch(FRAMES)                           # 4 frames into a batch of 3
    with pytest.raises(RuntimeError, match="detect_batch"):
        d0.many.detect(FRAMES[0])                              # the single-frame call refuses a batch context


def test_no_per_image_state_leaks_between_calls(d0):
    """The black frame after the textured one in the same slot (and back): no stale top-k state, count or output rows."""
    seqs = [(0, 1, 2), (1, 2, 0), (0, 1, 2), (2, 2, 2), (1, 1, 1), (0, 1, 2)]
    for seq in seqs:
        outs = d0.many.detect_batch([FRAMES[i] for i in seq])
        for b, i in enumerate(seq):
            assert_same_result(outs[b], d0.ref[i], "sequence %s, image %d" % (seq, b))
        final = d0.many.stage("final_count")
        assert [int(v) for v in final.reshape(-1)] == [len(d0.ref[i]["final_probs"]) for i in seq]


# ---- 5. launch count -------------------------------------------------------------------------------------------------
def test_only_the_projections_launch_per_image(d0):
    n_blocks = mbconv_blocks(d0.bb)
    assert n_blocks == 16
    assert d0.many.num_launches == d0.one.num_launches + (3 - 1) * n_blocks


# ---- 4. post-processing on adversarial inputs, per image -------------------------------------------------------------
class PostCtx:
    def __init__(self, batch, name="efficientdet-d0", h=128, w=256, **over):
        from object_detection_tracking_b200.effdet import EffdetEngine
        from object_detection_tracking_b200.effdet_config import make_effdet_config
        from object_detection_tracking_b200.synth import synth_effdet_weights
        self.cfg = make_effdet_config(name, h, w, fpn_cell_repeats=1, box_class_repeats=1, **over)
        W = synth_effdet_weights(self.cfg)
        self.one = EffdetEngine(self.cfg, W)
        self.many = EffdetEngine(self.cfg, W, batch=batch)
        self.sizes = ep.level_sizes(self.cfg)
        self.na, self.nc, self.F = ep.num_anchors(self.cfg), self.cfg.num_classes, self.cfg.fpn_num_filters
        self.total = ep.level_offsets(self.cfg)[1]

    def close(self):
        self.one.close()
        self.many.close()

    def stages(self, case):
        """(cls, box, feats, scale) -> {stage name: stored array}"""
        cls, box, feats, scale = case
        st = {}
        for l in range(3, 8):
            st["cls%d" % l] = ep.padded(cls[l], ep.pad16(self.na * self.nc))
            st["box%d" % l] = ep.padded(box[l], ep.pad16(self.na * 4))
            st["fpn%d" % l] = ep.padded(feats[l], ep.pad64(self.F), F32(0))
        st["image_scale"] = np.array([scale], F32)
        return st

    def check(self, cases):
        from object_detection_tracking_b200.effdet import POST_STAGES
        per = [self.stages(c) for c in cases]
        for name in per[0]:
            self.many.set_stage(name, np.stack([p[name] for p in per]))
        self.many.run_phases(POST | BOX_FEAT)
        counts = []
        for b, st in enumerate(per):
            for name, v in st.items():
                self.one.set_stage(name, v)
            self.one.run_phases(POST | BOX_FEAT)
            n = int(self.one.stage("topk_count")[0])
            assert int(self.many.stage("topk_count", image=b)[0]) == n, ("topk_count", b)
            for name in POST_STAGES:
                exp, got = self.one.stage(name), self.many.stage(name, image=b)
                if name.startswith("topk_") and name != "topk_count":
                    exp, got = exp[:n], got[:n]                 # rows past the count are scratch
                assert same_bits(got, exp), "%s of image %d" % (name, b)
            counts.append(int(self.one.stage("final_count")[0]))
        return counts


def feats_of(c, salt):
    return {l: ep.feature_values(1, h, w, c.F, salt=salt + l)[0] for l, (h, w) in c.sizes.items()}


def test_post_processing_per_image_on_adversarial_inputs():
    c = PostCtx(5)
    try:
        rng = np.random.default_rng(21)
        split = lambda x: ep.split_levels(c.cfg, x, c.na * c.nc)
        deltas = lambda s: ep.exact_deltas(c.cfg, np.random.default_rng(s))
        k = c.cfg.max_detection_topk
        ties = ep.si.quantised_logits(rng, c.total, k)                  # thousands of ties across the k-th value
        s = np.sort(ties)[::-1]
        assert s[k - 1] == s[k]
        zeros = ep.signed_zero_logits(rng, c.total, 2000)               # +0.0 / -0.0 at the k-th value
        dense = rng.standard_normal(c.total).astype(F32)                # the output cap of 100
        none = np.full(c.total, F32(-30))                               # every score below the threshold
        band = ep.band_logits(rng, c.total, k)                          # ties in every radix block
        cases = [(split(ties), deltas(1), feats_of(c, 10), 1.0), (split(zeros), deltas(2), feats_of(c, 20), 1.37),
                 (split(dense), deltas(3), feats_of(c, 30), 0.5), (split(none), deltas(4), feats_of(c, 40), 2.0),
                 (split(band), deltas(5), feats_of(c, 50), 1.0)]
        counts = c.check(cases)
        assert counts[2] == c.cfg.result_per_im and counts[3] == 0 and counts[1] > 0
        # the same images in another order, then again: nothing carried over from the previous run
        order = [3, 0, 4, 2, 1]
        assert c.check([cases[i] for i in order]) == [counts[i] for i in order]
    finally:
        c.close()


def test_post_processing_d7_geometry_per_image():
    """D7 at 1536^2 (39.8 M logits per image over the 1056 radix blocks), two images with ties in every block."""
    c = PostCtx(2, name="efficientdet-d7", h=1536, w=1536)
    try:
        k = c.cfg.max_detection_topk
        cases = []
        for seed in (3, 4):
            x = ep.band_logits(np.random.default_rng(seed), c.total, k)
            cls = ep.split_levels(c.cfg, x, c.na * c.nc)
            del x
            cases.append((cls, ep.exact_deltas(c.cfg, np.random.default_rng(seed)), feats_of(c, seed), 1.0 + seed / 8))
        c.check(cases)
    finally:
        c.close()


# ---- 6. the headline configuration: D7 at 1536^2, batch 4 ------------------------------------------------------------
def _condition_d7_heads(Wt):
    """As test_effdet_gpu.py: scale the two predict kernels so D7's deep heads give a trained detector's output range."""
    Wt["class_net/class-predict/pointwise_kernel"] = Wt["class_net/class-predict/pointwise_kernel"] * np.float32(0.03)
    Wt["box_net/box-predict/pointwise_kernel"] = Wt["box_net/box-predict/pointwise_kernel"] * np.float32(0.08)


def test_d7_full_size_batch4_equals_batch1():
    from object_detection_tracking_b200.effdet import EffdetEngine
    from object_detection_tracking_b200.effdet_config import BACKBONE_OF, make_effdet_config
    cfg = make_effdet_config("efficientdet-d7", 1536, 1536)
    Wt = weights("efficientdet-d7", cfg, tweak=_condition_d7_heads)
    # the frame of test_d7_full_size_matches_oracle, then three other cameras
    frames = [textured(1080, 1920, 3), textured(720, 1280, 4), textured(1536, 1536, 5), np.zeros((480, 640, 3), np.uint8)]
    one = EffdetEngine(cfg, Wt, backbone=BACKBONE_OF["efficientdet-d7"])
    try:
        ref = [one.detect(f) for f in frames]
    finally:
        one.close()                                            # the two contexts never share device memory
    assert len(ref[0]["final_probs"]) > 0
    many = EffdetEngine(cfg, Wt, backbone=BACKBONE_OF["efficientdet-d7"], batch=4)
    try:
        outs = many.detect_batch(frames)
        for b in range(4):
            assert_same_result(outs[b], ref[b], "D7 image %d" % b)
    finally:
        many.close()


# ---- 7. the batch drivers' call surface ------------------------------------------------------------------------------
def test_multi_model_object_drop_in():
    """The consumer loop of obj_detect_tracking_multi_queuer.py:472-515 against get_model(config, is_multi=True)."""
    from types import SimpleNamespace
    from object_detection_tracking_b200.backend import EfficientDet, EfficientDet_multi, Session, get_model
    from object_detection_tracking_b200.effdet_config import make_effdet_config
    config = SimpleNamespace(is_efficientdet=True, efficientdet_modelname="efficientdet-d0", short_edge_size=128,
                             max_size=256, efficientdet_min_level=3, efficientdet_max_level=7,
                             efficientdet_max_detection_topk=5000, result_score_thres=1e-4, result_per_im=100,
                             use_partial_classes=True, partial_classes=["person", "car", "bus", "truck", "bicycle"],
                             is_load_from_pb=False)
    Wt = weights("efficientdet-d0", make_effdet_config("efficientdet-d0", 128, 256))
    single = get_model(config, gpuid=0)
    model = get_model(config, gpuid=0, is_multi=True)
    assert isinstance(model, EfficientDet_multi) and type(single) is EfficientDet
    single.set_weights(Wt)
    model.set_weights(Wt)
    sess = Session()
    frame_stack = [(FRAMES[0].astype(np.float32), 1.0, 0), (FRAMES[3].astype(np.float32), 1.0, 1),
                   (FRAMES[0].astype(np.float32), 1.0, 2)]             # the driver pads a short batch with its last frame
    valid_frame_num = 2
    resized_images, scales, frame_idxs = zip(*frame_stack)
    feed_dict = model.get_feed_dict_forward_multi(resized_images)
    sess_input = [model.final_boxes, model.final_labels, model.final_probs, model.final_valid_indices, model.fpn_box_feat]
    batch_boxes, batch_labels, batch_probs, valid_indices, batch_box_feats = sess.run(sess_input, feed_dict=feed_dict)
    assert np.sum(valid_indices) == batch_box_feats.shape[0]
    m = config.result_per_im
    assert batch_boxes.shape == (3, m, 4) and batch_labels.shape == (3, m) and batch_probs.shape == (3, m)
    assert batch_labels.dtype == np.float32 and valid_indices.shape == (3,)
    for b in range(valid_frame_num):
        final_boxes = batch_boxes[b][:valid_indices[b]]
        final_labels = batch_labels[b][:valid_indices[b]]
        final_probs = batch_probs[b][:valid_indices[b]]
        previous_box_num = sum(valid_indices[:b])
        box_feats = batch_box_feats[previous_box_num:previous_box_num + valid_indices[b]]
        assert len(box_feats) == len(final_boxes) > 0
        sb, sl, sp, sf = sess.run([single.final_boxes, single.final_labels, single.final_probs, single.fpn_box_feat],
                                  feed_dict=single.get_feed_dict_forward(resized_images[b]))
        assert same_bits(final_boxes, sb) and same_bits(final_probs, sp) and same_bits(box_feats, sf)
        np.testing.assert_array_equal(final_labels, sl.astype(np.float32))
        assert final_labels.min() >= 1 and final_labels.max() <= 5
        assert np.all(batch_boxes[b][valid_indices[b]:] == 0) and np.all(batch_probs[b][valid_indices[b]:] == 0)
