"""use_bg_score on the CPU: the oracle's filtered fastrcnn_predictions (bg_score_oracle) against its op-by-op transcription
of models.py:1263-1304 + 925-932, on random and adversarial inputs; the flag-off oracle unchanged; the ABI struct."""
import copy

import numpy as np
import pytest

import bg_score_oracle as bo
from test_abi import _header_struct_words

F32 = np.float32


def _cfg(**kw):
    from object_detection_tracking_b200.config import make_config
    return make_config(**kw)


def _boxes(rng, K, nc1, grid=12):
    """[K, nc1, 4] boxes on a coarse grid: many overlaps, and exact ties of IoU."""
    xy = rng.integers(0, grid, (K, nc1, 2)).astype(F32) * F32(8)
    wh = rng.integers(1, 4, (K, nc1, 2)).astype(F32) * F32(8)
    return np.concatenate([xy, xy + wh], -1).astype(F32)


def _softmax(logits):
    from oracle import frcnn
    return frcnn.softmax(np.asarray(logits, F32))


def _quantised_logits(rng, K, nc, bg_shift=0.0):
    """Logits from a few values, so probabilities tie within and across rows."""
    lg = rng.integers(-4, 5, (K, nc)).astype(F32) / F32(2)
    lg[:, 0] += F32(bg_shift)
    return lg


def _check(boxes, probs, cfg, no_score_filter=False):
    fcfg = copy.copy(cfg)
    if no_score_filter:
        fcfg.result_score_thres = -np.inf
    got = bo.final_outputs(boxes, probs, fcfg)
    exp = bo.literal(boxes, probs, cfg, no_score_filter=no_score_filter)
    for g, e, what in zip(got, exp, ("boxes", "labels", "probs")):
        assert g.shape == e.shape and np.array_equal(g.view(np.uint8), np.ascontiguousarray(e).view(np.uint8)), what
    return got


@pytest.mark.parametrize("seed", range(6))
def test_oracle_equals_transcription_random(seed):
    rng = np.random.default_rng(seed)
    cfg = _cfg(result_per_im=int(rng.integers(5, 40)))
    K, nc = int(rng.integers(1, 120)), cfg.num_class
    probs = _softmax(rng.standard_normal((K, nc)).astype(F32) * 2 + np.r_[rng.uniform(-1, 2), np.zeros(nc - 1)])
    _check(_boxes(rng, K, nc - 1), probs, cfg)


def test_argmax_ties_and_nan():
    x = np.array([[1, 1, 0], [0, 2, 2], [np.nan, 5, 6], [1, np.nan, 2], [np.nan] * 3, [-0.0, 0.0, -1], [0, 3, np.nan]],
                 F32)
    np.testing.assert_array_equal(bo.argmax(x), [0, 1, 0, 2, 0, 0, 1])
    np.testing.assert_array_equal(bo.bg_rank(x), [-1, 0, -1, 1, -1, -1, 2])
    np.testing.assert_array_equal(bo.bg_rank(x, count=4), [-1, 0, -1, 1, -1, -1, -1])


def test_bg_class_ties_drop_the_row():
    """A row whose background logit equals its best class logit has equal probabilities and is dropped."""
    rng = np.random.default_rng(1)
    cfg = _cfg()
    K, nc = 60, cfg.num_class
    lg = _quantised_logits(rng, K, nc)
    lg[::2, 0] = lg[::2, 1:].max(1)
    probs = _softmax(lg)
    assert np.all(probs[::2, 0] == probs[::2, 1:].max(1))
    rank = bo.bg_rank(probs)
    assert np.all(rank[::2] == -1)
    _check(_boxes(rng, K, nc - 1), probs, cfg)


def test_all_rows_background_gives_empty_outputs():
    rng = np.random.default_rng(2)
    cfg = _cfg()
    probs = _softmax(_quantised_logits(rng, 50, cfg.num_class, bg_shift=10.0))
    fb, fl, fp = _check(_boxes(rng, 50, cfg.num_class - 1), probs, cfg)
    assert fb.shape == (0, 4) and fl.shape == (0,) and fp.shape == (0,)
    assert np.all(bo.bg_rank(probs) == -1)


def test_no_row_background_equals_the_unfiltered_oracle():
    from oracle import frcnn
    rng = np.random.default_rng(3)
    cfg = _cfg()
    K = 80
    probs = _softmax(_quantised_logits(rng, K, cfg.num_class, bg_shift=-10.0))
    boxes = _boxes(rng, K, cfg.num_class - 1)
    fb, fl, fp = _check(boxes, probs, cfg)
    pred, p = frcnn.fastrcnn_predictions(boxes, probs, cfg)
    assert len(pred) > 0
    np.testing.assert_array_equal(fb, boxes[pred[:, 0], pred[:, 1]])
    np.testing.assert_array_equal(fl, pred[:, 1] + 1)
    np.testing.assert_array_equal(fp, p)
    np.testing.assert_array_equal(bo.bg_rank(probs), np.arange(K))


def test_background_rows_first_move_every_box():
    """The first half of the rows are background: every kept ROI i has rank j = i - K/2, and the reference's gather takes
    ROI j's box, which here never equals ROI i's."""
    rng = np.random.default_rng(4)
    cfg = _cfg()
    K, nc = 64, cfg.num_class
    lg = _quantised_logits(rng, K, nc)
    lg[:K // 2, 0] = 20.0
    lg[K // 2:, 0] = -20.0
    probs = _softmax(lg)
    boxes = _boxes(rng, K, nc - 1)
    boxes[:, :, :2] += np.arange(K, dtype=F32)[:, None, None] * F32(1000)        # every ROI's boxes distinct
    boxes[:, :, 2:] += np.arange(K, dtype=F32)[:, None, None] * F32(1000)
    fb, fl, fp = _check(boxes, probs, cfg)
    assert len(fb) > 0
    roi = (fb[:, 0] // 1000).astype(int)                  # the ROI whose box was taken
    pred, _ = bo.fastrcnn_predictions(boxes, probs, cfg)
    np.testing.assert_array_equal(roi, pred[:, 0])
    assert np.all(roi < K // 2)                           # a background ROI's box, for every detection
    # the probabilities are the selected (non-background) ROI's
    i = pred[:, 0] + K // 2
    np.testing.assert_array_equal(fp, probs[i, pred[:, 1] + 1])


def test_partial_classes_layout():
    """With use_partial_classes the argmax runs over the [K, P + 1] gathered probabilities."""
    import partial_oracle
    rng = np.random.default_rng(5)
    cfg = _cfg(num_class=81, use_partial_classes=True, version=2, use_dilations=False)
    ids = cfg.partial_class_ids
    K = 90
    cls = rng.standard_normal((K, 81)).astype(F32) * 2
    cls[:, 0] += 1.0
    box = rng.standard_normal((K, 80, 4)).astype(F32)
    pc, _ = partial_oracle.gather(cls, box, ids)
    probs = _softmax(pc)
    assert probs.shape == (K, len(ids) + 1)
    rank = bo.bg_rank(probs)
    assert 0 < int((rank < 0).sum()) < K
    # the full 81-way argmax would drop a different set: the filter must see the partial columns only
    assert not np.array_equal(rank < 0, bo.argmax(_softmax(cls)) == 0)
    pcfg = copy.copy(cfg)
    pcfg.num_class = len(ids) + 1
    _check(_boxes(rng, K, len(ids)), probs, pcfg)


@pytest.mark.parametrize("thres", [False, True])
def test_small_object_logit_layout(thres):
    """The branch's [K, C + 1] logits: column 0 the mean background logit, negative values, no score filter unless
    use_so_score_thres."""
    rng = np.random.default_rng(6)
    cfg = _cfg(result_per_im=100)
    K, C = 20, 4
    lg = (rng.standard_normal((K, C + 1)) * 1.5 - 0.5).astype(F32)
    lg[3, 0] = lg[3, 1:].max()                                       # a tie: dropped
    lg[5] = np.nan                                                   # argmax 0: dropped
    lg[7, 2] = np.nan                                                # NaN never wins: kept if a finite class beats BG
    rank = bo.bg_rank(lg)
    assert rank[3] == -1 and rank[5] == -1 and 0 < int((rank < 0).sum()) < K
    fb, fl, fp = _check(_boxes(rng, K, C), lg, cfg, no_score_filter=not thres)
    if not thres:
        assert (fp < 0).any()


def test_forward_composes_and_flag_off_is_unchanged():
    """oracle.frcnn.forward under use_bg_score() equals the transcription on its own decoded boxes and probabilities, and
    outside it the oracle is the unfiltered one again."""
    from object_detection_tracking_b200.synth import synth_frame, synth_weights
    from oracle import frcnn
    cfg = _cfg(resnet_num_block=(1, 1, 1, 1), max_size=256, short_edge_size=192)
    frame = synth_frame(192, 256, seed=3).astype(np.float32)
    W0 = synth_weights(cfg, 7)
    Wt = bo.with_background_shift(W0, bo.background_shift(frcnn.forward(cfg, W0, frame)["cls_logits"]))
    off = frcnn.forward(cfg, Wt, frame)
    with bo.use_bg_score():
        on = frcnn.forward(cfg, Wt, frame)
    assert frcnn.fastrcnn_predictions is bo._UNFILTERED
    again = frcnn.forward(cfg, Wt, frame, stages=False)
    for k in ("final_boxes", "final_labels", "final_probs", "fpn_box_feat"):
        np.testing.assert_array_equal(again[k], off[k])
    dropped = int((bo.bg_rank(off["probs"]) < 0).sum())
    assert 0.25 * len(off["probs"]) < dropped < 0.75 * len(off["probs"])
    assert bo.min_background_margin(off["probs"]) > 1e-3
    fb, fl, fp = bo.literal(off["decoded_boxes"], off["probs"], cfg)
    np.testing.assert_array_equal(on["final_boxes"], fb)
    np.testing.assert_array_equal(on["final_labels"], fl)
    np.testing.assert_array_equal(on["final_probs"], fp)


def test_config_and_ext5():
    import ctypes
    from object_detection_tracking_b200 import _lib
    assert ctypes.sizeof(_lib.B2ConfigExt5) == 4 * _header_struct_words("b2_config_ext5")
    assert _cfg().use_bg_score is False
    assert _lib.make_config_ext5(_cfg()).use_bg_score == 0
    assert _lib.make_config_ext5(_cfg(use_bg_score=True)).use_bg_score == 1
