"""The exactness the selection-kernel tests rely on, checked on the CPU: if a builder in selection_inputs.py stops producing
exact values, the bit-exact GPU comparisons would turn vacuous or flaky, so this fails first."""
import math

import numpy as np
import pytest

import selection_inputs as si

F32 = np.float32


@pytest.mark.parametrize("hw", [(192, 256), (512, 768), (200, 300)])
def test_rpn_deltas_decode_exactly_in_float32(hw):
    from object_detection_tracking_b200.config import make_config
    from oracle import frcnn
    from oracle.anchors import get_all_anchors
    H, W = hw
    cfg = make_config(max_size=W, short_edge_size=H)
    rng = np.random.default_rng(0)
    for lvl, (s, size) in enumerate(zip(cfg.anchor_strides, cfg.anchor_sizes)):
        fh, fw = int(math.ceil(H / s)), int(math.ceil(W / s))
        anchors = get_all_anchors(s, [size], cfg.anchor_ratios, cfg.max_size)[:fh, :fw]
        t = si.rpn_deltas(rng, fh, fw)
        assert np.all(t[..., 2:] == 0) and np.all(t * 8 == np.round(t * 8)) and np.abs(t).max() <= 1
        dec = frcnn.decode_bbox_target(t, anchors, cfg.bbox_decode_clip).astype(np.float64)
        a = anchors.astype(np.float64)
        wa, ha = a[..., 2] - a[..., 0], a[..., 3] - a[..., 1]
        xc = t[..., 0] * wa + (a[..., 0] + a[..., 2]) / 2
        yc = t[..., 1] * ha + (a[..., 1] + a[..., 3]) / 2
        exact = np.stack([xc - wa / 2, yc - ha / 2, xc + wa / 2, yc + ha / 2], -1)
        np.testing.assert_array_equal(dec, exact, err_msg="level %d" % lvl)
        # clip_boxes is a min/max of exact values: still exact
        np.testing.assert_array_equal(frcnn.clip_boxes(dec.astype(F32), hw), np.clip(exact, 0, [W, H, W, H]))


def test_quantised_logits_tie_at_the_kth_value():
    rng = np.random.default_rng(1)
    for n, k in [(9216, 300), (2304, 300), (73728, 300), (9216, 1000), (2304, 1024), (9216, 1)]:
        x = si.quantised_logits(rng, n, k)
        kth = np.sort(x)[::-1][k - 1]
        above, tied = int((x > kth).sum()), int((x == kth).sum())
        assert above < k <= above + tied and tied - (k - above) >= 100, (n, k, above, tied)


def test_feature_values_survive_the_plane_round_trip():
    v = si.feature_stage(2, (56, 80), (50, 75), 256, salt=3)
    np.testing.assert_array_equal(si.planes_value(v), v)          # fp16-exact: lo plane 0, hi + lo/2048 == v
    np.testing.assert_array_equal(v.astype(np.float16).astype(F32), v)
    body = v[:, :50, :75]
    assert np.abs(body).max() < 8 and np.all(v[:, 50:] == si.SENTINEL) and np.all(v[:, :, 75:] == si.SENTINEL)
    # neighbours along every axis differ, so a wrong row, column, channel or image shows in the output
    for ax in range(4):
        assert np.all(np.diff(body, axis=ax) != 0), ax
    assert len(np.unique(body)) > 4000


def test_plane_split_restatement_is_lossy_where_the_kernel_is():
    # planes_value is not the identity on general float32 values: the test of roi_feat exercises the lo plane
    v = np.array([1.0 / 3.0, 0.1, -2.7182817, 1e-3], F32)
    pv = si.planes_value(v)
    assert np.all(np.abs(pv - v) <= np.abs(v) * 2.0 ** -21) and not np.array_equal(pv, v)


def test_iou_threshold_pairs_sit_exactly_at_and_just_above_one_half():
    from oracle import tf_ops
    (a0, b0), (a1, b1) = si.iou_threshold_pairs()
    assert tf_ops.iou_tf(a0, b0) == F32(0.5)
    assert tf_ops.iou_tf(a1, b1) > F32(0.5)
    assert tf_ops.iou_tf(a1, b1) == np.nextafter(F32(0.5), F32(1))
    # the pairs are far apart: no cross-pair overlap
    assert tf_ops.iou_tf(a0, a1) == 0 and tf_ops.iou_tf(b0, b1) == 0


def test_signed_zero_top_k_ties_by_index_in_the_oracle():
    from oracle import tf_ops
    _, idx = tf_ops.top_k(np.array([1, -0.0, 0.0, -0.0, 0.0, -1], F32), 4)
    np.testing.assert_array_equal(idx, [0, 1, 2, 3])
