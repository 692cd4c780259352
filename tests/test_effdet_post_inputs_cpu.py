"""The exactness claims of effdet_post_inputs.py, checked on the CPU: what test_effdet_post_gpu.py compares bit for bit
must be computable bit for bit."""
import numpy as np
import pytest

import effdet_post_inputs as ep

F32 = np.float32


def _cfg(**over):
    from object_detection_tracking_b200.effdet_config import make_effdet_config
    return make_effdet_config("efficientdet-d0", 128, 256, **over)


def test_fast_top_k_equals_tf_top_k():
    from oracle import tf_ops
    rng = np.random.default_rng(0)
    cases = [ep.band_logits(rng, 5000, 300), ep.signed_zero_logits(rng, 3000, 40), ep.prefix_logits(rng, 4000, -2.5, 24),
             rng.integers(-3, 3, 2000).astype(F32), rng.standard_normal(100).astype(F32)]
    for x in cases:
        for k in (1, 7, 64, 65, 300, len(x), len(x) + 5):
            v, i = ep.fast_top_k(x, k)
            rv, ri = tf_ops.top_k(x, k)
            np.testing.assert_array_equal(i, ri)
            assert ep.same_bits(v, rv)


def test_band_logits_tie_the_kth_value_in_every_radix_block():
    rng = np.random.default_rng(1)
    n, k = 441936 * 90 // 16, 5000
    x = ep.band_logits(rng, n, k)
    s = np.sort(x)[::-1]
    assert s[k - 1] == s[k] == F32(0.75) and (x > s[k - 1]).sum() < k
    grid = min((n + 255) // 256, 132 * 8)
    chunk = (n + grid - 1) // grid
    assert grid == 1056
    assert all(np.any(x[b * chunk:(b + 1) * chunk] == F32(0.75)) for b in range(grid))


def test_key_helpers_and_prefix_logits():
    rng = np.random.default_rng(2)
    x = rng.standard_normal(10000).astype(F32)
    assert np.array_equal(np.argsort(ep.key_of(x), kind="stable"), np.argsort(x, kind="stable"))
    assert ep.key_of(np.array([0.0, -0.0], F32)).tolist() == [0x80000000] * 2
    assert ep.same_bits(ep.float_of_key(ep.key_of(x)), x)
    for bits in (8, 16, 24):
        for v in (-2.5, 3.75):
            y = ep.prefix_logits(rng, 5000, v, bits)
            assert np.all(np.isfinite(y)) and len(np.unique(y)) > 100
            assert np.all(ep.key_of(y) >> (32 - bits) == ep.key_of(np.array([v], F32))[0] >> (32 - bits))


def test_signed_zero_logits():
    x = ep.signed_zero_logits(np.random.default_rng(3), 2000, 30)
    z = x[x == 0]
    assert (x > 0).sum() == 30 and np.signbit(z).sum() > 500 and (~np.signbit(z)).sum() > 500


def test_exact_deltas_decode_exactly():
    from object_detection_tracking_b200.effdet_config import feat_sizes
    from oracle import effdet as oe
    cfg = _cfg(num_scales=1, aspect_ratios=((1.0, 1.0), (2.0, 1.0)))      # dyadic anchors
    d = ep.exact_deltas(cfg, np.random.default_rng(4))
    t = np.concatenate([d[l].reshape(-1, 4) for l in range(3, 8)])
    assert np.all(t[:, 2:] == 0) and np.all(t[:, :2] * 8 == np.round(t[:, :2] * 8))
    a = oe.anchor_boxes(cfg, feat_sizes(cfg))
    got = oe.decode_boxes(t, a).astype(np.float64)
    a64 = a.astype(np.float64)
    ha, wa = a64[:, 2] - a64[:, 0], a64[:, 3] - a64[:, 1]
    yc, xc = t[:, 0] * ha + (a64[:, 0] + a64[:, 2]) / 2, t[:, 1] * wa + (a64[:, 1] + a64[:, 3]) / 2
    np.testing.assert_array_equal(got, np.stack([yc - ha / 2, xc - wa / 2, yc + ha / 2, xc + wa / 2], 1))


def test_iou_shift_hits_the_threshold_and_one_ulp_above():
    from object_detection_tracking_b200.effdet_config import feat_sizes
    from oracle import effdet as oe
    from oracle import tf_ops
    cfg = _cfg(anchor_scale=3.0)                  # square anchors of 3 strides: neighbours overlap at IoU 1/2
    a = oe.anchor_boxes(cfg, feat_sizes(cfg))
    # level 7 (1 x 2 cells) and level 3's first two cells, anchor 0 of each (9 anchors per cell)
    for pair, target, zero in (((a[-18], a[-9]), F32(0.5), True), ((a[0], a[9]), ep.IOU_ABOVE, False)):
        t = ep.iou_shift(*pair, target)
        assert t is not None and (t == (0, 0)) == zero
        b1 = oe.decode_boxes(np.array([[t[0], t[1], 0, 0]], F32), pair[1][None])[0]
        assert tf_ops.iou_tf(pair[0], b1) == target


def test_exact_feature_boxes_pool_exactly():
    """The float32 oracle box feature of exact_feature_boxes equals its float64 evaluation, and the per-box sum of the
    49 bins is the same in any order."""
    import torch
    from oracle import effdet as oe
    cfg = _cfg(fpn_num_filters=16)
    sizes = ep.level_sizes(cfg)
    rng = np.random.default_rng(5)
    boxes, levels = ep.exact_feature_boxes(rng, sizes, 40)
    assert set(levels.tolist()) == {3, 4, 5, 6, 7}
    feats = {l: ep.feature_values(1, h, w, 16, salt=l)[0] for l, (h, w) in sizes.items()}
    for f in feats.values():
        assert np.array_equal(f.astype(np.float16).astype(F32), f)
    got = oe.box_features({l: torch.from_numpy(f.transpose(2, 0, 1)[None].copy()) for l, f in feats.items()},
                          boxes, levels, cfg)
    for i, (b, l) in enumerate(zip(boxes.astype(np.float64) / 2.0 ** levels[:, None], levels)):
        h, w = sizes[l]
        ys = ep.sample_coords(b[1], b[3], h).astype(np.float64)
        xs = ep.sample_coords(b[0], b[2], w).astype(np.float64)
        f = feats[l].astype(np.float64)

        def sample(y, x):
            if not (0 <= y <= h - 1 and 0 <= x <= w - 1):
                return np.zeros(16)
            y0, x0, y1, x1 = int(np.floor(y)), int(np.floor(x)), int(np.ceil(y)), int(np.ceil(x))
            top = f[y0, x0] + (f[y0, x1] - f[y0, x0]) * (x - x0)
            bot = f[y1, x0] + (f[y1, x1] - f[y1, x0]) * (x - x0)
            return top + (bot - top) * (y - y0)
        bins = [sum(sample(ys[2 * by + dy], xs[2 * bx + dx]) for dy in (0, 1) for dx in (0, 1)) / 4
                for by in range(7) for bx in range(7)]
        total = np.sum(bins, 0)
        assert np.array_equal(total.astype(F32).astype(np.float64), total)           # exact in float32
        np.testing.assert_array_equal(got[i], (total.astype(F32) / F32(49)).astype(F32))


def test_one_pixel_axis_samples_its_only_pixel():
    """The oracle's definition of a 1-pixel axis (TF's is undefined there): its only pixel, wherever the box lies; an
    infinite box side on a longer axis: outside."""
    from oracle import frcnn
    f = np.arange(1, 7, dtype=F32).reshape(2, 1, 3)     # [C=2, H=1, W=3]
    a = frcnn.roi_align(f, np.array([[0.25, -3.0, 2.0, 5.0]], F32), 7)
    b = frcnn.roi_align(f, np.array([[0.25, 7.0, 2.0, 9.5]], F32), 7)
    assert np.all(np.isfinite(a)) and np.all(a[:, :, :, 1:] != 0)
    np.testing.assert_array_equal(a, b)
    c = frcnn.roi_align(np.full((2, 1, 1), 3.0, F32), np.array([[-5.0, -5.0, 9.0, 9.0]], F32), 7)
    assert np.all(c == 3)
    g = np.arange(1, 13, dtype=F32).reshape(2, 2, 3)
    assert np.all(frcnn.roi_align(g, np.array([[0.0, -np.inf, 1.0, np.inf]], F32), 7) == 0)
