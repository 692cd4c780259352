"""EfficientDet's post-processing, bit for bit, on adversarial inputs: the global top-k (multi-block radix select, tie
scan and lowest-index tie write), sigmoid + anchor decode, the class-agnostic NMS (effdet.cu) and the own-level box
feature (roialign.cu level_roi_feat_kernel).

Each test writes the head outputs (cls3..7 / box3..7, with +1e30 in their padding columns) and the BiFPN levels
(fpn3..7) through the stage API, runs the post-processing phases eagerly and compares with oracle.effdet: the candidate
list before NMS (topk_*: count, classes, levels, boxes, in top-k order) and the outputs (final_*, box_feat) index-aligned
and bit for bit.  The only tolerance is on exp(): the GPU's expf and numpy's exp may differ in the last ulps, so scores
are compared within 6 ulps (4 seen) and the oracle's NMS runs on the GPU's own candidate scores and boxes.  The inputs are built by
effdet_post_inputs.py, whose exactness test_effdet_post_inputs_cpu.py checks."""
import numpy as np
import pytest

import effdet_post_inputs as ep

pytestmark = pytest.mark.gpu

F32 = np.float32
POST, BOX_FEAT = 4, 8          # B2_EFFDET_PHASE_POST / _BOX_FEAT
SCORE_ULPS = 6                 # expf against numpy's exp, through 1 / (1 + e)

CONTEXTS = {
    "base": dict(),                                                     # 128 x 256: 552 420 logits, 1056 radix blocks
    "tiny": dict(h=128, w=128, num_scales=1, aspect_ratios=((1.0, 1.0),), num_classes=1),   # 341 logits; level 7 is 1x1
    "partial": dict(num_classes=5),                                     # rows of 45 logits, 3 padding columns
    "thr": dict(result_score_thres=0.5),
    "iou": dict(anchor_scale=3.0),                                      # neighbouring anchors overlap at IoU 1/2
    "d7": dict(name="efficientdet-d7", h=1536, w=1536),                 # 441 936 anchors x 90 classes
}
for _k in (1, 64, 65, 4096, 4097, 8192):
    CONTEXTS["k%d" % _k] = dict(max_detection_topk=_k)


class Ctx:
    def __init__(self, name="efficientdet-d0", h=128, w=256, **over):
        from object_detection_tracking_b200.effdet import EffdetEngine
        from object_detection_tracking_b200.effdet_config import feat_sizes, make_effdet_config
        from object_detection_tracking_b200.synth import synth_effdet_weights
        self.cfg = make_effdet_config(name, h, w, fpn_cell_repeats=1, box_class_repeats=1, **over)
        self.eng = EffdetEngine(self.cfg, synth_effdet_weights(self.cfg))
        self.fs = feat_sizes(self.cfg)
        self.sizes = ep.level_sizes(self.cfg)
        self.na, self.nc = ep.num_anchors(self.cfg), self.cfg.num_classes
        self.offsets, self.total = ep.level_offsets(self.cfg)
        self.k, self.m, self.F = self.cfg.max_detection_topk, self.cfg.result_per_im, self.cfg.fpn_num_filters

    def split(self, flat):
        return ep.split_levels(self.cfg, flat, self.na * self.nc)


@pytest.fixture(scope="module")
def ctx():
    made = {}

    def get(name):
        if name not in made:
            made[name] = Ctx(**CONTEXTS[name])
        return made[name]
    yield get
    for c in made.values():
        c.eng.close()


def assert_bits(got, exp, what):
    assert ep.same_bits(got, exp), "%s: not bit-identical\n  got %s\n  exp %s" % (what, np.asarray(got)[:6],
                                                                                  np.asarray(exp)[:6])


def ulps(a, b):
    return np.abs(np.asarray(a, F32).view(np.int32).astype(np.int64) - np.asarray(b, F32).view(np.int32).astype(np.int64))


def set_inputs(c, cls, box, scale=1.0, feats=None):
    for l in range(3, 8):
        if cls is not None:
            c.eng.set_stage("cls%d" % l, ep.padded(cls[l], ep.pad16(c.na * c.nc)))
        if box is not None:
            c.eng.set_stage("box%d" % l, ep.padded(box[l], ep.pad16(c.na * 4)))
        if feats is not None:
            c.eng.set_stage("fpn%d" % l, ep.padded(feats[l], ep.pad64(c.F), F32(0)))
    c.eng.set_stage("image_scale", np.array([scale], F32))


def run(c, cls, box, scale=1.0, feats=None):
    """Head outputs {level: [h, w, A*C]} / {level: [h, w, A*4]} (and BiFPN levels {level: [h, w, F]}) -> the stages after
    the post-processing (and box-feature) phase."""
    from object_detection_tracking_b200.effdet import POST_STAGES
    set_inputs(c, cls, box, scale, feats)
    c.eng.run_phases(POST | (BOX_FEAT if feats is not None else 0))
    return {n: c.eng.stage(n) for n in POST_STAGES}


def check(c, cls, box, out, scale=1.0, top_k=None):
    """Candidates and outputs against the oracle; returns (oracle candidates, final count)."""
    from oracle import effdet as oe
    from oracle import tf_ops
    rb, rs, rc, rl = oe.topk_candidates(cls, box, c.cfg, c.fs, top_k=top_k or tf_ops.top_k)
    n = int(out["topk_count"][0])
    assert n == len(rs) == min(c.k, c.total), ("topk_count", n, len(rs))
    np.testing.assert_array_equal(out["topk_classes"][:n], rc)
    np.testing.assert_array_equal(out["topk_levels"][:n], rl)
    assert_bits(out["topk_boxes"][:n], rb, "topk_boxes")
    gs = out["topk_scores"][:n]
    assert ulps(gs, rs).max() <= SCORE_ULPS, ("topk_scores", int(ulps(gs, rs).max()))
    # the NMS visits the candidates in top-k order, the oracle by score: the same order while the scores never increase
    assert np.all(gs[1:] <= gs[:-1])
    fb, fsc, fc, fl = oe.nms_select(out["topk_boxes"][:n], gs, out["topk_classes"][:n], out["topk_levels"][:n], c.cfg,
                                    scale)
    m = int(out["final_count"][0])
    assert m == len(fsc), ("final_count", m, len(fsc))
    assert_bits(out["final_boxes"][:m], fb, "final_boxes")
    assert_bits(out["final_scores"][:m], fsc, "final_scores")
    np.testing.assert_array_equal(out["final_classes"][:m], fc)
    np.testing.assert_array_equal(out["final_levels"][:m], fl)
    assert np.all(out["final_boxes"][m:] == 0) and np.all(out["final_scores"][m:] == 0)
    assert np.all(out["final_classes"][m:] == 0) and np.all(out["final_levels"][m:] == 3)
    return (rb, rs, rc, rl), m


def check_box_feat(c, feats, out):
    import torch
    from oracle import effdet as oe
    m = int(out["final_count"][0])
    ref = oe.box_features({l: torch.from_numpy(np.ascontiguousarray(f.transpose(2, 0, 1))[None]) for l, f in feats.items()},
                          out["final_boxes"][:m], out["final_levels"][:m], c.cfg)
    assert_bits(out["box_feat"][:m], ref, "box_feat")
    assert np.all(out["box_feat"][m:] == 0)


def constant_maps(c):
    """Every level constant per channel (a different constant per level): every bilinear sample inside a level is that
    constant whatever its weights, so the box feature is exact for any box."""
    ch = np.arange(c.F)
    return {l: np.broadcast_to(((l * 37 + ch * 11) % 512 - 256).astype(F32) / F32(64), (h, w, c.F)).astype(F32)
            for l, (h, w) in c.sizes.items()}


def deltas(c, seed=0):
    return ep.exact_deltas(c.cfg, np.random.default_rng(seed))


# ---- top-k ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dense", [False, True])
def test_quantised_ties_across_the_kth_value(ctx, dense):
    """The k-th logit is tied thousands of times: sparse ties (a few in every radix block, the first sixth of the blocks
    supply them) or dense ones (a third of all logits); the selected ties are the lowest flat indices."""
    c = ctx("base")
    rng = np.random.default_rng(1 + dense)
    x = (ep.si.quantised_logits(rng, c.total, c.k) if dense else ep.band_logits(rng, c.total, c.k))
    s = np.sort(x)[::-1]
    assert s[c.k - 1] == s[c.k] and s[0] > s[c.k - 1]
    cls, box = c.split(x), deltas(c, 1)
    check(c, cls, box, run(c, cls, box))


def test_d7_geometry_ties_in_every_radix_block(ctx):
    """D7 at 1536^2: 39.8 M logits over the 1056 radix blocks, each holding ties at the k-th value."""
    c = ctx("d7")
    assert c.total == 441936 * 90
    x = ep.band_logits(np.random.default_rng(3), c.total, c.k)
    chunk = -(-c.total // 1056)
    assert np.all(np.add.reduceat((x == F32(0.75)).astype(np.int64), np.arange(0, c.total, chunk)) > 0)
    cls, box = c.split(x), deltas(c, 3)
    del x
    check(c, cls, box, run(c, cls, box), top_k=ep.fast_top_k)


@pytest.mark.parametrize("k", [1, 64, 65, 4096, 4097, 8192])
def test_topk_sizes(ctx, k):
    """k at and across powers of two (sort size, shared memory, NMS mask words), up to the 8192 maximum."""
    c = ctx("k%d" % k)
    x = ep.si.quantised_logits(np.random.default_rng(k), c.total, k)
    cls, box = c.split(x), deltas(c, k)
    check(c, cls, box, run(c, cls, box))


def test_k_larger_than_the_logit_count(ctx):
    """1 anchor, 1 class at 128^2: 341 logits < k = 5000, so every logit is a candidate; 15 padding columns per row."""
    c = ctx("tiny")
    assert c.total == 341 < c.k
    x = np.random.default_rng(4).standard_normal(c.total).astype(F32)
    cls, box = c.split(x), deltas(c, 4)
    check(c, cls, box, run(c, cls, box))


@pytest.mark.parametrize("k", [0, 8193])
def test_topk_out_of_range_is_refused(k):
    from object_detection_tracking_b200.effdet import EffdetEngine
    from object_detection_tracking_b200.effdet_config import make_effdet_config
    from object_detection_tracking_b200.synth import synth_effdet_weights
    cfg = make_effdet_config("efficientdet-d0", 128, 128, fpn_cell_repeats=1, box_class_repeats=1, max_detection_topk=k)
    with pytest.raises(RuntimeError, match="max_detection_topk"):
        EffdetEngine(cfg, synth_effdet_weights(cfg))


@pytest.mark.parametrize("bits", [8, 16, 24])
@pytest.mark.parametrize("value", [-2.5, 3.75])
def test_logits_sharing_key_prefixes(ctx, bits, value):
    """Every logit agrees with the others in its top 8, 16 or 24 key bits, so the radix passes before the last see one
    bucket; with -2.5 the k-th value is negative."""
    c = ctx("base")
    x = ep.prefix_logits(np.random.default_rng(bits), c.total, value, bits)
    cls, box = c.split(x), deltas(c, bits)
    check(c, cls, box, run(c, cls, box))


def test_signed_zeros_tie_at_the_kth_value(ctx):
    """+0.0 and -0.0 interleaved at the k-th value tie by index alone."""
    c = ctx("base")
    x = ep.signed_zero_logits(np.random.default_rng(6), c.total, 2000)
    cls, box = c.split(x), deltas(c, 6)
    _, m = check(c, cls, box, run(c, cls, box))
    assert m > 0


def test_first_and_last_index_of_every_level(ctx):
    """The first logit of every level and its last one (last cell, last anchor, last class) on top."""
    c = ctx("base")
    x = np.full(c.total, F32(-10), F32)
    ends = [c.offsets[l] for l in range(3, 8)] + [c.offsets[l] - 1 for l in range(4, 8)] + [c.total - 1]
    x[ends] = np.arange(len(ends), 0, -1).astype(F32)
    cls, box = c.split(x), deltas(c, 7)
    (rb, rs, rc, rl), _ = check(c, cls, box, run(c, cls, box))
    assert sorted(rl[:len(ends)].tolist()) == [3, 3, 4, 4, 5, 5, 6, 6, 7, 7]
    assert rc[0] == 1 and rc[5] == c.nc and rc[9] == c.nc     # first of level 3; last of level 3 and of level 7


def test_partial_class_rows(ctx):
    """5 classes x 9 anchors: 45 logits per row of 48; the 3 padding columns hold +1e30 and must never be selected."""
    c = ctx("partial")
    x = ep.si.quantised_logits(np.random.default_rng(8), c.total, c.k)
    cls, box = c.split(x), deltas(c, 8)
    check(c, cls, box, run(c, cls, box))


# ---- scores, NMS -----------------------------------------------------------------------------------------------------
def test_saturated_scores_and_the_threshold(ctx):
    """result_score_thres 0.5: logit 0.0 scores exactly 0.5 and is dropped (the scan stops on !(s > thr)); logits from 17
    up score exactly 1.0 and keep their top-k order."""
    c = ctx("thr")
    rng = np.random.default_rng(9)
    x = np.full(c.total, F32(-30), F32)
    pos = rng.choice(c.total, 260, replace=False)
    x[pos[:200]] = F32(0.0)
    x[pos[200:230]] = rng.choice(np.array([17, 20, 25, 30, 88, 100], F32), 30)
    x[pos[230:]] = rng.integers(1, 200, 30).astype(F32) / F32(64)
    cls, box = c.split(x), deltas(c, 9)
    out = run(c, cls, box)
    (rb, rs, rc, rl), m = check(c, cls, box, out)
    assert np.sum(rs == F32(0.5)) == 200 and np.sum(rs == F32(1)) == 30
    # fewer than max_out candidates score above 0.5, so the scan reaches the ones at exactly 0.5
    assert 0 < m <= 60 < c.m and np.all(out["final_scores"][:m] > F32(0.5))


def test_iou_at_the_threshold_and_one_ulp_above(ctx):
    """Pair 1 overlaps at IoU exactly 0.5 (kept: suppression needs IoU > 0.5), pair 2 one float32 ulp above (suppressed)."""
    c = ctx("iou")
    from oracle import effdet as oe
    a = oe.anchor_boxes(c.cfg, c.fs)
    t = ep.iou_shift(a[0], a[9], ep.IOU_ABOVE)
    assert ep.iou_shift(a[-18], a[-9], F32(0.5)) == (0, 0) and t is not None
    x = np.full(c.total, F32(-30), F32)
    nc = c.nc
    x[c.offsets[7] + 0 * nc + 0] = 5.0             # level 7, cell 0, anchor 0, class 1
    x[c.offsets[7] + 9 * nc + 1] = 4.0             # level 7, cell 1, anchor 0, class 2
    x[c.offsets[3] + 0 * nc + 2] = 3.0             # level 3, cell (0, 0), anchor 0, class 3
    x[c.offsets[3] + 9 * nc + 3] = 2.0             # level 3, cell (0, 1), anchor 0, class 4
    box = {l: np.zeros((h, w, c.na * 4), F32) for l, (h, w) in c.sizes.items()}
    box[3][0, 1, 0:2] = t
    cls = c.split(x)
    out = run(c, cls, box)
    _, m = check(c, cls, box, out)
    assert m == 3 and out["final_classes"][:3].tolist() == [1, 2, 3]


def test_dense_clusters_and_the_output_cap(ctx):
    """Distinct logits over densely overlapping candidates: the cap of 100 hit, reached exactly, and not reached (zero
    padding rows)."""
    from object_detection_tracking_b200.effdet import EffdetEngine
    from object_detection_tracking_b200.synth import synth_effdet_weights
    from oracle import effdet as oe
    import copy
    c = ctx("base")
    x = np.random.default_rng(10).standard_normal(c.total).astype(F32)
    cls, box = c.split(x), deltas(c, 10)
    _, m = check(c, cls, box, run(c, cls, box))
    assert m == c.m
    cand = oe.topk_candidates(cls, box, c.cfg, c.fs)
    free = copy.copy(c.cfg)
    free.result_per_im = 10 ** 6
    n_all = len(oe.nms_select(*cand, free, 1.0)[1])
    assert c.m < n_all < c.k
    for cap in (n_all, n_all + 7):
        d = copy.copy(c)
        d.cfg = copy.copy(c.cfg)
        d.cfg.result_per_im = d.m = cap
        d.eng = EffdetEngine(d.cfg, synth_effdet_weights(d.cfg))
        try:
            _, m = check(d, cls, box, run(d, cls, box))
            assert m == n_all
        finally:
            d.eng.close()


def test_degenerate_boxes(ctx):
    """th / tw of -200 (exp -> 0: zero-area boxes) and of 100 (exp -> inf: infinite sides) among exact boxes; their box
    features (an infinite side samples nothing: zero) on constant maps."""
    c = ctx("base")
    rng = np.random.default_rng(11)
    x = rng.standard_normal(c.total).astype(F32)
    box = deltas(c, 11)
    for l in range(3, 8):
        b = box[l].reshape(-1, 4)
        u = rng.random(len(b))
        b[u < 0.2, 2] = -200.0
        b[(u >= 0.2) & (u < 0.3), 3] = -200.0
        b[(u >= 0.3) & (u < 0.4), 2] = 100.0
        b[(u >= 0.4) & (u < 0.45), 3] = 100.0
    cls, feats = c.split(x), constant_maps(c)
    out = run(c, cls, box, 1.0, feats)
    (rb, _, _, _), m = check(c, cls, box, out)
    fb = out["final_boxes"][:m]
    assert np.any(np.isinf(rb)) and np.any(np.isinf(fb)) and np.any((fb[:, 2] - fb[:, 0]) * (fb[:, 3] - fb[:, 1]) == 0)
    check_box_feat(c, feats, out)


# ---- box features ----------------------------------------------------------------------------------------------------
def test_box_features_of_scaled_detections(ctx):
    """A non-dyadic image_scale: the box feature samples the scaled boxes, as the reference does (wrapper :348-361)."""
    c = ctx("base")
    x = ep.si.quantised_logits(np.random.default_rng(12), c.total, c.k)
    cls, box, feats = c.split(x), deltas(c, 12), constant_maps(c)
    out = run(c, cls, box, 1.37, feats)
    _, m = check(c, cls, box, out, 1.37)
    assert m > 0
    check_box_feat(c, feats, out)


@pytest.mark.parametrize("name", ["base", "tiny"])
def test_box_features_on_chosen_boxes(ctx, name):
    """Boxes written straight into final_*: partly or wholly outside their level, on every level (level 7 is 1 x 2 at
    128 x 256 and a single pixel at 128 x 128, whose 1-pixel axes sample their only pixel), with sample coordinates on
    quarter pixels so that bilinear weights, bins and the 49-bin mean are exact; varied fp16-exact feature values."""
    c = ctx(name)
    n = c.m - 9
    boxes, levels = ep.exact_feature_boxes(np.random.default_rng(13), c.sizes, n)
    feats = {l: ep.feature_values(1, h, w, c.F, salt=l)[0] for l, (h, w) in c.sizes.items()}
    fb = np.zeros((c.m, 4), F32)
    fl = np.full(c.m, 3, np.int32)
    fb[:n], fl[:n] = boxes, levels
    set_inputs(c, None, None, 1.0, feats)
    c.eng.set_stage("final_boxes", fb)
    c.eng.set_stage("final_levels", fl)
    c.eng.set_stage("final_count", np.array([n], np.int32))
    c.eng.run_phases(BOX_FEAT)
    out = {k: c.eng.stage(k) for k in ("final_boxes", "final_levels", "final_count", "box_feat")}
    assert int(out["final_count"][0]) == n
    check_box_feat(c, feats, out)
    if name == "tiny":                             # a 1 x 1 level: every box samples its pixel
        assert np.all(np.any(out["box_feat"][:n] != 0, axis=1)[levels == 7])


# ---- the NMS visit order: sigmoid(expf) must never decrease as the logit grows ---------------------------------------
def test_scores_never_increase_along_the_topk_order(ctx):
    """2^20 consecutive float32 logits around -9.2, 0 and 17, and 2^20 logits evenly over [-20, 20], 8192 per run (the
    rest of the logits far below): topk_scores, in logit-descending order, must never increase, within a run and from
    one run to the next.  A counter-example would let the NMS (top-k order) and the reference (score order) diverge."""
    c = ctx("k8192")
    from oracle import effdet as oe
    k = c.k
    sweeps = []
    for centre in (-9.2, 0.0, 17.0):
        key = int(ep.key_of(np.array([centre], F32))[0])
        sweeps.append(ep.float_of_key(np.arange(key - 2 ** 19, key + 2 ** 19, dtype=np.int64).astype(np.uint32)))
    sweeps.append(np.unique(np.linspace(-20, 20, 2 ** 20).astype(F32)))
    base = {l: np.full((h, w, c.na * c.nc), F32(-3e38), F32) for l, (h, w) in c.sizes.items()}
    set_inputs(c, base, deltas(c, 14))
    for vals in sweeps:
        vals = np.sort(vals)[::-1]
        prev = None
        for s0 in range(0, len(vals), k):
            chunk = vals[s0:s0 + k]
            cls3 = base[3].reshape(-1).copy()
            cls3[:len(chunk)] = chunk
            c.eng.set_stage("cls3", ep.padded(cls3.reshape(base[3].shape), ep.pad16(c.na * c.nc)))
            c.eng.run_phases(POST)
            sc = c.eng.stage("topk_scores")[:len(chunk)]
            ref = oe.sigmoid(chunk)
            assert ulps(sc, ref).max() <= SCORE_ULPS
            bad = np.flatnonzero(sc[1:] > sc[:-1])
            assert len(bad) == 0, ("score increases", chunk[bad[0]], chunk[bad[0] + 1], sc[bad[0]], sc[bad[0] + 1])
            assert prev is None or sc[0] <= prev, ("score increases across runs", prev, sc[0])
            prev = sc[-1]


# ---- graph replay --------------------------------------------------------------------------------------------------
def test_graph_replay_equals_the_eager_phases():
    """run_features (the captured graph) and the eager post-processing + box-feature phases on the stages it left."""
    from object_detection_tracking_b200.effdet import EffdetEngine
    from object_detection_tracking_b200.effdet_config import feat_sizes, make_effdet_config
    from object_detection_tracking_b200.synth import synth_effdet_weights
    cfg = make_effdet_config("efficientdet-d0", 256, 384, fpn_cell_repeats=1, box_class_repeats=1)
    eng = EffdetEngine(cfg, synth_effdet_weights(cfg))
    try:
        rng = np.random.default_rng(15)
        fs = feat_sizes(cfg)
        feats = {l: np.abs(rng.standard_normal((cfg.backbone_channels[l - 3],) + fs[l])).astype(F32) for l in (3, 4, 5)}
        g = eng.run_features(feats, image_scale=1.37)
        m = len(g["final_probs"])
        assert m > 0
        eng.set_stage("final_count", np.zeros(1, np.int32))
        eng.run_phases(POST | BOX_FEAT)
        assert int(eng.stage("final_count")[0]) == m
        for key, st in (("final_boxes", "final_boxes"), ("final_probs", "final_scores"), ("final_labels", "final_classes"),
                        ("levels", "final_levels"), ("fpn_box_feat", "box_feat")):
            got = eng.stage(st)[:m]
            assert ep.same_bits(got, g[key]) if got.dtype == F32 else np.array_equal(got, g[key]), key
    finally:
        eng.close()
