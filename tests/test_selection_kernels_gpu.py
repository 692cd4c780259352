"""The detector's selection kernels, bit for bit, on adversarial inputs: RPN top-k + NMS + level merge (rpn.cu), box-head
post-processing (head.cu), multi-level ROIAlign (roialign.cu).

Each test drives one phase through the stage API on exact inputs (selection_inputs.py; its exactness is checked in
test_selection_inputs_cpu.py) and compares with the oracle's ops (oracle.frcnn / oracle.tf_ops) index-aligned:
counts, labels, boxes, scores and features must be the same bits.  The only tolerance is on exp(): the GPU's expf and
numpy's exp may differ in the last ulps, so probabilities are compared within a few ulps and the NMS / top-k selection of
the head is checked on the GPU's own probabilities and boxes.

Phases: 8 = proposals (rpn_l* -> lvl_*, proposal_*), 16 = ROIAlign of the proposals (p2..p5, proposal_* -> roi_feat),
64 = post-processing (head_logits, proposal_* -> probs, dec_boxes, final_*), 128 = box features (final_*, p2..p5 ->
fpn_box_feat)."""
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

import selection_inputs as si

pytestmark = pytest.mark.gpu

F32 = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RPN_STAGES = ("lvl_count", "lvl_boxes", "lvl_scores", "proposal_count", "proposal_boxes", "proposal_scores")
HEAD_STAGES = ("probs", "dec_boxes", "final_count", "final_labels", "final_boxes", "final_probs")

# small contexts (tiny backbone: only the phases under test matter), created on first use and shared by the module
CONTEXTS = {
    "base": dict(),
    "large": dict(H=512, W=768, B=1),                   # p2 = 128 x 192 x 3 = 73 728 anchors: all 8 cluster slices
    "odd": dict(H=200, W=300, B=1),                     # p2..p4 padded past the cropped ceil(H/stride) extent
    "k1": dict(B=1, rpn_test_post_nms_topk=1),
    "k1000": dict(B=1, rpn_test_post_nms_topk=1000),
    "k1024": dict(B=1, rpn_test_post_nms_topk=1024),
    "minsize": dict(B=1, rpn_min_size=32),
    "multi": dict(multi=True),
    "coco": dict(B=1, num_class=81, rpn_test_post_nms_topk=1000),
    "agnostic": dict(B=1, use_frcnn_class_agnostic=True),
}


class Ctx:
    def __init__(self, H=192, W=256, B=2, multi=False, **over):
        from object_detection_tracking_b200.config import backbone_geometry, make_config
        from object_detection_tracking_b200.engine import Detector
        from object_detection_tracking_b200.synth import synth_weights
        self.cfg = make_config(resnet_num_block=(1, 1, 1, 1), max_size=W, short_edge_size=H, **over)
        self.H, self.W, self.B, self.multi = H, W, B, multi
        self.K, self.R = self.cfg.rpn_test_post_nms_topk, self.cfg.result_per_im
        self.det = Detector(self.cfg, B, H, W, precision="split", use_cuda_graph=False, multi_semantics=multi)
        self.det.load_weights(synth_weights(self.cfg, 7))
        self.lvl_hw = [self.det.stage_shape("rpn_l%d" % l)[0][1:3] for l in range(5)]
        assert self.lvl_hw == [tuple(p) for p in backbone_geometry(H, W, self.cfg)["p"]]
        self.ld = self.det.stage_shape("head_logits")[0][2]

    def stages(self, names):
        return {n: self.det.get_stage(n) for n in names}


@pytest.fixture(scope="module")
def ctx():
    made = {}

    def get(name):
        if name not in made:
            made[name] = Ctx(**CONTEXTS[name])
        return made[name]
    yield get
    for c in made.values():
        c.det.close()


def assert_bits(got, exp, what):
    assert si.same_bits(got, exp), "%s: %s\n  got %s\n  exp %s" % (what, "not bit-identical", np.asarray(got)[:8],
                                                                    np.asarray(exp)[:8])


# ---- RPN (phase 8) ---------------------------------------------------------------------------------------------------
def run_rpn(c, inputs):
    """inputs[b][l] = (cls [fh,fw,3], box [fh,fw,3,4]).  Returns the proposal stages after phase 8."""
    for l in range(5):
        buf = np.zeros(c.det.stage_shape("rpn_l%d" % l)[0], F32)
        for b in range(c.B):
            buf[b] = si.rpn_stage(*inputs[b][l])
        c.det.set_stage("rpn_l%d" % l, buf)
    c.det.run_phases(8)
    return c.stages(RPN_STAGES)


def check_rpn(c, inputs, out):
    """Every level's kept set and the merged proposals against oracle.frcnn, index-aligned and bit for bit.  Returns the
    oracle's per-image (level results, merged boxes, merged scores)."""
    from oracle import frcnn
    K = c.K
    res = []
    for b in range(c.B):
        cnt = out["lvl_count"][b].reshape(5)
        lb = out["lvl_boxes"][b].reshape(5, K, 4)
        ls = out["lvl_scores"][b].reshape(5, K)
        lv = []
        for l in range(5):
            rb, rs = frcnn.level_proposals(c.cfg, l, *inputs[b][l], (c.H, c.W), multi=c.multi)
            lv.append((rb, rs))
            assert int(cnt[l]) == len(rs), ("lvl_count", b, l, int(cnt[l]), len(rs))
            assert_bits(lb[l, :len(rs)], rb, "lvl_boxes b%d l%d" % (b, l))
            assert_bits(ls[l, :len(rs)], rs, "lvl_scores b%d l%d" % (b, l))
        merge = frcnn.merge_level_proposals_multi if c.multi else frcnn.merge_level_proposals
        pb, ps = merge(lv, K)
        pc = int(out["proposal_count"][b].reshape(-1)[0])
        assert pc == len(ps), ("proposal_count", b, pc, len(ps))
        gb = out["proposal_boxes"][b].reshape(K, 4)
        gs = out["proposal_scores"][b].reshape(K)
        assert_bits(gb[:pc], pb, "proposal_boxes b%d" % b)
        assert_bits(gs[:pc], ps, "proposal_scores b%d" % b)
        assert np.all(gb[pc:] == 0) and np.all(gs[pc:] == 0)
        res.append((lv, pb, ps))
    return res


def level_inputs(c, seed, logits):
    """inputs[b][l] with exact deltas and logits(rng, b, l, n) -> [n]; a different pattern per image."""
    inputs = []
    for b in range(c.B):
        per = []
        for l, (fh, fw) in enumerate(c.lvl_hw):
            rng = np.random.default_rng(seed + 1000 * b + l)
            cls = np.asarray(logits(rng, b, l, fh * fw * 3), F32).reshape(fh, fw, 3)
            per.append((cls, si.rpn_deltas(rng, fh, fw)))
        inputs.append(per)
    return inputs


def tie_inputs(c, seed=11):
    return level_inputs(c, seed, lambda rng, b, l, n: si.quantised_logits(rng, n, c.K))


def rpn_tie_outputs(c):
    """Case-1 inputs through phase 8 (also run in a subprocess with single-CTA clusters)."""
    inputs = tie_inputs(c)
    return inputs, run_rpn(c, inputs)


@pytest.mark.parametrize("name", ["base", "large"])
def test_rpn_quantised_logits_tie_across_the_kth_value(ctx, name):
    """Thousands of equal logits straddle the k-th value on every level larger than top-k: the selected ties are the
    lowest anchor indices, across the cluster's slices (all 8 filled on the large frame), in both images of a batch."""
    c = ctx(name)
    inputs, out = rpn_tie_outputs(c)
    res = check_rpn(c, inputs, out)
    for b in range(c.B):
        for l, (fh, fw) in enumerate(c.lvl_hw):
            n = fh * fw * 3
            if n > c.K:                       # the k-th value is tied: a wrong tie order selects other anchors
                x = np.sort(inputs[b][l][0].reshape(-1))[::-1]
                assert x[c.K - 1] == x[c.K] and x[0] > x[c.K - 1]
        assert len(res[b][2]) > 0
    if c.B == 2:
        assert not np.array_equal(inputs[0][0][0], inputs[1][0][0])


def test_rpn_constant_level(ctx):
    """A level of one constant logit: every anchor ties at the k-th value (need_eq == top-k, none above it)."""
    c = ctx("base")
    inputs = level_inputs(c, 21, lambda rng, b, l, n: np.full(n, 0.25, F32) if l < 2 else si.quantised_logits(rng, n, c.K))
    check_rpn(c, inputs, run_rpn(c, inputs))


def test_rpn_levels_smaller_than_topk(ctx):
    """Top-k 1024: p4..p6 have fewer anchors than k, so the upper cluster ranks get empty slices; distinct logits."""
    c = ctx("k1024")
    assert [h * w * 3 < c.K for h, w in c.lvl_hw] == [False, False, True, True, True]
    inputs = level_inputs(c, 31, lambda rng, b, l, n: rng.standard_normal(n).astype(F32))
    check_rpn(c, inputs, run_rpn(c, inputs))


@pytest.mark.parametrize("name", ["k1", "k1000", "k1024"])
def test_rpn_post_nms_topk(ctx, name):
    c = ctx(name)
    inputs = tie_inputs(c, 41)
    res = check_rpn(c, inputs, run_rpn(c, inputs))
    assert len(res[0][2]) == min(c.K, sum(len(s) for _, s in res[0][0]))


def test_rpn_topk_above_1024_is_refused():
    from object_detection_tracking_b200.config import make_config
    from object_detection_tracking_b200.engine import Detector
    cfg = make_config(resnet_num_block=(1, 1, 1, 1), max_size=256, short_edge_size=192, rpn_test_post_nms_topk=1025)
    with pytest.raises(RuntimeError, match="rpn_topk"):
        Detector(cfg, 1, 192, 256, precision="split", use_cuda_graph=False)


def test_rpn_nms_on_dense_overlapping_boxes(ctx):
    """Distinct logits, the highest on a 10 x 10-cell patch of every level, boxes shifted by multiples of 1/8 of a
    quarter anchor side: neighbouring candidates overlap densely, many of them within 0.02 of the 0.7 threshold."""
    from oracle import frcnn, tf_ops
    from oracle.anchors import get_all_anchors
    c = ctx("base")
    inputs = []
    for b in range(c.B):
        per = []
        for l, (fh, fw) in enumerate(c.lvl_hw):
            rng = np.random.default_rng(51 + 1000 * b + l)
            cls = rng.standard_normal((fh, fw, 3)).astype(F32)
            cls[2 + b:12 + b, 3:13] += F32(8.0)
            per.append((cls, si.rpn_deltas(rng, fh, fw, span=2)))
        inputs.append(per)
    res = check_rpn(c, inputs, run_rpn(c, inputs))
    # non-vacuous: the p2 candidates the NMS sees have many overlaps near the threshold, and it suppresses some
    cls, box = inputs[0][0]
    fh, fw = cls.shape[:2]
    dec = frcnn.decode_bbox_target(box, get_all_anchors(4, [32], c.cfg.anchor_ratios, c.cfg.max_size)[:fh, :fw],
                                   c.cfg.bbox_decode_clip).reshape(-1, 4)
    _, idx = tf_ops.top_k(cls.reshape(-1), c.K)
    bx = frcnn.clip_boxes(dec[idx], (c.H, c.W)).astype(np.float64)
    lo, hi = np.maximum(bx[:, None, :2], bx[None, :, :2]), np.minimum(bx[:, None, 2:], bx[None, :, 2:])
    inter = np.prod(np.clip(hi - lo, 0, None), -1)
    area = np.prod(bx[:, 2:] - bx[:, :2], -1)
    iou = inter / (area[:, None] + area[None, :] - inter)
    near = int((np.abs(iou[np.triu_indices(len(bx), 1)] - 0.7) < 0.02).sum())
    assert near >= 50 and len(res[0][0][0][1]) < c.K // 2, (near, len(res[0][0][0][1]))


def test_rpn_everything_filtered_gives_empty_outputs(ctx):
    """Boxes pushed outside the image clip to zero width and are dropped on every level: no proposal, and the following
    ROIAlign, box head and post-processing yield no detection and zeroed outputs."""
    c = ctx("base")
    inputs = level_inputs(c, 61, lambda rng, b, l, n: rng.standard_normal(n).astype(F32))
    for per in inputs:
        for _, box in per:
            box[..., 0] = 100.0                      # x centre far right of the frame: x1 = x2 = W after the clip
    out = run_rpn(c, inputs)
    check_rpn(c, inputs, out)
    assert np.all(out["lvl_count"] == 0) and np.all(out["proposal_count"] == 0)
    c.det.run_phases(16 | 32 | 64 | 128)
    o = c.stages(("final_count", "final_boxes", "final_probs", "final_labels", "roi_feat", "fpn_box_feat"))
    o["roi_feat"] = o["roi_feat"].reshape(-1, 49 * 256)[:c.B * c.K]
    assert np.all(o["final_count"] == 0)
    for k in ("final_boxes", "final_probs", "final_labels", "roi_feat", "fpn_box_feat"):
        assert np.all(o[k] == 0), k


def test_rpn_min_size_empties_a_level(ctx):
    """rpn_min_size = 32: every p2 anchor (48x24, 32x32, 24x48) has a side <= 32 and is dropped; the other levels keep
    theirs."""
    c = ctx("minsize")
    inputs = tie_inputs(c, 71)
    out = run_rpn(c, inputs)
    check_rpn(c, inputs, out)
    cnt = out["lvl_count"][0].reshape(5)
    assert cnt[0] == 0 and np.all(cnt[1:] > 0)


def test_rpn_signed_zero_logits_tie_by_index(ctx):
    """-0.0 and +0.0 logits at the k-th value tie by anchor index, as in tf.nn.top_k: the selected zeros are the lowest
    indices whatever their sign, and their scores keep their sign."""
    c = ctx("base")

    def logits(rng, b, l, n):
        x = np.full(n, -1.0, F32)
        pos = rng.permutation(n)
        npos = min(c.K // 3, n // 4)
        x[pos[:npos]] = 1.0
        zeros = pos[npos:npos + max(n // 4, 1)]
        x[zeros] = np.where(rng.random(len(zeros)) < 0.5, F32(-0.0), F32(0.0))
        return x
    inputs = level_inputs(c, 81, logits)
    res = check_rpn(c, inputs, run_rpn(c, inputs))
    sel = res[0][0][0][1]
    assert np.any(np.signbit(sel) & (sel == 0)) and np.any(~np.signbit(sel) & (sel == 0))


def test_rpn_batch_graph_semantics(ctx):
    """multi_semantics: negative logits rank below the zero padding of the level merge, and zero-area boxes (positive
    scores, pushed outside the frame) are dropped after it, as in oracle.frcnn.forward_multi."""
    c = ctx("multi")

    def logits(rng, b, l, n):
        x = si.quantised_logits(rng, n, c.K) - F32(2.0)          # all negative
        if l == 0:
            x[rng.permutation(n)[:40 + 10 * b]] = F32(1.0) + rng.integers(0, 8, 40 + 10 * b).astype(F32) / F32(8)
        return x
    inputs = level_inputs(c, 91, logits)
    for b in range(c.B):
        cls, box = inputs[b][0]
        hot = np.argwhere(cls > 0)[:12]
        box[hot[:, 0], hot[:, 1], hot[:, 2], 0] = 100.0          # zero width after the clip
    res = check_rpn(c, inputs, run_rpn(c, inputs))
    for b in range(c.B):
        lv, pb, ps = res[b]
        assert np.all(ps >= 0) and len(ps) < sum(len(s) for _, s in lv)
        b0 = lv[0][0]
        assert np.any((b0[:, 2] - b0[:, 0]) * (b0[:, 3] - b0[:, 1]) == 0)


def test_rpn_cluster_matches_single_cta(ctx):
    """The 8-CTA cluster path and single-CTA clusters (B2_RPN_CLUSTER=1, read once per process, so in a subprocess)
    give the same bits on the tie-heavy inputs."""
    code = ("import sys, numpy as np; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
            "import test_selection_kernels_gpu as t\n"
            "out = {}\n"
            "for name in ('base', 'large'):\n"
            "    c = t.Ctx(**t.CONTEXTS[name])\n"
            "    _, o = t.rpn_tie_outputs(c)\n"
            "    out.update({name + '/' + k: v for k, v in o.items()})\n"
            "    c.det.close()\n"
            "np.savez(sys.argv[1], **out)\n") % (ROOT, os.path.join(ROOT, "tests"))
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "single.npz")
        subprocess.run([sys.executable, "-c", code, path], check=True, env=dict(os.environ, B2_RPN_CLUSTER="1"),
                       timeout=300)
        single = dict(np.load(path))
    assert len(single) == 2 * len(RPN_STAGES)
    for name in ("base", "large"):
        c = ctx(name)
        _, o = rpn_tie_outputs(c)
        s = {k: single[name + "/" + k] for k in RPN_STAGES}
        for k in ("lvl_count", "proposal_count", "proposal_boxes", "proposal_scores"):
            assert si.same_bits(o[k].view(F32), s[k].view(F32)), (name, k)
        # per level, the kept entries (the rest of a level's rows is not written)
        for b in range(c.B):
            for l in range(5):
                n = int(o["lvl_count"][b].reshape(5)[l])
                assert n > 0
                for k in ("lvl_boxes", "lvl_scores"):
                    assert si.same_bits(o[k][b, l, :n], s[k][b, l, :n]), (name, k, b, l)


# ---- box-head post-processing (phase 64) -----------------------------------------------------------------------------
def run_head(c, logits, boxes, counts):
    """logits [B, K, ld], proposal boxes [B, K, 4], counts [B] -> the post-processing stages."""
    c.det.set_stage("head_logits", logits[..., None])
    c.det.set_stage("proposal_boxes", boxes[..., None])
    c.det.set_stage("proposal_count", np.asarray(counts, np.int32).reshape(c.B, 1, 1, 1))
    c.det.run_phases(64)
    return c.stages(HEAD_STAGES)


def check_head(c, logits, boxes, counts, out, dec_atol=None):
    """probs within a few ulps of the oracle's softmax (the GPU sums the exponentials in order, numpy pairwise);
    dec_boxes bit-exact, or within dec_atol px where expf of a size delta enters; the per-class NMS + final top-k
    bit-exact against oracle.frcnn.fastrcnn_predictions on the GPU's own probs / dec_boxes.  Returns the per-image
    (pred_indices, probs) of that selection."""
    from oracle import frcnn
    nc, nc1, R = c.cfg.num_class, c.cfg.num_class - 1, c.R
    sel = []
    for b in range(c.B):
        n = int(counts[b])
        cls = logits[b, :n, :nc]
        if c.cfg.use_frcnn_class_agnostic:
            bl = np.tile(logits[b, :n, None, nc:nc + 4], (1, nc1, 1))
        else:
            bl = logits[b, :n, nc:nc + 4 * nc].reshape(n, nc, 4)[:, 1:]
        dec, probs, pred, fprobs = frcnn.head_postprocess(cls, bl, boxes[b, :n], (c.H, c.W), c.cfg)
        gp = out["probs"][b, :n, :, 0]
        gd = out["dec_boxes"][b, :n]
        np.testing.assert_array_max_ulp(gp, probs, maxulp=16)
        if dec_atol is not None:
            assert np.abs(gd - dec).max() <= dec_atol, np.abs(gd - dec).max()
        else:
            assert_bits(gd, dec, "dec_boxes b%d" % b)
        gpred, gfp = frcnn.fastrcnn_predictions(gd, gp, c.cfg)
        fc = int(out["final_count"][b].reshape(-1)[0])
        assert fc == len(gpred), ("final_count", b, fc, len(gpred))
        np.testing.assert_array_equal(out["final_labels"][b].reshape(R)[:fc], gpred[:, 1] + 1)
        assert_bits(out["final_boxes"][b].reshape(R, 4)[:fc], gd[gpred[:, 0], gpred[:, 1]], "final_boxes b%d" % b)
        assert_bits(out["final_probs"][b].reshape(R)[:fc], gfp, "final_probs b%d" % b)
        for k in ("final_boxes", "final_probs", "final_labels"):
            assert np.all(out[k][b].reshape(R, -1)[fc:] == 0), k
        # the oracle's own probabilities select the same detections
        assert len(pred) == fc and np.array_equal(pred, gpred)
        sel.append((gpred, gfp))
    return sel


def head_inputs(c, n_rois, cls_fn, box_fn):
    """head_logits [B, K, ld] with class logits cls_fn(b, i) and zero box deltas, proposal boxes box_fn(b) [n_rois, 4]."""
    logits = np.zeros((c.B, c.K, c.ld), F32)
    boxes = np.zeros((c.B, c.K, 4), F32)
    for b in range(c.B):
        boxes[b, :n_rois] = box_fn(b)
        for i in range(n_rois):
            logits[b, i] = si.head_logits_row(c.cfg.num_class, cls_fn(b, i), np.zeros(4 * c.cfg.num_class), c.ld,
                                              c.cfg.use_frcnn_class_agnostic)
    return logits, boxes


def pair_grid(n_pairs, cols=15, step=16, size=12, x0=2, y0=2):
    """n_pairs pairs of size x size boxes on a grid; the second of a pair is the first shifted 1 px right (IoU 0.85)."""
    out = []
    for p in range(n_pairs):
        x, y = x0 + step * (p % cols), y0 + step * (p // cols)
        out += [[x, y, x + size, y + size], [x + 1, y, x + 1 + size, y + size]]
    return np.asarray(out, F32)


def test_head_identical_rows_tie_by_class_then_box(ctx):
    """Every ROI has the same logits: within a class all probabilities tie (NMS keeps the lowest ROI of each overlapping
    pair), and across classes the final top-k ties go by (class, box) ascending."""
    c = ctx("base")
    nc = c.cfg.num_class
    rows = [np.r_[0.0, np.ones(nc - 1)].astype(F32),
            np.r_[0.0, np.resize([1.0, 0.5, 0.25], nc - 1)].astype(F32)]
    logits, boxes = head_inputs(c, c.K, lambda b, i: rows[b], lambda b: pair_grid(c.K // 2))
    counts = [c.K] * c.B
    sel = check_head(c, logits, boxes, counts, run_head(c, logits, boxes, counts))
    pred = sel[0][0]
    assert len(pred) == c.R and np.all(pred[:, 1] == 0) and np.array_equal(pred[:, 0], np.arange(0, 2 * c.R, 2))


def test_head_per_class_and_final_caps(ctx):
    """Non-overlapping boxes: one class keeps more than result_per_im survivors (capped per class) and many classes
    together exceed result_per_im (capped in the final top-k)."""
    c = ctx("base")
    nc = c.cfg.num_class
    rng = np.random.default_rng(3)
    g = np.asarray([[12 * (i % 20), 12 * (i // 20), 12 * (i % 20) + 12, 12 * (i // 20) + 12] for i in range(c.K)], F32)
    cls = rng.standard_normal((c.B, c.K, nc)).astype(F32)
    cls[:, :, 1] += 6.0
    logits, boxes = head_inputs(c, c.K, lambda b, i: cls[b, i], lambda b: g)
    counts = [c.K] * c.B
    out = run_head(c, logits, boxes, counts)
    sel = check_head(c, logits, boxes, counts, out)
    pred = sel[0][0]
    assert len(pred) == c.R and np.all(pred[:, 1] == 0)       # class 1 alone fills the result (capped at 100 of 300)
    probs = out["probs"][0, :, 1:, 0]
    assert int((probs > c.cfg.result_score_thres).sum()) > 5 * c.R


def test_head_coco_81_classes_1000_rois(ctx):
    c = ctx("coco")
    rng = np.random.default_rng(4)
    nc = c.cfg.num_class
    xy = rng.integers(0, 200, (c.K, 2))
    wh = rng.integers(4, 64, (c.K, 2))
    bx = np.concatenate([xy, xy + wh], 1).astype(F32)
    cls = (rng.standard_normal((c.K, nc)) * 2).astype(F32)
    logits, boxes = head_inputs(c, c.K, lambda b, i: cls[i], lambda b: bx)
    sel = check_head(c, logits, boxes, [c.K], run_head(c, logits, boxes, [c.K]))
    assert len(sel[0][0]) == c.R and len(np.unique(sel[0][0][:, 1])) > 20


def test_head_iou_exactly_at_threshold_is_kept(ctx):
    """IoU == f32(0.5) does not suppress; the next float32 overlap above it does."""
    c = ctx("base")
    nc = c.cfg.num_class
    (a0, b0), (a1, b1) = si.iou_threshold_pairs()
    bx = np.stack([a0, b0, a1, b1])

    def row(b, i):
        r = np.full(nc, -20.0, F32)
        r[0], r[1] = 0.0, (3.0, 2.0, 3.0, 2.0)[i]
        return r
    logits, boxes = head_inputs(c, 4, row, lambda b: bx)
    counts = [4] * c.B
    sel = check_head(c, logits, boxes, counts, run_head(c, logits, boxes, counts))
    assert sorted(sel[0][0][:, 0].tolist()) == [0, 1, 2]


def test_head_degenerate_boxes(ctx):
    """Zero-width / zero-height boxes (as given, or after the clip to the frame) have IoU 0 with everything: they neither
    suppress nor are suppressed."""
    c = ctx("base")
    rng = np.random.default_rng(6)
    base = pair_grid(20)
    deg = base.copy()
    deg[0::4, 2] = deg[0::4, 0]                       # zero width
    deg[1::4, 3] = deg[1::4, 1]                       # zero height
    deg[2::4, 0] += 400.0                             # outside the frame: x1 = x2 = W after the clip
    deg[2::4, 2] += 400.0
    bx = np.concatenate([base, deg])
    n = len(bx)
    cls = rng.standard_normal((n, c.cfg.num_class)).astype(F32)
    logits, boxes = head_inputs(c, n, lambda b, i: cls[i], lambda b: bx)
    counts = [n] * c.B
    out = run_head(c, logits, boxes, counts)
    check_head(c, logits, boxes, counts, out)
    d = out["dec_boxes"][0, 40:n]
    assert np.sum((d[..., 2] - d[..., 0]) * (d[..., 3] - d[..., 1]) == 0) >= 30 * (c.cfg.num_class - 1)


def test_head_rows_beyond_the_count_have_no_effect(ctx):
    """NaN / 1e30 logits and boxes in the rows beyond roi_count change nothing; an image with roi_count 0 next to a full
    one yields no detection."""
    c = ctx("base")
    rng = np.random.default_rng(7)
    nc = c.cfg.num_class
    xy = rng.integers(0, 180, (c.K, 2))
    bx = np.concatenate([xy, xy + rng.integers(4, 60, (c.K, 2))], 1).astype(F32)
    cls = rng.standard_normal((c.B, c.K, nc)).astype(F32) * 2
    logits, boxes = head_inputs(c, c.K, lambda b, i: cls[b, i], lambda b: bx)
    for counts in ([37, c.K], [0, c.K], [c.K, 0]):
        clean = run_head(c, logits, boxes, counts)
        check_head(c, logits, boxes, counts, clean)
        dirty_l, dirty_b = logits.copy(), boxes.copy()
        for b in range(c.B):
            n = counts[b]
            dirty_l[b, n:] = np.where(rng.random(dirty_l[b, n:].shape) < 0.5, np.nan, 1e30)
            dirty_b[b, n:] = np.where(rng.random(dirty_b[b, n:].shape) < 0.5, np.nan, -1e30)
        dirty = run_head(c, dirty_l, dirty_b, counts)
        for k in ("final_count", "final_labels", "final_boxes", "final_probs"):
            assert si.same_bits(dirty[k].view(F32), clean[k].view(F32)), (counts, k)
        for b in range(c.B):
            if counts[b] == 0:
                assert int(clean["final_count"][b].reshape(-1)[0]) == 0
            else:
                assert int(clean["final_count"][b].reshape(-1)[0]) > 0


def test_head_class_agnostic_regression(ctx):
    """use_frcnn_class_agnostic (versions 4-6): one box regression shared by every class."""
    c = ctx("agnostic")
    rng = np.random.default_rng(8)
    nc = c.cfg.num_class
    assert c.ld >= nc + 4
    xy = rng.integers(0, 180, (c.K, 2))
    bx = np.concatenate([xy, xy + rng.integers(8, 60, (c.K, 2))], 1).astype(F32)
    logits = np.zeros((1, c.K, c.ld), F32)
    logits[0, :, :nc] = rng.standard_normal((c.K, nc)) * 2
    logits[0, :, nc:nc + 4] = rng.integers(-4, 5, (c.K, 4)) / F32(8)     # tx, ty (/10) and tw, th (/5): expf ulps
    logits[0, :, nc + 4:] = np.nan                                       # no per-class box columns are read
    out = run_head(c, logits, bx[None], [c.K])
    # expf of the size deltas: a few ulps at the frame's coordinate scale
    check_head(c, np.nan_to_num(logits), bx[None], [c.K], out, dec_atol=4 * float(np.spacing(F32(c.W))))
    d = out["dec_boxes"][0]
    assert np.all(d == d[:, :1])                      # the same box for every class


def test_head_all_below_score_threshold(ctx):
    c = ctx("base")
    nc = c.cfg.num_class
    logits, boxes = head_inputs(c, c.K, lambda b, i: np.r_[30.0, np.zeros(nc - 1)].astype(F32),
                                lambda b: pair_grid(c.K // 2))
    counts = [c.K] * c.B
    out = run_head(c, logits, boxes, counts)
    check_head(c, logits, boxes, counts, out)
    assert np.all(out["final_count"] == 0) and np.all(out["final_boxes"] == 0) and np.all(out["final_labels"] == 0)


def test_head_saturated_size_deltas(ctx):
    """tw, th above the decode clip log(1333/16): labels and counts exact, boxes within a few ulps of the oracle."""
    c = ctx("base")
    rng = np.random.default_rng(9)
    nc = c.cfg.num_class
    xy = rng.integers(20, 160, (c.K, 2))
    bx = np.concatenate([xy, xy + rng.integers(4, 20, (c.K, 2))], 1).astype(F32)
    logits = np.zeros((c.B, c.K, c.ld), F32)
    logits[:, :, :nc] = rng.standard_normal((c.B, c.K, nc)) * 2
    d = rng.integers(-4, 5, (c.B, c.K, nc, 4)).astype(F32) / F32(8)
    d[..., 2:] = np.where(rng.random((c.B, c.K, nc, 2)) < 0.5, F32(50.0), F32(-0.25))
    logits[:, :, nc:nc + 4 * nc] = d.reshape(c.B, c.K, 4 * nc)
    counts = [c.K] * c.B
    boxes = np.broadcast_to(bx, (c.B, c.K, 4)).copy()
    out = run_head(c, logits, boxes, counts)
    # exp(clip) boxes reach ~1300 px before the clip: a few ulps at that scale
    check_head(c, logits, boxes, counts, out, dec_atol=4 * float(np.spacing(F32(2048))))


# ---- ROIAlign (phases 16 and 128) -----------------------------------------------------------------------------------
def set_features(c, salt=0):
    """p2..p5 with fp16-exact values over the cropped extent and SENTINEL in the padded tail.  Returns the oracle's
    per-image cropped levels [C, h, w]."""
    feats = [[] for _ in range(c.B)]
    for l in range(4):
        shape = c.det.stage_shape("p%d" % (l + 2))[0]
        h, w = c.lvl_hw[l]
        s = si.feature_stage(c.B, shape[1:3], (h, w), shape[3], salt + l)
        c.det.set_stage("p%d" % (l + 2), s)
        for b in range(c.B):
            feats[b].append(np.ascontiguousarray(s[b, :h, :w].transpose(2, 0, 1)))
    return feats


def check_roi_feat(c, feats, boxes, counts):
    """Phase 16 on the given proposals: roi_feat == the oracle's multilevel_roi_align through the plane split, rows
    beyond the count exactly zero.  Returns the oracle's levels per image."""
    from oracle import frcnn
    c.det.set_stage("proposal_boxes", boxes[..., None])
    c.det.set_stage("proposal_count", np.asarray(counts, np.int32).reshape(c.B, 1, 1, 1))
    c.det.run_phases(16)
    rf = c.det.get_stage("roi_feat").reshape(-1, 7, 7, 256)
    lv = []
    for b in range(c.B):
        n = int(counts[b])
        exp, lvl = frcnn.multilevel_roi_align(feats[b], boxes[b, :n], 7, c.cfg.anchor_strides)
        got = rf[b * c.K:b * c.K + n].transpose(0, 3, 1, 2)
        assert_bits(got, si.planes_value(exp), "roi_feat b%d" % b)
        assert np.all(rf[b * c.K + n:(b + 1) * c.K] == 0)
        lv.append(lvl)
    return lv


def check_box_feat(c, feats, boxes, counts):
    """Phase 128 on the given final boxes: fpn_box_feat (float32) == the oracle's multilevel_roi_align bit for bit."""
    from oracle import frcnn
    R = c.R
    fb = np.zeros((c.B, R, 4), F32)
    for b in range(c.B):
        fb[b] = boxes[b, :R]
    c.det.set_stage("final_boxes", fb[..., None])
    c.det.set_stage("final_count", np.asarray(counts, np.int32).reshape(c.B, 1, 1, 1))
    c.det.run_phases(128)
    bf = c.det.get_stage("fpn_box_feat")
    for b in range(c.B):
        n = int(counts[b])
        exp, _ = frcnn.multilevel_roi_align(feats[b], fb[b, :n], 7, c.cfg.anchor_strides)
        assert_bits(bf[b * R:b * R + n], exp, "fpn_box_feat b%d" % b)
        assert np.all(bf[b * R + n:(b + 1) * R] == 0)


def level_boundary_boxes():
    """Integer-sided boxes with sqrt(area) at 56, 112, 224, 448 and areas one or two px^2 either side."""
    out = []
    for s in (56, 112, 224, 448):
        for area in (s * s - 2, s * s - 1, s * s, s * s + 1, s * s + 2):
            for w in range(int(s * 0.8), int(s * 1.25) + 1):
                if area % w == 0 and int(s * 0.8) <= area // w <= int(s * 1.25) + 1:
                    out.append((w, area // w))
                    if sum(1 for a, b in out if a * b == area) >= 3:
                        break
    return out


def test_roialign_level_boundaries(ctx):
    c = ctx("large")
    sides = level_boundary_boxes()
    assert len(sides) <= c.K
    boxes = np.zeros((1, c.K, 4), F32)
    for i, (w, h) in enumerate(sides):
        x, y = 7 + (i * 37) % max(1, c.W - w - 14), 3 + (i * 23) % max(1, c.H - min(h, c.H - 6) - 6)
        boxes[0, i] = (x, y, x + w, y + h)
    feats = set_features(c, salt=1)
    lvl = check_roi_feat(c, feats, boxes, [len(sides)])[0]
    # the oracle's level is the float64 one: these boxes sit on both sides of every boundary
    a = np.array([w * h for w, h in sides], np.float64)
    exp = np.clip(np.floor(4 + np.log2(np.sqrt(a) / 224 + 1e-6)), 2, 5).astype(int)
    np.testing.assert_array_equal(lvl, exp)
    assert set(exp.tolist()) == {2, 3, 4, 5}
    check_box_feat(c, feats, boxes, [min(len(sides), c.R)])


def _samples(c0, c1, dim, crop=14):
    """The float32 sample coordinates of oracle.frcnn.roi_align / tf_ops.crop_and_resize along one axis."""
    f = F32
    sp = f(f(c1 - c0) / f(crop))
    n0 = f(f(f(c0 + f(sp / f(2))) - f(0.5)) / f(dim - 1))
    nl = f(f(sp * f(crop - 1)) / f(dim - 1))
    n1 = f(n0 + nl)
    sc = f(f(f(n1 - n0) * f(dim - 1)) / f(crop - 1))
    return f(n0 * f(dim - 1)) + np.arange(crop, dtype=f) * sc


def test_roialign_edges_outside_and_degenerate_boxes(ctx):
    """Boxes partly and wholly outside the level (extrapolation 0), boxes whose last sample lands exactly on dim - 1,
    zero-width / zero-height and 1-px boxes."""
    c = ctx("base")
    rng = np.random.default_rng(12)
    H, W = c.H, c.W
    bx = [[-30, -20, 40, 50], [W - 40, H - 30, W + 60, H + 20], [-80, 10, -10, 60], [W + 10, 5, W + 90, 70],
          [10, -90, 70, -5], [20, 30, 20, 80], [20, 30, 90, 30], [50, 60, 51, 61], [0, 0, 1, 1], [W - 1, H - 1, W, H],
          [0, 0, W, H], [-W, -H, 2 * W, 2 * H]]
    # p2 (stride 4, dim = level width): right edges whose last sample is exactly dim - 1
    dim = c.lvl_hw[0][1]
    hits = 0
    for c1 in np.arange(dim - 2, dim + 2, 0.125, dtype=F32):
        c0 = F32(c1 - 28)
        if _samples(c0, c1, dim)[-1] == F32(dim - 1):
            bx.append([c0 * 4, 40, c1 * 4, 80])
            hits += 1
    assert hits >= 1
    for _ in range(40):
        x0, y0 = rng.uniform(-40, W), rng.uniform(-40, H)
        bx.append([x0, y0, x0 + rng.uniform(0, 160), y0 + rng.uniform(0, 160)])
    bx = np.round(np.asarray(bx, np.float64) * 8) / 8
    boxes = np.zeros((c.B, c.K, 4), F32)
    for b in range(c.B):
        boxes[b, :len(bx)] = bx[rng.permutation(len(bx))] if b else bx
    feats = set_features(c, salt=2)
    counts = [len(bx)] * c.B
    check_roi_feat(c, feats, boxes, counts)
    check_box_feat(c, feats, boxes, [min(len(bx), c.R)] * c.B)


def test_roialign_odd_geometry_never_reads_the_pitch_tail(ctx):
    """200 x 300: p2..p4 are padded beyond the cropped ceil(H/stride) extent; the tail holds SENTINEL, which must never
    reach an output."""
    c = ctx("odd")
    shapes = [c.det.stage_shape("p%d" % (l + 2))[0][1:3] for l in range(3)]
    assert all(s != hw for s, hw in zip(shapes, c.lvl_hw[:3]))
    rng = np.random.default_rng(13)
    bx = [[c.W - 30, c.H - 30, c.W + 30, c.H + 30], [0, c.H - 8, c.W, c.H], [c.W - 8, 0, c.W, c.H], [0, 0, c.W, c.H]]
    for _ in range(60):
        x0, y0 = rng.uniform(c.W * 0.5, c.W), rng.uniform(c.H * 0.5, c.H)
        bx.append([x0, y0, x0 + rng.uniform(1, 300), y0 + rng.uniform(1, 300)])
    boxes = np.zeros((1, c.K, 4), F32)
    boxes[0, :len(bx)] = np.round(np.asarray(bx) * 4) / 4
    feats = set_features(c, salt=3)
    check_roi_feat(c, feats, boxes, [len(bx)])
    assert np.abs(c.det.get_stage("roi_feat").reshape(-1, 49 * 256)[:c.K]).max() < 8
    check_box_feat(c, feats, boxes, [len(bx)])
    assert np.abs(c.det.get_stage("fpn_box_feat")).max() < 8


def test_roialign_garbage_rows_beyond_the_count_are_zero(ctx):
    c = ctx("base")
    rng = np.random.default_rng(14)
    boxes = np.zeros((c.B, c.K, 4), F32)
    for b in range(c.B):
        xy = rng.uniform(0, 180, (c.K, 2))
        boxes[b] = np.round(np.concatenate([xy, xy + rng.uniform(2, 120, (c.K, 2))], 1) * 4) / 4
    counts = [23, 0]
    for b in range(c.B):
        boxes[b, counts[b]:] = np.where(rng.random((c.K - counts[b], 4)) < 0.5, F32(1e30), F32(-3e29))
        boxes[b, counts[b]:counts[b] + 4] = [[10, 10, 90, 90]] * 4            # plausible boxes right after the count
    feats = set_features(c, salt=4)
    check_roi_feat(c, feats, boxes, counts)
    check_box_feat(c, feats, boxes, counts)
