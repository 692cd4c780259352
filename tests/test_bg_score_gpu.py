"""--use_bg_score on the GPU (models.py:1263-1270): the background filter ahead of the box head's class NMS and in the
small-object branch's final selection.

* Stage level (phase 64 on exact inputs, as test_selection_kernels_gpu.py): bg_rank, final_count, labels, probabilities and
  boxes bit-exact with bg_score_oracle on the engine's own probabilities and decoded boxes -- BG / class ties, every row
  background, none, background rows first (every box moves), garbage beyond the count, 81 classes x 1000 ROIs, the
  class-agnostic head, batch 2 with single-image semantics.
* End to end with a background bias that drops about half of the ROIs: detections, fpn_box_feat and final_masks against
  the oracle under the bars of test_baseline_configs_gpu.py.
* The small-object branch's so_final_* with the filter over its rebuilt logits.
* No effect on the batch graph and the use_cpu_nms outputs; the flag-off plan launches what the default one does."""
import numpy as np
import pytest

import bg_score_oracle as bo
import selection_inputs as si
from test_baseline_configs_gpu import (assert_final, assert_stagewise, exact_margins, final_margins, log_margins, rel,
                                       stagewise)
from test_selection_kernels_gpu import HEAD_STAGES, Ctx, assert_bits, head_inputs, pair_grid

pytestmark = pytest.mark.gpu

F32 = np.float32
CONTEXTS = {
    "base": dict(),                                                  # batch 2, single-image semantics
    "coco": dict(B=1, num_class=81, rpn_test_post_nms_topk=1000),
    "agnostic": dict(B=1, use_frcnn_class_agnostic=True),
}
SMALL = dict(resnet_num_block=(1, 1, 2, 1), max_size=384, short_edge_size=256)


@pytest.fixture(scope="module")
def ctx():
    made = {}

    def get(name):
        if name not in made:
            made[name] = Ctx(use_bg_score=True, **CONTEXTS[name])
        return made[name]
    yield get
    for c in made.values():
        c.det.close()


def run_head(c, logits, boxes, counts):
    c.det.set_stage("head_logits", logits[..., None])
    c.det.set_stage("proposal_boxes", boxes[..., None])
    c.det.set_stage("proposal_count", np.asarray(counts, np.int32).reshape(c.B, 1, 1, 1))
    c.det.run_phases(64)
    return {n: c.det.get_stage(n) for n in HEAD_STAGES + ("bg_rank",)}


def check(c, logits, counts, out):
    """bg_rank and the final outputs bit-exact with the oracle on the GPU's own probs / dec_boxes; the oracle's softmax of
    the logits drops the same rows.  Returns per image (dropped rows, detections, kept ROI of each detection, its rank)."""
    from oracle import frcnn
    nc, K, R = c.cfg.num_class, c.K, c.R
    res = []
    for b in range(c.B):
        n = int(counts[b])
        gp = out["probs"][b, :n, :, 0]
        gd = out["dec_boxes"][b, :n]
        rank = out["bg_rank"][b].reshape(K)
        want = np.full(K, -1, np.int32)
        want[:n] = bo.bg_rank(gp)
        np.testing.assert_array_equal(rank, want, err_msg="bg_rank b%d" % b)
        np.testing.assert_array_equal(bo.bg_rank(frcnn.softmax(logits[b, :n, :nc])), want[:n])
        fb, fl, fp = bo.final_outputs(gd, gp, c.cfg)
        lb, ll, lp = bo.literal(gd, gp, c.cfg)
        assert si.same_bits(fb, lb) and np.array_equal(fl, ll) and si.same_bits(fp, lp)
        fc = int(out["final_count"][b].reshape(-1)[0])
        assert fc == len(fl), ("final_count", b, fc, len(fl))
        np.testing.assert_array_equal(out["final_labels"][b].reshape(R)[:fc], fl)
        assert_bits(out["final_boxes"][b].reshape(R, 4)[:fc], fb, "final_boxes b%d" % b)
        assert_bits(out["final_probs"][b].reshape(R)[:fc], fp, "final_probs b%d" % b)
        for k in ("final_boxes", "final_probs", "final_labels"):
            assert np.all(out[k][b].reshape(R, -1)[fc:] == 0), k
        pred, _ = bo.fastrcnn_predictions(gd, gp, c.cfg)
        kept = np.nonzero(want[:n] >= 0)[0]
        res.append(dict(dropped=int(n - len(kept)), final=fc, roi=kept[pred[:, 0]] if fc else pred[:, 0],
                        rank=pred[:, 0], dec=gd, cls=pred[:, 1]))
    return res


def test_ties_and_background_rows_first(ctx):
    """Image 0: every other row's background logit equals its best class (dropped: ties go to column 0).  Image 1: the
    first half of the rows are background, so every detection's box is a background ROI's (the reference's gather)."""
    c = ctx("base")
    nc = c.cfg.num_class
    rng = np.random.default_rng(21)
    cls = (rng.integers(-4, 5, (c.B, c.K, nc)) / 2).astype(F32)
    cls[0, ::2, 0] = cls[0, ::2, 1:].max(1)
    cls[1, :c.K // 2, 0] = 20.0
    cls[1, c.K // 2:, 0] = -20.0
    logits, boxes = head_inputs(c, c.K, lambda b, i: cls[b, i], lambda b: pair_grid(c.K // 2))
    counts = [c.K] * c.B
    r = check(c, logits, counts, run_head(c, logits, boxes, counts))
    assert r[0]["dropped"] >= c.K // 2 and r[0]["final"] > 0
    assert r[1]["dropped"] == c.K // 2 and r[1]["final"] > 0
    assert np.all(r[1]["rank"] < c.K // 2) and np.all(r[1]["roi"] >= c.K // 2)
    own = r[1]["dec"][r[1]["roi"], r[1]["cls"]]
    taken = r[1]["dec"][r[1]["rank"], r[1]["cls"]]
    assert np.all(np.any(own != taken, axis=1))                   # every box is another ROI's


def test_all_and_no_rows_background(ctx):
    c = ctx("base")
    nc = c.cfg.num_class
    rng = np.random.default_rng(22)
    cls = rng.standard_normal((c.B, c.K, nc)).astype(F32)
    cls[0, :, 0] = 30.0
    cls[1, :, 0] = -30.0
    logits, boxes = head_inputs(c, c.K, lambda b, i: cls[b, i], lambda b: pair_grid(c.K // 2))
    counts = [c.K] * c.B
    out = run_head(c, logits, boxes, counts)
    r = check(c, logits, counts, out)
    assert r[0]["dropped"] == c.K and r[0]["final"] == 0 and np.all(out["bg_rank"][0] == -1)
    assert r[1]["dropped"] == 0 and r[1]["final"] > 0
    np.testing.assert_array_equal(out["bg_rank"][1].reshape(-1), np.arange(c.K))


def test_rows_beyond_the_count_have_no_effect(ctx):
    c = ctx("base")
    rng = np.random.default_rng(23)
    nc = c.cfg.num_class
    xy = rng.integers(0, 180, (c.K, 2))
    bx = np.concatenate([xy, xy + rng.integers(4, 60, (c.K, 2))], 1).astype(F32)
    cls = rng.standard_normal((c.B, c.K, nc)).astype(F32) * 2
    cls[:, :, 0] += 1.5
    logits, boxes = head_inputs(c, c.K, lambda b, i: cls[b, i], lambda b: bx)
    for counts in ([37, c.K], [0, c.K], [c.K, 0]):
        clean = run_head(c, logits, boxes, counts)
        r = check(c, logits, counts, clean)
        assert any(0 < x["dropped"] < n for x, n in zip(r, counts))
        dirty_l, dirty_b = logits.copy(), boxes.copy()
        for b in range(c.B):
            n = counts[b]
            dirty_l[b, n:] = np.where(rng.random(dirty_l[b, n:].shape) < 0.5, np.nan, 1e30)
            dirty_b[b, n:] = np.where(rng.random(dirty_b[b, n:].shape) < 0.5, np.nan, -1e30)
        dirty = run_head(c, dirty_l, dirty_b, counts)
        for k in ("bg_rank", "final_count", "final_labels", "final_boxes", "final_probs"):
            assert si.same_bits(dirty[k].view(F32), clean[k].view(F32)), (counts, k)


def test_coco_81_classes_1000_rois(ctx):
    c = ctx("coco")
    rng = np.random.default_rng(24)
    nc = c.cfg.num_class
    xy = rng.integers(0, 200, (c.K, 2))
    bx = np.concatenate([xy, xy + rng.integers(4, 64, (c.K, 2))], 1).astype(F32)
    cls = (rng.standard_normal((c.K, nc)) * 2).astype(F32)
    cls[:, 0] += 3.0
    logits, boxes = head_inputs(c, c.K, lambda b, i: cls[i], lambda b: bx)
    r = check(c, logits, [c.K], run_head(c, logits, boxes, [c.K]))
    assert 100 < r[0]["dropped"] < 900 and r[0]["final"] > 0


def test_class_agnostic_head(ctx):
    c = ctx("agnostic")
    rng = np.random.default_rng(25)
    nc = c.cfg.num_class
    xy = rng.integers(0, 180, (c.K, 2))
    bx = np.concatenate([xy, xy + rng.integers(8, 60, (c.K, 2))], 1).astype(F32)
    logits = np.zeros((1, c.K, c.ld), F32)
    logits[0, :, :nc] = rng.standard_normal((c.K, nc)) * 2
    logits[0, :, 0] += 2.0
    logits[0, :, nc:nc + 4] = rng.integers(-4, 5, (c.K, 4)) / F32(8)
    r = check(c, logits, [c.K], run_head(c, logits, bx[None], [c.K]))
    assert 0 < r[0]["dropped"] < c.K and r[0]["final"] > 0


# ---- end to end --------------------------------------------------------------------------------------------------------
def _shifted_weights(cfg, frame, seed):
    """Synthetic weights with the background bias moved so that about half of this frame's ROIs are background, and the
    oracle's forward (stages) under use_bg_score with them."""
    from object_detection_tracking_b200.synth import synth_weights
    from oracle import frcnn
    W0 = synth_weights(cfg, seed)
    Wt = bo.with_background_shift(W0, bo.background_shift(frcnn.forward(cfg, W0, frame, stages=True)["cls_logits"]))
    with bo.use_bg_score():
        o = frcnn.forward(cfg, Wt, frame)
        with frcnn.exact():
            o64 = frcnn.forward(cfg, Wt, frame, stages=False)
    return Wt, o, o64


@pytest.mark.parametrize("seed", [5, 6])
def test_end_to_end_with_masks(seed):
    from object_detection_tracking_b200.config import make_config
    from object_detection_tracking_b200.engine import Detector
    from object_detection_tracking_b200.synth import synth_frame
    H, W = 256, 384
    cfg = make_config(use_bg_score=True, add_mask=True, **SMALL)
    frame = synth_frame(H, W, seed=seed).astype(np.float32)
    Wt, o, o64 = _shifted_weights(cfg, frame, 77)
    K = len(o["probs"])
    dropped = int((bo.bg_rank(o["probs"]) < 0).sum())
    assert 0.25 * K < dropped < 0.75 * K, (dropped, K)
    # no near-tie between background and the best class: a failure below points at the kernels, not at a rank flip
    assert bo.min_background_margin(o["probs"]) > 1e-3
    R = cfg.result_per_im
    det = Detector(cfg, 1, H, W, precision="split", use_cuda_graph=True)
    det.load_weights(Wt)
    try:
        det.set_stage("image", frame[None])
        det.run_phases(255)
        rec = stagewise(det, cfg, 0, o, {"config": "bg_score", "seed": seed, "H": H, "W": W, "dropped": dropped})
        n = int(det.get_stage("proposal_count")[0].reshape(-1)[0])
        gp = det.get_stage("probs")[0, :n, :, 0]
        np.testing.assert_array_equal(det.get_stage("bg_rank")[0].reshape(-1)[:n], bo.bg_rank(gp))
        fc = int(det.get_stage("final_count")[0].reshape(-1)[0])
        got = (det.get_stage("final_labels")[0].reshape(-1)[:fc], det.get_stage("final_boxes")[0].reshape(R, 4)[:fc],
               det.get_stage("final_probs")[0].reshape(-1)[:fc])
        final_margins(*got, o["final_labels"], o["final_boxes"], o["final_probs"], rec)
        exact_margins(*got, (o["final_labels"], o["final_boxes"], o["final_probs"]),
                      (o64["final_labels"], o64["final_boxes"], o64["final_probs"]), rec)
        feat = det.get_stage("fpn_box_feat")
        masks = det.get_masks()[0]
    finally:
        det.close()
    log_margins(rec)
    assert_stagewise(rec)
    assert_final(rec)
    assert rec["final"] > 0
    m = min(fc, len(o["final_probs"]))
    if rec["order_equal"]:
        assert rel(feat[:m], o["fpn_box_feat"][:m]) < 1e-4
    d = (np.abs(got[1][:, None, :] - o["final_boxes"][None, :, :]).max(-1)
         + 10.0 * (got[0][:, None] != o["final_labels"][None, :]))
    match = d.argmin(1)
    assert d.min(1).max() < 2e-3
    assert np.abs(masks[:fc] - o["final_masks"][match]).max() < 2e-4
    assert (masks[fc:] == 0).all()


def test_small_object_branch():
    from object_detection_tracking_b200.engine import Detector
    from object_detection_tracking_b200.synth import synth_weights
    from test_small_objects_gpu import _cfg as so_cfg
    from test_small_objects_gpu import _run, check_branch
    cfg = so_cfg(result_per_im=20, use_bg_score=True)
    W0 = synth_weights(cfg, 5)
    C, R = len(cfg.small_object_class_ids), cfg.result_per_im

    def run(Wt):
        det = Detector(cfg, 1, 192, 256, precision="split", use_cuda_graph=True)
        det.load_weights(Wt)
        try:
            o = _run(cfg, Wt, 1, det=det)
            o["so_bg_rank"] = det.get_stage("so_bg_rank").reshape(-1)
        finally:
            det.close()
        return o
    o0 = run(W0)
    assert int(o0["st"]["so_k"].reshape(-1)[0]) == R
    shift = bo.background_shift(o0["st"]["so_logits"].reshape(R, C + 1))
    Wt = dict(W0)
    for s in range(C):
        Wt = bo.with_background_shift(Wt, shift, "fastrcnn/small_objects/small_object_classification_c%d/b" % (s + 1))
    o = run(Wt)
    fl = o["st"]["so_logits"].reshape(R, C + 1)
    rank = bo.bg_rank(fl)
    np.testing.assert_array_equal(o["so_bg_rank"], rank)
    assert 0 < int((rank < 0).sum()) < R
    with bo.use_bg_score():
        rec = check_branch(cfg, Wt, o, 192, 256)
    assert rec["K"] == R and rec["n"] > 0


# ---- where the flag does nothing ----------------------------------------------------------------------------------------
def test_batch_graph_and_use_cpu_nms_ignore_the_flag_and_launch_counts():
    from object_detection_tracking_b200.backend import Mask_RCNN_FPN, Session
    from object_detection_tracking_b200.config import make_config
    from object_detection_tracking_b200.engine import Detector
    from object_detection_tracking_b200.synth import synth_frame, synth_weights
    H, W = 192, 256
    small = dict(resnet_num_block=(1, 1, 1, 1), max_size=W, short_edge_size=H)
    base = make_config(**small)
    frames = np.stack([synth_frame(H, W, seed=s) for s in (1, 2)]).astype(np.float32)
    Wt = bo.with_background_shift(synth_weights(base, 7), 3.0)
    outs, launches = {}, {}
    for flag in (None, False, True):
        cfg = make_config(**small) if flag is None else make_config(use_bg_score=flag, **small)
        for multi in (False, True):
            det = Detector(cfg, 2, H, W, precision="split", use_cuda_graph=True, multi_semantics=multi)
            det.load_weights(Wt)
            try:
                outs[flag, multi] = {k: v.copy() for k, v in det.detect_host(frames).items()}
                launches[flag, multi] = det.kernel_launches()
            finally:
                det.close()
    for multi in (False, True):
        assert launches[False, multi] == launches[None, multi]
        for k in outs[None, multi]:
            assert si.same_bits(outs[False, multi][k].view(F32), outs[None, multi][k].view(F32)), (multi, k)
    assert launches[True, True] == launches[None, True]
    for k in outs[None, True]:
        assert si.same_bits(outs[True, True][k].view(F32), outs[None, True][k].view(F32)), k
    assert launches[True, False] == launches[None, False] + 1
    assert not np.array_equal(outs[True, False]["boxes"], outs[None, False]["boxes"])      # the flag bites here
    # use_cpu_nms returns before fastrcnn_predictions (models.py:899-916)
    res = {}
    for flag in (False, True):
        m = Mask_RCNN_FPN(make_config(use_cpu_nms=True, use_bg_score=flag, **small))
        m.set_weights(Wt)
        res[flag] = Session().run([m.final_boxes, m.final_labels, m.final_probs], m.get_feed_dict_forward(frames[0]))
    for a, b in zip(res[False], res[True]):
        assert si.same_bits(a, b)
