"""Writes every output of the three engines and the GEMM entry points at fixed seeds to one npz, so that two builds can be
compared byte for byte (a host-side refactor must leave all of them unchanged).

    python tools/engine_fingerprint.py --out a.npz [--root <tree>]

--root selects the source tree whose package (and library, built in that tree) is exercised; default: this tree.
Covers: the detector (BN R101 at batch 2 with multi semantics, GN with the conv box head at batch 2, add_mask, and at
192x256 with few blocks use_se (v6), use_resnext, add_relation_nn, use_deformable alone and with use_gn, use_basic_block
alone and with use_gn + use_conv_frcnn_head), each in split and fp16 precision, CUDA graph and eager, B2_SPLIT=1 and 2,
all four feat_modes, several stages, the step list and launch count; b2_box_features; op_relation, op_deform_conv2d
(tensor and CUDA cores, with the offsets) and op_squeeze_excite (with and without a residual, with the gate) in both
precisions; OSNet and ResNet-101 ReID embeddings, activations and launch counts; EfficientDet-D0 with
an EfficientNet-b0 backbone (run_features, detect, stages, step list, launch count); b2_cosine_cost, b2_distance_matrix
and b2_track_pair_cost over a growing-then-shrinking shape sequence."""
import argparse
import os
import sys

import numpy as np

ap = argparse.ArgumentParser()
ap.add_argument("--out", required=True)
ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
args = ap.parse_args()
sys.path.insert(0, os.path.abspath(args.root))

from object_detection_tracking_b200 import _lib  # noqa: E402
from object_detection_tracking_b200.config import make_config  # noqa: E402
from object_detection_tracking_b200.effdet import EffdetEngine  # noqa: E402
from object_detection_tracking_b200.effdet_config import feat_sizes, make_effdet_config  # noqa: E402
from object_detection_tracking_b200.engine import (Detector, cosine_cost, op_deform_conv2d, op_relation,  # noqa: E402
                                                  op_squeeze_excite)
from object_detection_tracking_b200.reid import ReidEngine, compute_distance_matrix  # noqa: E402
from object_detection_tracking_b200.synth import (synth_effdet_weights, synth_efficientnet_weights, synth_frame,  # noqa: E402
                                                  synth_osnet_state, synth_resnet101_reid_state, synth_weights)

out = {}
H, W = 192, 256
STAGES = ["c1", "pool", "c2", "c5", "p2", "p6", "rpn_l0", "lvl_count", "proposal_boxes", "proposal_count", "roi_feat",
          "head_logits", "probs", "final_count"]


def steps(name, lst, launches):
    out[name + "/step_names"] = np.array([s[0] for s in lst])
    out[name + "/step_kind"] = np.array([s[1] for s in lst], np.int64)
    out[name + "/step_flops"] = np.array([s[2] for s in lst], np.float64)
    out[name + "/step_bytes"] = np.array([s[3] for s in lst], np.float64)
    out[name + "/launches"] = np.array([launches], np.int64)


def detector(tag, cfg, Wt, batch, multi, extra_stages=()):
    frames = np.stack([synth_frame(H, W, seed=70 + s) for s in range(batch)]).astype(np.float32)
    for prec in ("split", "fp16"):
        for graph in (True, False):
            for nsplit in ("1", "2"):
                os.environ["B2_SPLIT"] = nsplit
                name = "%s/%s/%s/split%s" % (tag, prec, "graph" if graph else "eager", nsplit)
                det = Detector(cfg, batch, H, W, precision=prec, use_cuda_graph=graph, multi_semantics=multi)
                det.load_weights(Wt)
                for mode in range(4):
                    r = det.detect_host(frames, feat_mode=mode)
                    for k, v in r.items():
                        out["%s/mode%d/%s" % (name, mode, k)] = np.array(v).copy()
                for s in STAGES + list(extra_stages):
                    out[name + "/stage/" + s] = det.get_stage(s)
                if det.cfg.add_mask:
                    out[name + "/masks"] = det.get_masks()
                prof = det.profile_steps(reps=1)
                steps(name, [(p["name"], p["kind"], p["flops"], p["bytes"]) for p in prof], det.kernel_launches())
                det.close()
    os.environ.pop("B2_SPLIT", None)


bn = make_config(resnet_num_block=(3, 4, 23, 3), max_size=W, short_edge_size=H, num_class=81)
Wbn = synth_weights(bn, 11)
detector("bn_r101", bn, Wbn, 2, True, ["c3", "c4", "fc6", "fc7"])
gn = make_config(resnet_num_block=(1, 1, 2, 2), max_size=W, short_edge_size=H, num_class=81, use_gn=True,
                 use_conv_frcnn_head=True)
detector("gn_head", gn, synth_weights(gn, 12), 2, True, ["fc"])
mk = make_config(resnet_num_block=(1, 1, 2, 1), max_size=W, short_edge_size=H, add_mask=True)
detector("mask", mk, synth_weights(mk, 13), 1, False, ["mask_logits", "final_masks"])
# the detector variants at small geometry (as in their feature tests), batch 2 with multi semantics
SMALL = dict(max_size=W, short_edge_size=H)
DEFORM_BLOCKS = ["group%d/block0/conv2_%s" % (g, k) for g in (1, 2, 3) for k in ("offset", "sample")]
for tag, kw, seed, extra in (
        ("se_v6", dict(resnet_num_block=(1, 1, 2, 2), use_se=True, use_frcnn_class_agnostic=True, use_dilations=False,
                       version=6), 14, ["c3", "c4"]),
        ("resnext", dict(resnet_num_block=(1, 1, 2, 2), use_resnext=True), 15, ["c3", "c4"]),
        ("relation", dict(resnet_num_block=(1, 1, 2, 2), add_relation_nn=True), 16, ["fc6", "fc7", "rm_r1", "rm_r2"]),
        ("deform", dict(resnet_num_block=(1, 1, 2, 1), use_deformable=True, use_dilations=False), 17, DEFORM_BLOCKS),
        ("deform_gn", dict(resnet_num_block=(1, 1, 2, 1), use_deformable=True, use_dilations=False, use_gn=True), 18,
         DEFORM_BLOCKS),
        ("basic", dict(resnet_num_block=(1, 2, 1, 1), use_basic_block=True), 19, ["c3", "c4"]),
        ("basic_gn_head", dict(resnet_num_block=(1, 2, 1, 1), use_basic_block=True, use_gn=True, use_conv_frcnn_head=True),
         20, ["c3", "c4", "fc"])):
    cfg = make_config(**dict(SMALL, **kw))
    detector(tag, cfg, synth_weights(cfg, seed), 2, True, extra)

# the composite single-op entry points at fixed seeds
orng = np.random.default_rng(21)
for prec in ("split", "fp16"):
    sp = prec == "split"
    B, K, D = 2, 50, 256
    h = np.maximum(orng.standard_normal((B, K, D)), 0).astype(np.float32)
    xy = orng.uniform(0, 200, (B, K, 2))
    boxes = np.concatenate([xy, xy + orng.uniform(8, 60, (B, K, 2))], -1).astype(np.float32)
    rw = {k: (orng.standard_normal(s) * 0.1).astype(np.float32)
          for k, s in (("geo_emb/W", (4, 64)), ("geo_emb/b", (64,)), ("geo_conv/W", (1, 1, 64, 16)), ("geo_conv/b", (16,)),
                       ("query_linear/W", (D, D)), ("key_linear/W", (D, D)), ("output_linear/W", (16 * D, D)))}
    out["op/relation/" + prec] = op_relation(h, boxes, np.array([K, 31], np.int32), rw, split=sp)
    B, Hd, Wd, C = 2, 13, 19, 128
    x = np.maximum(orng.standard_normal((B, Hd, Wd, C)), 0).astype(np.float32)
    ow = (orng.standard_normal((3, 3, C, 18)) * 0.05).astype(np.float32)
    ob = (orng.standard_normal(18) * 0.5).astype(np.float32)
    w = (orng.standard_normal((3, 3, C, C)) / np.sqrt(9 * C)).astype(np.float32)
    for impl in ("tcgen05", "simt"):
        o, off = op_deform_conv2d(x, ow, ob, w, impl=impl, split=sp, return_offsets=True)
        out["op/deform/%s/%s/out" % (impl, prec)] = o
        out["op/deform/%s/%s/offsets" % (impl, prec)] = off
    B, Hs, Ws, C = 2, 10, 12, 256
    x = orng.standard_normal((B, Hs, Ws, C)).astype(np.float32)
    w1 = (orng.standard_normal((C, C // 16)) * 0.2).astype(np.float32)
    b1 = orng.uniform(0, 0.1, C // 16).astype(np.float32)
    w2 = (orng.standard_normal((C // 16, C)) * 0.3).astype(np.float32)
    b2 = (orng.standard_normal(C) * 0.4).astype(np.float32)
    r = orng.standard_normal((B, Hs, Ws, C)).astype(np.float32)
    for name, res in (("res", r), ("nores", None)):
        o, g = op_squeeze_excite(x, w1, b1, w2, b2, res=res, split=sp)
        out["op/se/%s/%s/out" % (name, prec)] = o
        out["op/se/%s/%s/gate" % (name, prec)] = g

# given-box features (batch-1 context, uncropped levels)
det = Detector(bn, 1, H, W, precision="split")
det.load_weights(Wbn)
boxes = np.array([[10, 12, 80, 90], [100, 20, 250, 180], [0, 0, 255, 191], [30.5, 40.25, 31.5, 41.0]] * 30, np.float32)
out["box_features"] = det.box_features(synth_frame(H, W, seed=3).astype(np.float32), boxes)
det.close()

# ReID
rng = np.random.default_rng(5)
for model, state, n, acts in (("osnet_x1_0", synth_osnet_state(4321), 6, ["conv1", "maxpool", "conv2.0.x1", "conv2.0.s2",
                                                                          "conv2.0.x2", "conv3", "conv5"]),
                              ("resnet101", synth_resnet101_reid_state(2468), 3, ["conv1", "maxpool", "layer1.0",
                                                                                 "layer3.22", "layer4"])):
    for prec in ("split", "fp16"):
        eng = ReidEngine(batch=8 if n > 4 else 4, precision=prec, model=model)
        eng.load_state(state)
        crops = rng.integers(0, 256, (n,) + eng.image_size + (3,), dtype=np.uint8)
        name = "reid/%s/%s" % (model, prec)
        out[name + "/feats"] = eng.embed(crops)
        out[name + "/feats_small"] = eng.embed(crops[:2])
        for a in acts:
            out[name + "/act/" + a] = eng.get_activation(a)
        out[name + "/launches"] = np.array([eng.num_launches()], np.int64)
        eng.close()

# EfficientDet-D0 + EfficientNet-b0
for prec in ("split", "fp16"):
    cfg = make_effdet_config("efficientdet-d0", 256, 384, fpn_cell_repeats=2, box_class_repeats=2)
    Wt = dict(synth_effdet_weights(cfg))
    Wt.update(synth_efficientnet_weights("efficientnet-b0"))
    eng = EffdetEngine(cfg, Wt, precision=prec, backbone="efficientnet-b0")
    name = "effdet/" + prec
    frng = np.random.default_rng(7)
    fs = feat_sizes(cfg)
    feats = {l: np.abs(frng.standard_normal((cfg.backbone_channels[l - 3],) + fs[l])).astype(np.float32) for l in (3, 4, 5)}
    for k, v in eng.run_features(feats, image_scale=1.25).items():
        out[name + "/features/" + k] = np.array(v)
    frame = np.random.default_rng(8).integers(0, 256, (300, 500, 3), dtype=np.uint8)
    for k, v in eng.detect(frame).items():
        out[name + "/detect/" + k] = np.array(v)
    for s in ["image", "stem", "block_0", "c3", "c5", "fpn3", "fpn7", "cls3", "box5"]:
        out[name + "/stage/" + s] = eng.stage(s)
    steps(name, [(p[0], p[1], p[3], p[4]) for p in eng.profile_steps(reps=1)], eng.num_launches)
    eng.close()

# GEMM entry points over growing-then-shrinking shapes
grng = np.random.default_rng(9)
for i, (S, N, D) in enumerate([(5, 3, 128), (300, 40, 128), (1200, 150, 512), (700, 90, 2048), (40, 7, 128), (3, 2, 64)]):
    T = max(1, S // 7)
    seg = np.concatenate([[0], np.sort(grng.integers(0, S + 1, T - 1)), [S]]).astype(np.int32)
    gal = grng.standard_normal((S, D)).astype(np.float32)
    dets = grng.standard_normal((N, D)).astype(np.float32)
    for prec in ("split", "fp16"):
        out["cosine/%d/%s" % (i, prec)] = cosine_cost(gal, seg, dets, precision=prec)
        for metric in ("cosine", "euclidean"):
            out["distance/%d/%s/%s" % (i, prec, metric)] = compute_distance_matrix(gal, dets, metric, precision=prec).numpy()
        M = max(1, N // 3)
        segb = np.concatenate([[0], np.sort(grng.integers(0, N + 1, M - 1)), [N]]).astype(np.int32)
        gate = (grng.random((T, M)) < 0.8).astype(np.uint8)
        pc = np.zeros((T, M), np.float32)
        _lib.check(_lib.load().b2_track_pair_cost(0, _lib.ptr(gal), _lib.ptr(seg), T, _lib.ptr(dets), _lib.ptr(segb), M, D,
                                                  _lib.ptr(gate), 999.0, 1 if prec == "split" else 0, _lib.ptr(pc)),
                   "b2_track_pair_cost")
        out["pair/%d/%s" % (i, prec)] = pc

os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
np.savez(args.out, **out)
print("wrote %d arrays to %s" % (len(out), args.out))
