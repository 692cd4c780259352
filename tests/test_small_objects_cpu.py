"""Small-object branch (`use_small_object_head`) without a GPU: person_object_relation and geometric_encoding_pair
against a literal float64 loop (the key box's width as the divisor, a zero-width box, one key row), the logits-not-probs
final selection with the score filter, the manifest, config resolution and every refusal (in normalize_config and at
b2_create_ex4, before any device is touched), unchanged synthetic arrays for existing seeds and the b2_config_ext4
layout."""
import copy
import ctypes
import hashlib
import math

import numpy as np
import pytest

import so_oracle
from oracle import frcnn


def _cfg(**kw):
    from object_detection_tracking_b200.config import make_config
    return make_config(**dict(dict(num_class=17, use_small_object_head=True), **kw))


def _loop(h, boxes, ref_boxes, ref, W, scope=so_oracle.REL):
    """nn.py:194-332 restated as plain float64 loops."""
    h, ref = h.astype(np.float64), ref.astype(np.float64)
    K, D = h.shape
    R = ref.shape[0]
    g = {k.rsplit("/", 2)[-2] + "/" + k.rsplit("/", 1)[-1]: v.astype(np.float64) for k, v in W.items() if k.startswith(scope)}
    ew, eb, cw, cb = g["geo_emb/W"], g["geo_emb/b"], g["geo_conv/W"].reshape(64, 16), g["geo_conv/b"]
    q, k = h @ g["query_linear/W"], ref @ g["key_linear/W"]
    dg = D // 16
    out = np.zeros((K, 16 * D))
    for i in range(K):
        x1, y1, x2, y2 = boxes[i].astype(np.float64)
        for gg in range(16):
            logits = np.zeros(R)
            for j in range(R):
                a1, b1, a2, b2 = ref_boxes[j].astype(np.float64)
                wj, hj = a2 - a1, b2 - b1
                with np.errstate(divide="ignore", invalid="ignore"):
                    enc = [math.log(max(abs((0.5 * (x1 + x2) - 0.5 * (a1 + a2)) / wj), 1e-3)),
                           math.log(max(abs((0.5 * (y1 + y2) - 0.5 * (b1 + b2)) / wj), 1e-3)),
                           np.log(np.float64(x2 - x1) / wj), np.log(np.float64(y2 - y1) / hj)]
                e = np.tanh(np.asarray(enc) @ ew + eb)
                wg = max(e @ cw[:, gg] + cb[gg], 0.0)
                logits[j] = math.log(max(wg, 1e-6)) + q[i, gg * dg:(gg + 1) * dg] @ k[j, gg * dg:(gg + 1) * dg] / math.sqrt(dg)
            p = np.exp(logits - logits.max())
            p /= p.sum()
            out[i, gg * D:(gg + 1) * D] = p @ ref
    return out @ g["output_linear/W"]


def _weights(rng, D):
    f = np.float32
    s = so_oracle.REL
    return {s + "/geo_emb/W": (rng.standard_normal((4, 64)) * 0.3).astype(f), s + "/geo_emb/b": rng.standard_normal(64).astype(f) * 0.1,
            s + "/geo_conv/W": (rng.standard_normal((1, 1, 64, 16)) / 8).astype(f),
            s + "/geo_conv/b": (rng.standard_normal(16) * 0.05).astype(f),
            s + "/query_linear/W": (rng.standard_normal((D, D)) * 0.3).astype(f),
            s + "/key_linear/W": (rng.standard_normal((D, D)) * 0.3).astype(f),
            s + "/output_linear/W": (rng.standard_normal((16 * D, D)) * 0.1).astype(f)}


@pytest.mark.parametrize("K,R", [(3, 1), (4, 2), (5, 6)])
def test_person_object_relation_vs_loop(K, R):
    rng = np.random.default_rng(K * 10 + R)
    D = 32
    h, ref = rng.standard_normal((K, D)).astype(np.float32), rng.standard_normal((R, D)).astype(np.float32)
    boxes = np.array([[10, 20, 60, 90], [30, 30, 30, 80], [0, 0, 5, 5], [100, 50, 180, 70], [40, 40, 41, 200]],
                     np.float32)[:K]                       # row 1: a zero-width query box
    ref_boxes = np.array([[15, 10, 45, 120], [70, 5, 72, 60], [0, 0, 20, 20], [90, 90, 300, 100], [5, 5, 6, 6],
                          [1, 2, 3, 4]], np.float32)[:R]
    W = _weights(rng, D)
    with frcnn.exact():
        got = frcnn._np(so_oracle.person_object_relation(h, boxes, ref_boxes, ref, W))
    want = _loop(h, boxes, ref_boxes, ref, W)
    assert np.isfinite(got).all()   # the zero-width query box: dw = -inf, tanh saturates
    np.testing.assert_allclose(got, want, rtol=1e-6, atol=1e-6 * np.abs(want).max())
    if R == 1:   # one key row: weight 1 for every query row (the reference's tf.squeeze fails there)
        np.testing.assert_allclose(got, np.broadcast_to(ref.astype(np.float64) @ np.tile(np.eye(D), (1, 16)) @
                                                        W[so_oracle.REL + "/output_linear/W"].astype(np.float64), got.shape),
                                   rtol=1e-6)


def test_geometry_divides_by_key_width():
    import torch
    b1 = torch.tensor([[0.0, 0.0, 10.0, 10.0]], dtype=torch.float64)
    b2 = torch.tensor([[100.0, 0.0, 102.0, 40.0]], dtype=torch.float64)
    enc = so_oracle.geometric_encoding_pair(b1, b2)[0, 0].numpy()
    # centres (5, 5) and (101, 20): |dx| / w_j = 96 / 2, |dy| / w_j = 15 / 2 (the key's width, not the query's 10)
    np.testing.assert_allclose(enc, [math.log(48.0), math.log(7.5), math.log(10 / 2), math.log(10 / 40)])


def test_final_selection_uses_logits_and_filter():
    """fastrcnn_predictions on the rebuilt logits: negative scores kept without the filter, dropped with it."""
    cfg = _cfg(result_per_im=5)
    rng = np.random.default_rng(0)
    K, C = 5, 4
    xy = rng.uniform(0, 100, (K, C, 2)).astype(np.float32)
    boxes = np.concatenate([xy, xy + 30], 2).astype(np.float32)
    logits = (rng.standard_normal((K, C + 1)) - 2.0).astype(np.float32)
    f = copy.copy(cfg)
    f.result_score_thres = -np.inf
    pred, probs = frcnn.fastrcnn_predictions(boxes, logits, f)
    assert (probs < 0).any() and len(probs) == 5
    assert np.all(np.diff(probs) <= 0)
    pred_t, probs_t = frcnn.fastrcnn_predictions(boxes, logits, cfg)
    assert (probs_t > cfg.result_score_thres).all() and len(probs_t) < len(probs)


def test_manifest():
    from object_detection_tracking_b200.synth import frcnn_weight_shapes
    base = frcnn_weight_shapes(_cfg(use_small_object_head=False))
    sh = frcnn_weight_shapes(_cfg())
    extra = {k: v for k, v in sh.items() if k not in base}
    assert extra == {"fastrcnn/small_objects/small_object_classification_c%d/%s" % (i, n): s
                     for i in range(1, 5) for n, s in (("W", (1024, 2)), ("b", (2,)))}
    sh = frcnn_weight_shapes(_cfg(use_so_association=True))
    p = so_oracle.REL + "/"
    assert {k: v for k, v in sh.items() if k.startswith(p)} == {
        p + "geo_emb/W": (4, 64), p + "geo_emb/b": (64,), p + "geo_conv/W": (1, 1, 64, 16), p + "geo_conv/b": (16,),
        p + "query_linear/W": (1024, 1024), p + "key_linear/W": (1024, 1024), p + "output_linear/W": (16384, 1024)}


def test_incomplete_checkpoint_refused_by_name():
    from object_detection_tracking_b200.backend import check_weights
    from object_detection_tracking_b200.synth import synth_weights
    cfg = _cfg(resnet50=True, use_so_association=True)
    W = synth_weights(cfg, 1)
    del W[so_oracle.REL + "/key_linear/W"]
    with pytest.raises(ValueError, match="key_linear"):
        check_weights(cfg, W)


def test_config_resolution():
    from object_detection_tracking_b200.class_ids import targetClass2id_mergeProp
    assert targetClass2id_mergeProp["Prop_plus_Push_Pulled_Object"] == 16 and targetClass2id_mergeProp["BG"] == 0
    cfg = _cfg(use_so_association=True)
    assert cfg.small_object_class_ids == (12, 10, 16, 13) and cfg.so_person_class_id == 2
    table = {"BG": 0, "Person": 3, "Bike": 1, "Prop": 2}
    cfg = _cfg(num_class=4, small_objects=["Bike", "Prop"], classname2id=table, use_so_association=True)
    assert cfg.small_object_class_ids == (1, 2) and cfg.so_person_class_id == 3
    off = _cfg(use_small_object_head=False)
    assert off.small_object_class_ids == () and off.so_person_class_id == 0


@pytest.mark.parametrize("kw,match", [
    (dict(small_objects=["Prop", "Nope"]), "'Nope' is not a class name"),
    (dict(small_objects=["Prop", "Prop"]), "more than once"),
    (dict(small_objects=["BG"]), "'BG'"),
    (dict(small_objects=[]), "empty"),
    (dict(num_class=15), "outside 1..num_class-1"),
    (dict(use_so_association=True, classname2id={"BG": 0, "Prop": 1}, small_objects=["Prop"]), "'Person'"),
    (dict(use_so_association=True, so_person_topk=0), "so_person_topk"),
    (dict(use_frcnn_class_agnostic=True), "use_frcnn_class_agnostic"),
    (dict(use_partial_classes=True), "use_partial_classes"),
    (dict(use_conv_frcnn_head=True), "use_conv_frcnn_head"),
])
def test_config_refusals(kw, match):
    with pytest.raises(ValueError, match=match):
        _cfg(**kw)


def _create(cfg, batch=1, multi=False, **edit):
    from object_detection_tracking_b200 import _lib
    lib = _lib.load()
    c = _lib.make_config(cfg, batch, 192, 256, "float32", "split", "tcgen05", True, multi, 0)
    e = _lib.make_config_ext4(cfg)
    for k, v in edit.items():
        if hasattr(c, k):
            setattr(c, k, v)
        else:
            setattr(e, k, v)
    ctx = ctypes.c_void_p(0)
    rc = lib.b2_create_ex4(ctypes.byref(ctx), 0, ctypes.byref(c), None, None, None, ctypes.byref(e))
    assert rc != 0 and not ctx.value
    return lib.b2_last_error().decode()


@pytest.mark.parametrize("edit,match", [
    (dict(class_agnostic=1), "use_frcnn_class_agnostic"),
    (dict(conv_head_dim=256), "use_conv_frcnn_head"),
    (dict(num_small_objects=0), "num_small_objects"),
    (dict(num_small_objects=17), "num_small_objects"),
    (dict(so_person_topk=0), "so_person_topk"),
    (dict(so_person_class_id=17), "so_person_class_id"),
])
def test_abi_refusals(edit, match):
    assert match in _create(_cfg(use_so_association=True), **edit)


def test_abi_refuses_batch_and_multi():
    assert "batch 1" in _create(_cfg(), batch=2)
    assert "batch 1" in _create(_cfg(), multi=True)


def test_abi_refuses_bad_ids():
    cfg = _cfg()
    from object_detection_tracking_b200 import _lib
    lib = _lib.load()
    c = _lib.make_config(cfg, 1, 192, 256, "float32", "split", "tcgen05", True, False, 0)
    e = _lib.make_config_ext4(cfg)
    e.small_object_class_ids[1] = e.small_object_class_ids[0]
    ctx = ctypes.c_void_p(0)
    assert lib.b2_create_ex4(ctypes.byref(ctx), 0, ctypes.byref(c), None, None, None, ctypes.byref(e)) != 0
    assert "appears twice" in lib.b2_last_error().decode()
    e.small_object_class_ids[1] = 0
    assert lib.b2_create_ex4(ctypes.byref(ctx), 0, ctypes.byref(c), None, None, None, ctypes.byref(e)) != 0
    assert "not a class id" in lib.b2_last_error().decode()


def test_ext4_layout():
    from object_detection_tracking_b200._lib import B2ConfigExt4
    assert ctypes.sizeof(B2ConfigExt4) == 4 * (2 + 80 + 4)
    assert B2ConfigExt4.small_object_class_ids.offset == 8
    assert B2ConfigExt4.use_so_score_thres.offset == 4 * (2 + 80 + 3)


def _digest(w):
    h = hashlib.sha256()
    for k in sorted(w):
        h.update(k.encode())
        h.update(np.ascontiguousarray(w[k]).tobytes())
    return h.hexdigest()


def test_existing_seed_arrays_unchanged():
    """The branch's arrays come from a stream of their own: every other array of a seed is the same with the flag."""
    from object_detection_tracking_b200.synth import synth_weights
    for kw in (dict(), dict(add_relation_nn=True), dict(use_att_frcnn_head=True, add_mask=True)):
        base = synth_weights(_cfg(use_small_object_head=False, resnet50=True, **kw), 7)
        full = synth_weights(_cfg(resnet50=True, use_so_association=True, **kw), 7)
        assert _digest({k: full[k] for k in base}) == _digest(base)
        assert set(full) - set(base) and all(k.startswith("fastrcnn/small_objects/") for k in set(full) - set(base))


def test_oracle_raises_on_unequal_counts():
    """Prop's boxes all decode onto proposal 0's box, so its NMS keeps 1 while the other classes keep 3: the reference's
    tf.map_fn cannot stack that, and the oracle raises with the counts."""
    cfg = _cfg(result_per_im=3)
    N = 6
    x = np.arange(N, dtype=np.float32) * 50
    pb = np.stack([x, np.zeros(N, np.float32), x + 40, np.full(N, 40, np.float32)], 1)   # disjoint proposals
    cls = np.random.default_rng(1).standard_normal((N, 17)).astype(np.float32)
    box = np.zeros((N, 16, 4), np.float32)
    box[:, 11, 0] = (pb[0, 0] - pb[:, 0]) / 40 * 10         # Prop (id 12): every centre moved onto proposal 0's
    out = dict(proposal_boxes=pb, cls_logits=cls, box_logits=box, p23456=[])
    with pytest.raises(so_oracle.SoCountError) as e:
        so_oracle.branch(cfg, {}, out, (300, 300))
    assert e.value.counts == [1, 3, 3, 3]
