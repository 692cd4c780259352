"""Relation-network box head (`add_relation_nn`) on the host: the oracle's module against an independent float64 numpy
loop over (i, g, j), the weight manifest and the importer's refusals, the synthetic weights of existing seeds, the
synthetic head's attention being neither degenerate nor vacuous, and the config / ABI plumbing."""
import hashlib
import math

import numpy as np
import pytest
import torch

from object_detection_tracking_b200.config import make_config
from object_detection_tracking_b200.synth import frcnn_weight_shapes, synth_frame, synth_weights
import relation_oracle
from oracle import frcnn

REL = dict(add_relation_nn=True)
NAMES = {"geo_emb/W": (4, 64), "geo_emb/b": (64,), "geo_conv/W": (1, 1, 64, 16), "geo_conv/b": (16,),
         "query_linear/W": (1024, 1024), "key_linear/W": (1024, 1024), "output_linear/W": (16384, 1024)}


def np_relation(h, boxes, W, scope):
    """float64 numpy relation_network (nn.py:115-190), one loop over query rows i, heads g and keys j."""
    h = h.astype(np.float64)
    K, D = h.shape
    dg = D // 16
    g64 = lambda n: W[scope + "/" + n].astype(np.float64)
    ew, eb, cw, cb = g64("geo_emb/W"), g64("geo_emb/b"), g64("geo_conv/W").reshape(64, 16), g64("geo_conv/b")
    q = h @ g64("query_linear/W")
    k = h @ g64("key_linear/W")
    b = boxes.astype(np.float64)
    w, hh = b[:, 2] - b[:, 0], b[:, 3] - b[:, 1]
    cx, cy = 0.5 * (b[:, 0] + b[:, 2]), 0.5 * (b[:, 1] + b[:, 3])
    o = np.zeros((K, 16 * D))
    for i in range(K):
        for g in range(16):
            s = np.empty(K)
            for j in range(K):
                enc = np.array([math.log(max(abs((cx[i] - cx[j]) / w[i]), 1e-3)),
                                math.log(max(abs((cy[i] - cy[j]) / w[i]), 1e-3)),        # the width, for dy too
                                math.log(w[i] / w[j]), math.log(hh[i] / hh[j])])
                wg = max(np.tanh(enc @ ew + eb) @ cw[:, g] + cb[g], 0.0)
                s[j] = math.log(max(wg, 1e-6)) + q[i, g * dg:(g + 1) * dg] @ k[j, g * dg:(g + 1) * dg] / math.sqrt(dg)
            p = np.exp(s - s.max())
            p /= p.sum()
            o[i, g * D:(g + 1) * D] = p @ h
    return o @ g64("output_linear/W")


def small_module(D, seed):
    rng = np.random.default_rng(seed)
    cfg = make_config(fpn_frcnn_fc_head_dim=D, **REL)
    W = {k: v for k, v in synth_weights(cfg, seed).items() if "/RM_r1/" in k}
    return rng, W


def boxes_for(rng, K, dup_centres=False):
    xy = rng.uniform(0, 200, (K, 2))
    wh = rng.uniform(4, 120, (K, 2))
    if dup_centres and K >= 3:                      # equal centres (|d| = 0 -> the 1e-3 clamp), other sizes
        c = xy[0] + wh[0] / 2
        xy[1:3] = c - wh[1:3] / 2
    b = np.concatenate([xy, xy + wh], 1).astype(np.float32)
    return b


@pytest.mark.parametrize("K", [1, 2, 7, 64])
def test_oracle_module_matches_numpy_loop(K):
    rng, W = small_module(64, 5 + K)
    h = np.maximum(rng.standard_normal((K, 64)), 0).astype(np.float32)
    b = boxes_for(rng, K, dup_centres=True)
    with frcnn.exact():
        got = relation_oracle.relation(frcnn._t(h), b, W, "fastrcnn/RM_r1").numpy()
    ref = np_relation(h, b, W, "fastrcnn/RM_r1")
    assert np.abs(got - ref).max() <= 1e-10 * max(1.0, np.abs(ref).max())
    got32 = relation_oracle.relation(frcnn._t(h), b, W, "fastrcnn/RM_r1").numpy()
    assert np.abs(got32 - ref).max() < 1e-4 * max(1.0, np.abs(ref).max())


def test_k1_is_the_roi_itself():
    """K = 1: weight exactly 1 on the ROI, so the module is output_linear of h tiled over the 16 heads."""
    rng, W = small_module(64, 3)
    h = rng.uniform(0, 1, (1, 64)).astype(np.float32)
    b = boxes_for(rng, 1)
    with frcnn.exact():
        p = relation_oracle.attention(frcnn._t(h), b, W, "fastrcnn/RM_r1").numpy()
        got = relation_oracle.relation(frcnn._t(h), b, W, "fastrcnn/RM_r1").numpy()
    assert p.shape == (1, 16, 1) and (p == 1.0).all()
    np.testing.assert_allclose(got, np.tile(h.astype(np.float64), 16) @ W["fastrcnn/RM_r1/output_linear/W"], rtol=1e-12)


def test_padded_rows_do_not_feed_valid_rows():
    """The engine runs K rows with count valid: the module on the first `count` rows alone is what the valid rows get, and
    the oracle (which only ever sees the valid rows) is unaffected by what the padding would hold."""
    rng, W = small_module(64, 9)
    h = np.maximum(rng.standard_normal((12, 64)), 0).astype(np.float32)
    b = boxes_for(rng, 12)
    with frcnn.exact():
        full = relation_oracle.relation(frcnn._t(h[:7]), b[:7], W, "fastrcnn/RM_r1").numpy()
        h2 = h.copy(); h2[7:] = 1e3
        again = relation_oracle.relation(frcnn._t(h2[:7]), b[:7], W, "fastrcnn/RM_r1").numpy()
    np.testing.assert_array_equal(full, again)
    np.testing.assert_allclose(full, np_relation(h[:7], b[:7], W, "fastrcnn/RM_r1"), rtol=1e-10, atol=1e-12)


def test_dy_is_divided_by_the_width():
    """geometric_encoding divides the y offset by w_i (nn.py:287-289): boxes that differ only in height change dy only
    through the centres, never through h_i."""
    b = torch.tensor([[0, 0, 10, 40], [0, 20, 10, 60]], dtype=torch.float64)
    enc = relation_oracle.geometric_encoding(b)
    assert float(enc[0, 1, 1]) == pytest.approx(math.log(20 / 10))            # |cy0 - cy1| / w0, not / h0 (= log 0.5)
    assert float(enc[0, 1, 0]) == pytest.approx(math.log(1e-3))               # equal centres in x: the clamp


@pytest.mark.parametrize("agnostic", [False, True])
def test_manifest_lists_the_relation_variables(agnostic):
    cfg = make_config(use_frcnn_class_agnostic=agnostic, **REL)
    sh = frcnn_weight_shapes(cfg)
    base = frcnn_weight_shapes(make_config(use_frcnn_class_agnostic=agnostic))
    extra = {k: v for k, v in sh.items() if k not in base}
    assert extra == {"fastrcnn/%s/%s" % (m, n): s for m in ("RM_r1", "RM_r2") for n, s in NAMES.items()}
    w = synth_weights(cfg, 7)
    assert set(w) == set(sh)
    for k, v in w.items():
        assert tuple(v.shape) == tuple(sh[k]), k


def test_no_relation_variables_without_the_flag_or_with_the_conv_head():
    for cfg in (make_config(), make_config(use_conv_frcnn_head=True, **REL),
                make_config(use_conv_frcnn_head=True, use_gn=True, **REL)):
        assert not [k for k in frcnn_weight_shapes(cfg) if "/RM_r" in k]
        assert not [k for k in synth_weights(cfg, 3) if "/RM_r" in k]


@pytest.mark.parametrize("missing", ["fastrcnn/RM_r1/geo_conv/b", "fastrcnn/RM_r2/output_linear/W"])
def test_check_weights_refuses_a_relation_set_without_one_array(missing):
    from object_detection_tracking_b200.backend import check_weights
    cfg = make_config(**REL)
    w = synth_weights(cfg, 2)
    del w[missing]
    with pytest.raises(ValueError) as e:
        check_weights(cfg, w)
    assert "1 missing" in str(e.value) and missing in str(e.value)
    assert len(check_weights(make_config(), w)) == len(frcnn_weight_shapes(make_config()))   # ignored without the flag


# sha256 (first 16 hex digits) over the sorted names and bytes of synth_weights(cfg, 1234), as before add_relation_nn
SEED_DIGESTS = {
    "default": (dict(), "db0c69c79a4e1bee"),
    "gn_convhead": (dict(use_gn=True, use_conv_frcnn_head=True), "2934f7bc85fbfc2f"),
    "se": (dict(use_se=True, use_frcnn_class_agnostic=True, use_dilations=False), "35169c6700bc40d4"),
    "mask": (dict(add_mask=True), "95eb188a019875a2"),
    "r50": (dict(resnet_num_block=(3, 4, 6, 3), num_class=81), "d46a6e37cf6d8a28"),
}


def _digest(w):
    h = hashlib.sha256()
    for k in sorted(w):
        h.update(k.encode())
        h.update(w[k].tobytes())
    return h.hexdigest()[:16]


@pytest.mark.parametrize("name", sorted(SEED_DIGESTS))
def test_existing_seeds_are_unchanged(name):
    kw, digest = SEED_DIGESTS[name]
    assert _digest(synth_weights(make_config(**kw), 1234)) == digest
    # with the relation head every non-RM array is the seed's own
    w = synth_weights(make_config(**dict(kw, **REL)), 1234)
    assert _digest({k: v for k, v in w.items() if "/RM_r" not in k}) == digest


def test_config_and_abi_carry_add_relation_nn():
    from object_detection_tracking_b200 import _lib
    assert make_config().add_relation_nn is False
    assert _lib.make_config(make_config(), 1, 192, 256).add_relation_nn == 0
    assert _lib.make_config(make_config(**REL), 1, 192, 256).add_relation_nn == 1


SMALL = dict(resnet_num_block=(1, 1, 2, 2), max_size=256, short_edge_size=192)


def test_synthetic_relation_head_is_not_degenerate():
    """On the proposals and fc6 rows of a real (small) forward pass: a real share of the (i, g, j) geometry weights hits
    the 1e-6 clamp and a real share does not, the attention rows are neither one-hot nor uniform, and each module's
    output is the size of its input."""
    cfg = make_config(use_frcnn_class_agnostic=True, **dict(SMALL, **REL))
    W = synth_weights(cfg, 99)
    frame = synth_frame(192, 256, seed=3).astype(np.float32)
    o = relation_oracle.forward(cfg, W, frame, stages=True)
    pb = o["proposal_boxes"]
    K = len(pb)
    assert K > 50
    t = frcnn._t
    x = t(o["roi_feat"].reshape(K, -1))
    h = torch.relu(x @ t(W["fastrcnn/fc6/W"]) + t(W["fastrcnn/fc6/b"]))
    for m, hin in (("RM_r1", h), ):
        scope = "fastrcnn/" + m
        enc = relation_oracle.geometric_encoding(t(pb))
        e = torch.tanh(enc @ t(W[scope + "/geo_emb/W"]) + t(W[scope + "/geo_emb/b"]))
        wg = (e @ t(W[scope + "/geo_conv/W"]).reshape(64, 16) + t(W[scope + "/geo_conv/b"])).numpy()
        clamped = float((wg <= 1e-6).mean())
        assert 0.2 < clamped < 0.8, clamped
        p = relation_oracle.attention(hin, pb, W, scope).numpy()
        top = p.max(-1)
        assert np.median(top) < 0.9 and np.median(top) > 5.0 / K, (np.median(top), K)
        ent = -(p * np.log(np.maximum(p, 1e-30))).sum(-1) / math.log(K)
        assert 0.05 < np.median(ent) < 0.95, np.median(ent)
        out = relation_oracle.relation(hin, pb, W, scope).numpy()
        ratio = np.linalg.norm(out) / np.linalg.norm(hin.numpy())
        assert 0.2 < ratio < 5.0, ratio
    r1 = relation_oracle.LAST["rm_r1"]
    ratio2 = np.linalg.norm(r1 - h.numpy()) / np.linalg.norm(h.numpy())
    assert 0.2 < ratio2 < 5.0, ratio2
    assert len(o["final_boxes"]) > 0


def test_relation_oracle_is_frcnn_without_the_flag():
    cfg = make_config(**SMALL)
    W = synth_weights(cfg, 99)
    frame = synth_frame(192, 256, seed=4).astype(np.float32)
    a = frcnn.forward(cfg, W, frame, stages=False)
    b = relation_oracle.forward(cfg, W, frame, stages=False)
    for k in ("final_boxes", "final_labels", "final_probs"):
        np.testing.assert_array_equal(a[k], b[k])
    # the flag changes the detections, and the relation oracle sees the proposals of both graphs
    rcfg = make_config(**dict(SMALL, **REL))
    rw = synth_weights(rcfg, 99)
    c = relation_oracle.forward(rcfg, rw, frame, stages=True)
    d = frcnn.forward(rcfg, rw, frame, stages=True)
    np.testing.assert_array_equal(c["proposal_boxes"], d["proposal_boxes"])
    assert np.abs(c["cls_logits"] - d["cls_logits"]).max() > 1e-2
    m = relation_oracle.forward_multi(rcfg, rw, [frame, frame[::-1].copy()], stages=True)
    assert m["final_valid_indices"].min() > 0
