"""ResNet-18 / ResNet-34 detectors (`--resnet18` / `--resnet34`, `use_basic_block`) on the host: the oracle's basic block
against an independent float64 numpy loop (stride 1 and 2, TF SAME pads, odd sizes), the group0 identity shortcut, the
weight manifest and the importer's refusals both ways, the backbone flags of the reference CLI and their precedence, the
flags the block ignores, ResNeXt winning over it, the ABI field, the synthetic weights of existing seeds and bounded
synthetic activations."""
import hashlib

import numpy as np
import pytest
import torch

from object_detection_tracking_b200.config import make_config, normalize_config
from object_detection_tracking_b200.synth import frcnn_weight_shapes, synth_frame, synth_weights
import basic_block_oracle
from oracle import frcnn

R18 = dict(resnet_num_block=(2, 2, 2, 2), use_basic_block=True)
R34 = dict(resnet_num_block=(3, 4, 6, 3), use_basic_block=True)
SMALL = dict(resnet_num_block=(1, 2, 1, 1), use_basic_block=True)
F32 = np.float32


def np_conv3x3(x, w, stride, pad):
    """float64 loop over the taps: NCHW x, HWIO w [3, 3, cin, cout], pad = (top, bottom, left, right)."""
    n, c, h, wd = x.shape
    pt, pb, pl, pr = pad
    xp = np.zeros((n, c, h + pt + pb, wd + pl + pr))
    xp[:, :, pt:pt + h, pl:pl + wd] = x
    ho = (h + pt + pb - 3) // stride + 1
    wo = (wd + pl + pr - 3) // stride + 1
    out = np.zeros((n, w.shape[3], ho, wo))
    for r in range(3):
        for s in range(3):
            win = xp[:, :, r:r + (ho - 1) * stride + 1:stride, s:s + (wo - 1) * stride + 1:stride]
            out += np.einsum("nchw,co->nohw", win, w[r, s].astype(np.float64))
    return out


def np_bn(x, W, name):
    g, b = W[name + "/bn/gamma"].astype(np.float64), W[name + "/bn/beta"].astype(np.float64)
    m, v = W[name + "/bn/mean/EMA"].astype(np.float64), W[name + "/bn/variance/EMA"].astype(np.float64)
    inv = g / np.sqrt(v + frcnn.BN_EPS)
    return x * inv[None, :, None, None] + (b - m * inv)[None, :, None, None]


def np_basic_block(x, W, p, ch, stride):
    """relu(bn(conv2(relu(bn(conv1(x))))) + shortcut), TF SAME written out: at stride 2 the total pad of an n-wide axis is
    1 on even n (all of it bottom / right) and 2 on odd n (one each side)."""
    def same(n):
        if stride == 1:
            return (1, 1)
        total = 1 if n % 2 == 0 else 2
        return (total // 2, total - total // 2)
    pad = same(x.shape[2]) + same(x.shape[3])
    relu = lambda a: np.maximum(a, 0)
    l = relu(np_bn(np_conv3x3(x, W[p + "/conv1/W"], stride, pad), W, p + "/conv1"))
    l = np_bn(np_conv3x3(l, W[p + "/conv2/W"], 1, (1, 1, 1, 1)), W, p + "/conv2")
    sc = x
    if x.shape[1] != ch:
        xs = x[:, :, :-1:stride, :-1:stride] if stride == 2 else x
        sc = np_bn(np.einsum("nchw,co->nohw", xs, W[p + "/convshortcut/W"][0, 0].astype(np.float64)), W,
                   p + "/convshortcut")
    return relu(l + sc)


def _block_weights(rng, cin, ch):
    W = {}
    W["b/conv1/W"] = (rng.standard_normal((3, 3, cin, ch)) * np.sqrt(2.0 / (9 * cin))).astype(F32)
    W["b/conv2/W"] = (rng.standard_normal((3, 3, ch, ch)) * np.sqrt(2.0 / (9 * ch))).astype(F32)
    names = ["b/conv1", "b/conv2"]
    if cin != ch:
        W["b/convshortcut/W"] = (rng.standard_normal((1, 1, cin, ch)) / np.sqrt(cin)).astype(F32)
        names.append("b/convshortcut")
    for n in names:
        W[n + "/bn/gamma"] = rng.uniform(0.5, 1.5, ch).astype(F32)
        W[n + "/bn/beta"] = (rng.standard_normal(ch) * 0.1).astype(F32)
        W[n + "/bn/mean/EMA"] = (rng.standard_normal(ch) * 0.1).astype(F32)
        W[n + "/bn/variance/EMA"] = rng.uniform(0.5, 1.5, ch).astype(F32)
    return W


@pytest.mark.parametrize("h,w", [(12, 10), (11, 13), (8, 9)])
@pytest.mark.parametrize("cin,ch,stride", [(8, 8, 1), (4, 8, 2), (8, 16, 1)])
def test_oracle_block_matches_numpy_loop(h, w, cin, ch, stride):
    rng = np.random.default_rng(h * 100 + w + 7 * stride + cin)
    W = _block_weights(rng, cin, ch)
    x = rng.standard_normal((2, cin, h, w))
    if stride == 2 and (h % 2 or w % 2):
        # conv1's SAME output is ceil(n / 2), the shortcut's n // 2: the reference's sum fails on an odd axis, and so does
        # the oracle's (the backbone only sees even sizes there: its input is padded to a multiple of 32)
        with frcnn.exact(), pytest.raises(RuntimeError, match="size of tensor"):
            basic_block_oracle.basic_block(torch.from_numpy(x), W, "b", ch, stride, False)
        return
    with frcnn.exact():
        got = basic_block_oracle.basic_block(torch.from_numpy(x), W, "b", ch, stride, False).numpy()
    ref = np_basic_block(x, W, "b", ch, stride)
    assert got.shape == ref.shape == (2, ch, -(-h // stride), -(-w // stride))
    assert np.abs(got - ref).max() < 1e-12 * np.abs(ref).max()


@pytest.mark.parametrize("h,w", [(11, 13), (8, 9), (12, 10)])
def test_oracle_stride2_conv1_matches_numpy_loop_at_odd_sizes(h, w):
    """conv1 alone at stride 2: SAME pads 1 / 1 on an odd axis and 0 / 1 on an even one."""
    rng = np.random.default_rng(h * 10 + w)
    k = rng.standard_normal((3, 3, 4, 8))
    x = rng.standard_normal((1, 4, h, w))
    from resnext_oracle import same_pads
    pad = same_pads(h, 3, 2, 1) + same_pads(w, 3, 2, 1)
    assert pad == ((1, 1) if h % 2 else (0, 1)) + ((1, 1) if w % 2 else (0, 1))
    with frcnn.exact():
        got = frcnn._conv(torch.from_numpy(x), k, stride=2, pad=pad).numpy()
    ref = np_conv3x3(x, k, 2, pad)
    assert got.shape == ref.shape == (1, 8, -(-h // 2), -(-w // 2))
    assert np.abs(got - ref).max() < 1e-12 * np.abs(ref).max()


@pytest.mark.parametrize("n,pads", [(184, (0, 1)), (46, (0, 1)), (45, (1, 1)), (7, (1, 1))])
def test_stride2_same_pads_put_the_odd_pad_bottom_right(n, pads):
    from resnext_oracle import same_pads
    assert same_pads(n, 3, 2, 1) == pads
    assert (n + sum(pads) - 3) // 2 + 1 == -(-n // 2)


def test_stride2_pad_is_observable():
    """The basic block's SAME pad (0 top / 1 bottom) against the bottleneck's explicit [1, 0]: other numbers, same size."""
    rng = np.random.default_rng(3)
    x = rng.standard_normal((1, 4, 12, 16))
    k = rng.standard_normal((3, 3, 4, 8))
    same = np_conv3x3(x, k, 2, (0, 1, 0, 1))
    tfpad = np_conv3x3(x, k, 2, (1, 0, 1, 0))
    assert same.shape == tfpad.shape and np.abs(same - tfpad).max() > 0.1


def test_group0_block0_has_an_identity_shortcut():
    """The pool output has 64 channels and ch_out is 64: no convshortcut, the block adds its input."""
    rng = np.random.default_rng(5)
    W = _block_weights(rng, 64, 64)
    assert "b/convshortcut/W" not in W
    x = torch.from_numpy(np.abs(rng.standard_normal((1, 64, 9, 10))))
    with frcnn.exact():
        got = basic_block_oracle.basic_block(x, W, "b", 64, 1, False)
        branch = frcnn._bn(frcnn._conv(torch.relu(frcnn._bn(frcnn._conv(x, W["b/conv1/W"], pad=(1, 1, 1, 1)), W, "b/conv1")),
                                       W["b/conv2/W"], pad=(1, 1, 1, 1)), W, "b/conv2")
    assert torch.equal(got, torch.relu(branch + x))
    for cfg in (make_config(**R18), make_config(**R34)):
        sh = frcnn_weight_shapes(cfg)
        assert "group0/block0/convshortcut/W" not in sh
        assert [k for k in sh if "convshortcut/W" in k] == ["group%d/block0/convshortcut/W" % g for g in (1, 2, 3)]


@pytest.mark.parametrize("blocks", [(2, 2, 2, 2), (3, 4, 6, 3)], ids=["r18", "r34"])
@pytest.mark.parametrize("gn", [False, True], ids=["bn", "gn"])
def test_manifest_lists_the_basic_block_shapes(blocks, gn):
    cfg = make_config(resnet_num_block=blocks, use_basic_block=True, use_gn=gn)
    sh = frcnn_weight_shapes(cfg)
    w = synth_weights(cfg, 11)
    assert sorted(sh) == sorted(w)
    for k, v in w.items():
        assert tuple(v.shape) == tuple(sh[k]), k
    norm = ("gn/gamma", "gn/beta") if gn else ("bn/gamma", "bn/beta", "bn/mean/EMA", "bn/variance/EMA")
    cin, nconv = 64, 0
    for g, (ch, count) in enumerate(zip((64, 128, 256, 512), blocks)):
        for i in range(count):
            p = "group%d/block%d" % (g, i)
            assert sh[p + "/conv1/W"] == (3, 3, cin, ch)
            assert sh[p + "/conv2/W"] == (3, 3, ch, ch)
            for conv in ("conv1", "conv2") + (("convshortcut",) if cin != ch else ()):
                for n in norm:
                    assert sh["%s/%s/%s" % (p, conv, n)] == (ch,)
            assert (p + "/convshortcut/W" in sh) == (cin != ch)
            assert not any(k.startswith(p + "/conv3/") for k in sh)
            cin = ch
            nconv += 2
    assert 1 + nconv + 1 == {(2, 2, 2, 2): 18, (3, 4, 6, 3): 34}[blocks]        # conv0 + the blocks + the classifier
    for i, c in enumerate((64, 128, 256, 512)):
        assert sh["fpn/lateral_1x1_c%d/W" % (i + 2)] == (1, 1, c, 256)
    base = dict(resnet_num_block=blocks, use_gn=gn)
    rest = lambda s: {k: v for k, v in s.items() if not k.startswith(("group", "fpn/lateral"))}
    assert rest(sh) == rest(frcnn_weight_shapes(make_config(**base)))       # nothing past the backbone changes


def test_check_weights_refuses_the_other_block_by_name():
    from object_detection_tracking_b200.backend import check_weights
    basic, bottle = make_config(**R34), make_config(resnet_num_block=(3, 4, 6, 3))
    check_weights(basic, synth_weights(basic, 5))
    check_weights(bottle, synth_weights(bottle, 5))
    with pytest.raises(ValueError) as e:                      # a bottleneck checkpoint under --resnet34
        check_weights(basic, synth_weights(bottle, 5))
    msg = str(e.value)
    assert "mis-shaped" in msg and "group0/block0/conv1/W" in msg and "fpn/lateral_1x1_c2/W" in msg
    with pytest.raises(ValueError) as e:                      # a basic checkpoint under --resnet50: no conv3
        check_weights(bottle, synth_weights(basic, 5))
    assert "group0/block0/conv3/W" in str(e.value) and "group0/block0/convshortcut/W" in str(e.value)


def _reference_table(flags):
    """obj_detect_tracking.py:348-359 as written."""
    blocks, basic = [3, 4, 23, 3], False
    if flags.get("resnet152"):
        blocks = [3, 8, 36, 3]
    if flags.get("resnet50"):
        blocks = [3, 4, 6, 3]
    if flags.get("resnet34"):
        blocks, basic = [3, 4, 6, 3], True
    if flags.get("resnet18"):
        blocks, basic = [2, 2, 2, 2], True
    return tuple(blocks), basic


FLAGS = ("resnet152", "resnet50", "resnet34", "resnet18")


@pytest.mark.parametrize("mask", range(16))
def test_backbone_flags_follow_the_reference_table(mask):
    flags = {f: bool(mask >> k & 1) for k, f in enumerate(FLAGS)}
    ns = type("Args", (), {})()                          # a reference-style namespace: the flags, nothing derived
    for k, v in flags.items():
        setattr(ns, k, v)
    cfg = normalize_config(ns)
    assert (cfg.resnet_num_block, bool(cfg.use_basic_block)) == _reference_table(flags)
    assert (make_config(**flags).resnet_num_block, bool(make_config(**flags).use_basic_block)) == _reference_table(flags)


def test_backbone_flags_change_only_what_they_name():
    assert make_config(resnet152=True).resnet_num_block == (3, 8, 36, 3)          # was ResNet-101 before
    assert make_config(resnet_num_block=(1, 1, 2, 1)).use_basic_block is False
    assert make_config(resnet_num_block=(1, 2, 1, 1), use_basic_block=True).use_basic_block is True
    cfg = make_config(resnet34=True)
    assert normalize_config(cfg) is cfg and cfg.resnet_num_block == (3, 4, 6, 3) and cfg.use_basic_block


@pytest.mark.parametrize("blocks", [(2, 2, 2, 2), (3, 4, 6, 3)])
@pytest.mark.parametrize("gn", [False, True])
def test_se_deformable_and_dilations_are_ignored(blocks, gn):
    base = dict(resnet_num_block=blocks, use_basic_block=True, use_gn=gn, use_dilations=False)
    ref_sh = frcnn_weight_shapes(make_config(**base))
    ref_w = synth_weights(make_config(**base), 9)
    for extra in (dict(use_se=True), dict(use_deformable=True), dict(use_dilations=True),
                  dict(use_deformable=True, use_dilations=True, use_se=True)):
        cfg = make_config(**dict(base, **extra))
        assert frcnn_weight_shapes(cfg) == ref_sh, extra
        w = synth_weights(cfg, 9)
        assert sorted(w) == sorted(ref_w) and all(w[k].tobytes() == ref_w[k].tobytes() for k in w), extra


def test_resnext_wins_over_the_basic_block():
    rx = dict(resnet_num_block=(1, 2, 1, 1), use_resnext=True)
    assert frcnn_weight_shapes(make_config(use_basic_block=True, **rx)) == frcnn_weight_shapes(make_config(**rx))
    a, b = synth_weights(make_config(use_basic_block=True, **rx), 4), synth_weights(make_config(**rx), 4)
    assert sorted(a) == sorted(b) and all(a[k].tobytes() == b[k].tobytes() for k in a)
    assert not basic_block_oracle.use_basic(make_config(use_basic_block=True, **rx))


def test_config_and_abi_carry_use_basic_block():
    """use_basic_block travels in b2_config_ext through b2_create_ex; b2_config keeps its layout (use_deformable last, 196
    bytes), so a b2_config written against the previous header stays valid."""
    import ctypes
    from object_detection_tracking_b200 import _lib
    from test_abi import _header_struct_words
    assert make_config().use_basic_block is False
    assert _lib.make_config_ext(make_config()).use_basic_block == 0
    assert _lib.make_config_ext(make_config(resnet18=True)).use_basic_block == 1
    # the flag is passed as set; the engine lets use_resnext win over it
    assert _lib.make_config_ext(make_config(resnet34=True, use_resnext=True)).use_basic_block == 1
    assert _lib.B2Config._fields_[-1] == ("use_deformable", _lib.c_int32)
    assert ctypes.sizeof(_lib.B2Config) == 196 == 4 * _header_struct_words("b2_config")
    assert _lib.B2ConfigExt._fields_ == [("use_basic_block", _lib.c_int32)]
    assert ctypes.sizeof(_lib.B2ConfigExt) == 4 * _header_struct_words("b2_config_ext")
    assert dict((n, a) for n, _, a in _lib.SYMBOLS)["b2_create_ex"][2:] == [ctypes.POINTER(_lib.B2Config),
                                                                           ctypes.POINTER(_lib.B2ConfigExt)]


def test_create_ex_fails_loudly_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from object_detection_tracking_b200.engine import Detector
    with pytest.raises(RuntimeError, match="b2_create"):
        Detector(make_config(resnet18=True), 1, 64, 64)


# sha256 (first 16 hex digits) over the sorted names and bytes of synth_weights(cfg, 1234), as before use_basic_block existed
SEED_DIGESTS = {
    "resnext": (dict(use_resnext=True), "e946c08411b07616"),
    "relation": (dict(add_relation_nn=True), "ca2265f9aece29a9"),
    "deformable": (dict(use_deformable=True, use_dilations=False, version=2), "60ec43d391841838"),
    "r50_gn": (dict(resnet_num_block=(3, 4, 6, 3), use_gn=True), "703e54807290307f"),
    "r50_se_deform": (dict(resnet_num_block=(3, 4, 6, 3), use_se=True, use_deformable=True, use_dilations=False),
                      "d4636af6f900f8b9"),
    "small_gn_mask": (dict(resnet_num_block=(1, 1, 2, 1), use_gn=True, add_mask=True, use_frcnn_class_agnostic=True),
                      "71465ca0df6c13cf"),
}


@pytest.mark.parametrize("name", sorted(SEED_DIGESTS))
def test_existing_seeds_are_unchanged(name):
    kw, digest = SEED_DIGESTS[name]
    w = synth_weights(make_config(**kw), 1234)
    h = hashlib.sha256()
    for k in sorted(w):
        h.update(k.encode())
        h.update(w[k].tobytes())
    assert h.hexdigest()[:16] == digest


@pytest.mark.parametrize("flags", [dict(resnet34=True), dict(resnet18=True), dict(resnet34=True, use_gn=True)],
                         ids=["r34", "r18", "r34_gn"])
def test_synthetic_basic_activations_stay_bounded(flags):
    """The basic backbone on the synthetic weights keeps c2..c5 O(1): well inside the fp16 planes' range, and not dead."""
    cfg = make_config(max_size=256, short_edge_size=192, **flags)
    Wt = synth_weights(cfg, 1234)
    x = frcnn.preprocess(synth_frame(192, 256, 3).astype(F32))
    feats = basic_block_oracle.backbone(x, Wt, cfg)
    assert [f.shape[1] for f in feats] == [64, 128, 256, 512]
    assert [tuple(f.shape[2:]) for f in feats] == [(48, 64), (24, 32), (12, 16), (6, 8)]
    for f in feats:
        a = float(f.abs().max())
        assert 0.1 < a < 100.0, a
        assert float((f > 0).float().mean()) > 0.05


def test_oracle_is_frcnn_without_the_flag_and_restores_it():
    cfg = make_config(resnet_num_block=(1, 1, 1, 1), max_size=128, short_edge_size=96)
    Wt = synth_weights(cfg, 2)
    frame = synth_frame(96, 128, 1).astype(F32)
    before = (frcnn.backbone, frcnn.fpn, frcnn.fastrcnn_head)
    a = frcnn.forward(cfg, Wt, frame, stages=False)
    b = basic_block_oracle.forward(cfg, Wt, frame, stages=False)
    for k in ("final_boxes", "final_probs", "final_labels", "fpn_box_feat"):
        np.testing.assert_array_equal(a[k], b[k])
    bcfg = make_config(resnet_num_block=(1, 1, 1, 1), max_size=128, short_edge_size=96, use_basic_block=True)
    r = basic_block_oracle.forward(bcfg, synth_weights(bcfg, 2), frame)
    assert (frcnn.backbone, frcnn.fpn, frcnn.fastrcnn_head) == before
    assert [c.shape[-3] for c in r["c2345"]] == [64, 128, 256, 512] and len(r["final_boxes"]) > 0
