"""The ResNet stems' ingest on the GPU against tests/stem_oracle.py, in split and fp16 precision.

* The packs alone (b2_op_stem_pack), bit for bit in every element -- padding region and zero lanes included: the
  detector's compact 16-lane operand and the ReID engines' 64-lane operand, frames from 1x1 to 720x1280, B = 1 and 3
  (each image against itself packed alone), operands at the engines' sizes and larger, uint8 against the same integral
  float32 frame, and float32 frames with non-integral, negative and above-255 values.
* conv0 through the detector (set_stage("image") + run_phases(1)): c1 element-wise within the float64 stem's bound, the
  rows and columns that read only padding exactly relu(BN shift), the max-pool of the engine's own c1 bit for bit, and
  the GroupNorm stem.
* conv1 through both ReID models: the operand bit for bit and conv1 within the bound."""
import os

import numpy as np
import pytest

import elementwise_oracle as eo
import stem_oracle as so

pytestmark = pytest.mark.gpu

SIZES = [(1, 1), (2, 3), (7, 7), (13, 17), (193, 257), (200, 300), (720, 1280)]
PRECISIONS = pytest.mark.parametrize("split", [True, False], ids=["split", "fp16"])


def _engine():
    from object_detection_tracking_b200 import engine
    return engine


def _frames(B, H, W, seed):
    """uint8 frames [B][H][W][3] of uniform bytes with an all-0 block and an all-255 block in every image."""
    rng = np.random.default_rng(seed)
    f = rng.integers(0, 256, (B, H, W, 3)).astype(np.uint8)
    f[:, : (H + 2) // 3, : (W + 2) // 3] = 0
    f[:, H - H // 3:, W - W // 3:] = 255
    return f


def det_operand_hw(H, W):
    c1h, c1w = so.out_hw(H, W, so.detector_pads(H, W))
    return c1h + 3, c1w + 3                    # engine.cu: stem_u [B][c1h + 3][c1w + 3][16]


def reid_operand_hw(H, W):
    h1, w1 = so.out_hw(H, W, so.REID_PADS)
    return h1 + 3, w1                          # reid_engine.cu: stem_u [B][h1 + 3][w1][64]


def _pack(frames, layout, hw, split):
    return _engine().op_stem_pack(frames, layout, hw, split=split)


def assert_planes(hi, lo, P, split, what):
    """Raw planes equal those of the fp32 operand P in every element."""
    eh, el = so.raw_planes(P, split)
    bad = np.argwhere(hi != eh)
    assert bad.size == 0, "%s: hi differs at %d elements, first %s" % (what, len(bad), tuple(bad[0]))
    if split:
        bad = np.argwhere(lo != el)
        assert bad.size == 0, "%s: lo differs at %d elements, first %s" % (what, len(bad), tuple(bad[0]))


# ==== the packs alone ================================================================================================
LAYOUTS = {"detector": (so.pack16, det_operand_hw, 12), "reid": (so.pack64, reid_operand_hw, 48)}


@pytest.mark.parametrize("layout", sorted(LAYOUTS))
@pytest.mark.parametrize("H,W", SIZES)
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("extra", [(0, 0), (2, 5)], ids=["engine_size", "larger"])
@PRECISIONS
def test_pack_bit_exact(layout, H, W, B, extra, split):
    pack, hw_of, live = LAYOUTS[layout]
    Hu, Wx = hw_of(H, W)
    Hu, Wx = Hu + extra[0], Wx + extra[1]
    frames = _frames(B, H, W, H * 7919 + W * 31 + B)
    out, hi, lo = _pack(frames, layout, (Hu, Wx), split)
    P = pack(so.normalize(frames, layout), Hu, Wx)
    assert_planes(hi, lo, P, split, "%s %dx%d B=%d operand %dx%d" % (layout, H, W, B, Hu, Wx))
    np.testing.assert_array_equal(out, eo.value(*eo.planes(P, split)))
    assert not hi[..., live:].any() and (lo is None or not lo[..., live:].any()), "zero lanes"
    if extra != (0, 0):
        # rows past the engine's operand read only the bottom padding; so do the detector's columns past Wv, while a ReID
        # column q >= w1 still reads frame columns 2q - 3 .. 2q + 4
        h0, w0 = hw_of(H, W)
        assert not hi[:, h0:].any(), "the rows past the engine's operand are not zero"
        assert layout == "reid" or not hi[:, :, w0:].any(), "the columns past the engine's operand are not zero"
    if B > 1:
        for b in range(B):
            _, hb, lb = _pack(frames[b:b + 1], layout, (Hu, Wx), split)
            np.testing.assert_array_equal(hi[b:b + 1], hb)
            if split:
                np.testing.assert_array_equal(lo[b:b + 1], lb)


@pytest.mark.parametrize("H,W", [(1, 1), (13, 17), (200, 300), (720, 1280)])
@PRECISIONS
def test_detector_uint8_and_integral_float32_frames_give_the_same_operand(H, W, split):
    frames = _frames(2, H, W, H + W)
    hw = det_operand_hw(H, W)
    _, h8, l8 = _pack(frames, "detector", hw, split)
    _, hf, lf = _pack(frames.astype(np.float32), "detector", hw, split)
    np.testing.assert_array_equal(h8, hf)
    if split:
        np.testing.assert_array_equal(l8, lf)


@pytest.mark.parametrize("H,W", [(2, 3), (13, 17), (193, 257)])
@PRECISIONS
def test_detector_float32_frames_of_any_value(H, W, split):
    """The detector's float32 placeholder takes any float: non-integral, negative, above 255, -0 and values whose
    normalisation reaches the fp16 limits of the planes."""
    rng = np.random.default_rng(H * W)
    frames = rng.uniform(-300, 600, (2, H, W, 3)).astype(np.float32)
    special = np.array([0.5, -0.0, 255.5, -1e-3, 1e4, -1e4, 3.1e3, 1e-30, 254.99998], np.float32)
    flat = frames.reshape(-1)
    flat[:min(flat.size, special.size)] = special[:flat.size]
    hw = det_operand_hw(H, W)
    _, hi, lo = _pack(frames, "detector", hw, split)
    assert_planes(hi, lo, so.pack16(so.normalize(frames, "detector"), *hw), split, "float32 %dx%d" % (H, W))


def test_pack_refuses_bad_arguments():
    e = _engine()
    f8 = np.zeros((1, 4, 4, 3), np.uint8)
    with pytest.raises(RuntimeError, match="uint8 crops only"):
        e.op_stem_pack(f8.astype(np.float32), "reid", (5, 2))
    with pytest.raises(RuntimeError, match="positive sizes"):
        e.op_stem_pack(f8, "detector", (0, 4))
    from object_detection_tracking_b200 import _lib
    out = np.zeros(16, np.float32)   # refused before anything is written
    with pytest.raises(RuntimeError, match="too large"):
        _lib.check(_lib.load().b2_op_stem_pack(0, _lib.ptr(f8), 1, 1, 4, 4, 0, 1 << 16, 1 << 16, 1, _lib.ptr(out),
                                               None, None), "b2_op_stem_pack")


# ==== conv0 through the detector =====================================================================================
def _detector(H, W, input_dtype, split, use_gn=False, seed=77):
    from object_detection_tracking_b200.config import make_config
    from object_detection_tracking_b200.engine import Detector
    from object_detection_tracking_b200.synth import synth_weights
    cfg = make_config(resnet_num_block=(1, 1, 2, 1), max_size=max(H, W), short_edge_size=min(H, W), use_gn=use_gn)
    Wt = synth_weights(cfg, seed)
    det = Detector(cfg, 1, H, W, input_dtype=input_dtype, precision="split" if split else "fp16", use_cuda_graph=False)
    det.load_weights(Wt)
    return det, Wt


def _run_stem(det, frame, input_dtype):
    det.set_stage("image", frame[None].astype(np.uint8 if input_dtype == "uint8" else np.float32))
    det.run_phases(1)
    return det.get_stage("c1").astype(np.float64), det.get_stage("pool")


def assert_within(got, o, what):
    err = np.abs(got - o["ref"])
    assert np.isfinite(got).all(), what + ": non-finite output"
    worst = np.unravel_index(np.argmax(err - o["bound"]), err.shape)
    assert (err <= o["bound"]).all(), "%s: element %s |err| %.3g > bound %.3g (ref %.6g)" % (
        what, worst, err[worst], o["bound"][worst], o["ref"][worst])


def assert_pool_of(c1, pool, what):
    c1h, c1w = c1.shape[1:3]
    assert pool.shape[1:3] == ((c1h - 2) // 2 + 1, (c1w - 2) // 2 + 1), pool.shape   # engine.cu ch[0] x cw[0]
    ref = eo.maxpool_stem(c1, pool.shape[1:3]).astype(np.float32)
    np.testing.assert_array_equal(pool.view(np.uint32), ref.view(np.uint32), err_msg=what)


@pytest.mark.parametrize("H,W", [(192, 256), (200, 300), (193, 257), (720, 1280)])
@pytest.mark.parametrize("input_dtype", ["uint8", "float32"])
@PRECISIONS
def test_detector_conv0_within_the_float64_stem_bound(H, W, input_dtype, split):
    det, Wt = _detector(H, W, input_dtype, split)
    try:
        frame = _frames(1, H, W, H * W)[0]
        c1, pool = _run_stem(det, frame, input_dtype)
    finally:
        det.close()
    pads = so.detector_pads(H, W)
    o = so.stem_conv64(frame[None], Wt["conv0/W"], so.det_bn(Wt), pads, "detector", split)
    assert c1.shape == o["ref"].shape, (c1.shape, o["ref"].shape)
    what = "conv0 %dx%d %s %s" % (H, W, input_dtype, "split" if split else "fp16")
    assert_within(c1, o, what)
    # a window of padding alone sums to exactly 0: the output is the stored relu(fp32 BN shift)
    rows, cols = so.padding_only(H, W, pads, c1.shape[1:3])
    edge = eo.value(*eo.planes(np.maximum(o["shift32"], np.float32(0)), split)).astype(np.float64)
    assert (c1[:, rows] == edge).all() and (c1[:, :, cols] == edge).all(), what + ": padding-only rows / columns"
    assert_pool_of(c1.astype(np.float32), pool, what)


@PRECISIONS
def test_detector_groupnorm_stem(split):
    """use_gn: c1 is GroupNorm + ReLU of the conv without bias.  The conv's bound is carried through the normalisation to
    first order: with |dy| <= e in a group of standard deviation sigma, |d yhat| <= (e_i + mean e + 2 |yhat_i| max e) /
    sigma; the GroupNorm's own arithmetic is allowed what test_groupnorm_gpu allows it."""
    from test_groupnorm_gpu import ref_gn
    H, W = 200, 300
    det, Wt = _detector(H, W, "uint8", split, use_gn=True)
    try:
        frame = _frames(1, H, W, 5)[0]
        c1, pool = _run_stem(det, frame, "uint8")
    finally:
        det.close()
    o = so.stem_conv64(frame[None], Wt["conv0/W"], None, so.detector_pads(H, W), "detector", split, relu=False)
    gamma, beta = Wt["conv0/gn/gamma"].astype(np.float64), Wt["conv0/gn/beta"].astype(np.float64)
    ref = ref_gn(o["pre"], gamma, beta, relu=True)
    B, h, w, C = o["pre"].shape
    g = o["pre"].reshape(B, h * w, 32, C // 32)
    e = o["bound"].reshape(g.shape)
    mu, sigma = g.mean(axis=(1, 3), keepdims=True), g.std(axis=(1, 3), keepdims=True)
    yhat = (g - mu) / sigma
    tol = (e + e.mean(axis=(1, 3), keepdims=True) + 2 * np.abs(yhat) * e.max(axis=(1, 3), keepdims=True)) / sigma
    tol = tol.reshape(o["pre"].shape) * np.abs(gamma) * 1.01 + (2e-6 if split else 1.5e-3) * np.abs(ref).max()
    err = np.abs(c1 - ref)
    worst = np.unravel_index(np.argmax(err - tol), err.shape)
    assert (err <= tol).all(), "GN stem: element %s |err| %.3g > %.3g" % (worst, err[worst], tol[worst])
    assert_pool_of(c1.astype(np.float32), pool, "GN stem")


# ==== conv1 through the ReID engines =================================================================================
REID = {"osnet_x1_0": ("osnet.npz", "synth_osnet_state", 4321, "conv1.conv.weight", "conv1.bn"),
        "resnet101": ("resnet101_reid.npz", "synth_resnet101_reid_state", 2468, "conv1.weight", "bn1")}


@pytest.mark.parametrize("model", sorted(REID))
@PRECISIONS
def test_reid_stem_operand_and_conv1(model, split, golden_dir):
    from object_detection_tracking_b200 import synth
    from object_detection_tracking_b200.reid import ReidEngine
    npz, state_fn, seed, wname, bn = REID[model]
    resized = np.load(os.path.join(golden_dir, npz))["resized"]
    crops = np.concatenate([resized, np.zeros_like(resized[:1]), np.full_like(resized[:1], 255)])
    state = getattr(synth, state_fn)(seed)
    eng = ReidEngine(batch=len(crops), precision="split" if split else "fp16", model=model)
    try:
        eng.load_state(state)
        eng.embed(crops)
        u = eng.get_activation("stem_u")
        c1 = eng.get_activation("conv1").astype(np.float64)
    finally:
        eng.close()
    H, W = crops.shape[1:3]
    U = so.pack64(so.normalize(crops, "reid"), *reid_operand_hw(H, W))
    np.testing.assert_array_equal(u.view(np.uint32), eo.value(*eo.planes(U, split)).view(np.uint32))
    o = so.stem_conv64(crops, so.oihw_to_hwio(state[wname]), so.torch_bn(state, bn), so.REID_PADS, "reid", split)
    assert c1.shape == o["ref"].shape, (c1.shape, o["ref"].shape)
    assert_within(c1, o, "%s conv1 %s" % (model, "split" if split else "fp16"))
