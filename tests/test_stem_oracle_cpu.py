"""Pins tests/stem_oracle.py: the normalisations against oracle/frcnn.py's preprocess and torch, the packs convolved with
restatements of the engines' two weight re-indexings against the float64 7x7/2 conv, and that conv against
oracle/frcnn.py's backbone conv0 step."""
import numpy as np
import pytest
import torch

import stem_oracle as so

SIZES = [(1, 1), (2, 3), (7, 7), (13, 17), (193, 257), (200, 300)]


def _frames(B, H, W, seed, dtype=np.uint8):
    rng = np.random.default_rng(seed)
    f = rng.integers(0, 256, (B, H, W, 3))
    if B > 1:
        f[0, : H // 2] = 0                      # flat regions at both ends of the byte range
        f[-1, H // 2:] = 255
    return f.astype(dtype)


def test_detector_normalize_is_the_oracle_preprocess_bit_for_bit():
    from oracle import frcnn
    every = np.arange(256, dtype=np.float32)
    frame = np.stack(np.meshgrid(every, every, indexing="ij"), -1)[..., [0, 1, 0]]   # every byte in every channel
    frame = np.concatenate([frame, np.array([[[-3.5, 0.25, 1e3]] * 256], np.float32)])  # the float32 input accepts any
    ref = frcnn.preprocess(frame)[0].permute(1, 2, 0).numpy()
    got = so.normalize(frame, "detector")
    assert got.dtype == np.float32
    np.testing.assert_array_equal(got.view(np.uint32), ref.view(np.uint32))


def test_reid_normalize_is_torch_totensor_normalize_bit_for_bit():
    x = np.arange(256, dtype=np.uint8)[:, None, None].repeat(3, 2).repeat(2, 1)
    t = torch.from_numpy(x.astype(np.float32)).div(255)
    ref = t.sub(torch.tensor(so.REID_MEAN)).div(torch.tensor(so.REID_STD)).numpy()
    got = so.normalize(x, "reid")
    np.testing.assert_array_equal(got.view(np.uint32), ref.view(np.uint32))


def test_the_two_normalisations_differ_where_the_kernels_must_not_mix_them():
    """x * float32(1/255) and x / 255 differ for many byte values: a kernel using the other one's rounding fails the
    bit-exact pack tests."""
    x = np.arange(256, dtype=np.float32)
    assert int((x * np.float32(1 / 255) != x / np.float32(255)).sum()) > 100


def test_packs_follow_the_index_formulas():
    rng = np.random.default_rng(3)
    P = rng.standard_normal((2, 9, 11, 3))
    V, U = so.pack16(P, 8, 9), so.pack64(P, 8, 6)
    for b, y, x, j in np.ndindex(V.shape):
        ry, sx, c = j // 6, j % 6 // 3, j % 3
        iy, ix = 2 * y + ry - 3, 2 * x + sx - 3
        want = P[b, iy, ix, c] if j < 12 and 0 <= iy < 9 and 0 <= ix < 11 else 0.0
        assert V[b, y, x, j] == want
    for b, y, q, k in np.ndindex(U.shape):
        s, ry, sx, c = k // 12, k % 12 // 6, k % 6 // 3, k % 3
        iy, ix = 2 * y + ry - 3, 2 * (q + s) + sx - 3
        want = P[b, iy, ix, c] if k < 48 and 0 <= iy < 9 and 0 <= ix < 11 else 0.0
        assert U[b, y, q, k] == want


def _weights(seed, Cout=64):
    rng = np.random.default_rng(seed)
    W = (rng.standard_normal((7, 7, 3, Cout)) * 0.1).astype(np.float32)
    bn = (rng.uniform(0.5, 1.5, Cout).astype(np.float32), (rng.standard_normal(Cout) * 0.1).astype(np.float32),
          (rng.standard_normal(Cout) * 0.1).astype(np.float32), rng.uniform(0.5, 1.5, Cout).astype(np.float32), 1e-5)
    return W, bn


def det_weight_pack(W):
    """detplan.cu's kStem re-indexing restated: W'[o][r][s*16 + ry*6 + sx*3 + c] = W[2r + ry][2s + sx][c][o], zero for
    lanes 12..15 of each width tap and for taps 2r + ry == 7 or 2s + sx == 7."""
    Cout = W.shape[3]
    out = np.zeros((Cout, 4, 64))
    for r in range(4):
        for s in range(4):
            for ry in range(2):
                for sx in range(2):
                    if 2 * r + ry < 7 and 2 * s + sx < 7:
                        out[:, r, s * 16 + ry * 6 + sx * 3:s * 16 + ry * 6 + sx * 3 + 3] = W[2 * r + ry, 2 * s + sx].T
    return out


def reid_weight_pack(w_oihw):
    """reid_engine.cu's kStem re-indexing restated: W'[o][r][s*12 + ry*6 + sx*3 + c] = w[o][c][2r + ry][2s + sx]."""
    Cout = w_oihw.shape[0]
    out = np.zeros((Cout, 4, 64))
    for r in range(4):
        for s in range(4):
            for ry in range(2):
                for sx in range(2):
                    if 2 * r + ry < 7 and 2 * s + sx < 7:
                        out[:, r, s * 12 + ry * 6 + sx * 3:s * 12 + ry * 6 + sx * 3 + 3] = w_oihw[:, :, 2 * r + ry, 2 * s + sx]
    return out


def conv_detector_operand(V, Wp, Ho, Wo):
    """conv0 as engine.cu runs it: a 4x1 VALID conv whose 64-channel pixel (p, q) is V[p][q .. q+3][0..15]."""
    acc = 0.0
    for r in range(4):
        win = np.concatenate([V[:, r:r + Ho, s:s + Wo] for s in range(4)], -1)   # [B][Ho][Wo][64]
        acc = acc + win @ Wp[:, r].T
    return acc


def conv_reid_operand(U, Wp, Ho):
    acc = 0.0
    for r in range(4):
        acc = acc + U[:, r:r + Ho] @ Wp[:, r].T
    return acc


@pytest.mark.parametrize("H,W", SIZES)
def test_detector_pack_times_restated_weights_is_the_float64_stem(H, W):
    frames = _frames(2, H, W, H * 1000 + W)
    Wt, bn = _weights(H + W)
    pads = so.detector_pads(H, W)
    Ho, Wo = so.out_hw(H, W, pads)
    o = so.stem_conv64(frames, Wt, bn, pads, "detector")
    assert o["ref"].shape == (2, Ho, Wo, 64)
    V = so.pack16(so.held(frames, "detector"), Ho + 3, Wo + 3)
    scale, shift = so.bn_fold(bn)
    pre = conv_detector_operand(V, det_weight_pack(Wt.astype(np.float64)), Ho, Wo) * scale + shift
    np.testing.assert_allclose(pre, o["pre"], rtol=0, atol=1e-12 * max(1.0, np.abs(o["pre"]).max()))


@pytest.mark.parametrize("H,W", SIZES + [(256, 128), (128, 256)])
def test_reid_pack_times_restated_weights_is_the_float64_stem(H, W):
    frames = _frames(2, H, W, H * 1000 + W + 1)
    Wt, bn = _weights(H * W)
    w_oihw = np.ascontiguousarray(Wt.transpose(3, 2, 0, 1))
    Ho, Wo = so.out_hw(H, W, so.REID_PADS)
    assert (Ho, Wo) == ((H - 1) // 2 + 1, (W - 1) // 2 + 1)     # reid_engine.cu's h1, w1
    o = so.stem_conv64(frames, so.oihw_to_hwio(w_oihw), bn, so.REID_PADS, "reid")
    U = so.pack64(so.held(frames, "reid"), Ho + 3, Wo)
    scale, shift = so.bn_fold(bn)
    pre = conv_reid_operand(U, reid_weight_pack(w_oihw.astype(np.float64)), Ho) * scale + shift
    np.testing.assert_allclose(pre, o["pre"], rtol=0, atol=1e-12 * max(1.0, np.abs(o["pre"]).max()))


class _Stop(Exception):
    pass


@pytest.mark.parametrize("H,W", [(7, 7), (13, 17), (192, 256), (200, 300)])
def test_stem_conv64_is_the_oracle_backbone_conv0_step(H, W, monkeypatch):
    """oracle.frcnn.backbone evaluated in float64 up to its max-pool, whose input is the pad [1, 0] of conv0 + BN + ReLU:
    stem_conv64 with the detector pads on the same float64 input."""
    from oracle import frcnn
    from object_detection_tracking_b200.config import make_config
    from object_detection_tracking_b200.synth import synth_weights
    cfg = make_config(resnet_num_block=(1, 1, 2, 1), max_size=256, short_edge_size=192)
    Wt = synth_weights(cfg, 1234)
    frame = _frames(1, H, W, 11)[0].astype(np.float32)
    seen = {}

    class Fx:
        def __getattr__(self, name):
            return getattr(torch.nn.functional, name)

        def max_pool2d(self, x, *a, **k):
            seen["x"] = x
            raise _Stop()

    monkeypatch.setattr(frcnn, "F", Fx())
    with frcnn.exact():
        x = frcnn.preprocess(frame)
        with pytest.raises(_Stop):
            frcnn.backbone(x, Wt, cfg)
    c1 = seen["x"][0, :, 1:, 1:].permute(1, 2, 0).numpy()                # drop the [1, 0] pad
    x64 = x[0].permute(1, 2, 0).numpy()[None]
    o = so.stem_conv64(x64, Wt["conv0/W"], so.det_bn(Wt), so.detector_pads(H, W), None)
    assert c1.shape == o["ref"].shape[1:]
    np.testing.assert_allclose(o["ref"][0], c1, rtol=0, atol=1e-12 * np.abs(c1).max())


def test_padding_only_rows_and_columns():
    pads = so.detector_pads(200, 300)
    rows, cols = so.padding_only(200, 300, pads, so.out_hw(200, 300, pads))
    assert list(np.flatnonzero(rows)) == list(range(102, 112)) and list(np.flatnonzero(cols)) == list(range(152, 160))
    rows, cols = so.padding_only(256, 128, so.REID_PADS, so.out_hw(256, 128, so.REID_PADS))
    assert not rows.any() and not cols.any()


def test_bound_covers_the_fold_and_a_perturbed_weight_leaves_it():
    """The bound holds for the engines' own arithmetic restated coarsely (fp32 folded weights, fp32 accumulation), and a
    stem missing one tap row (rr == 6) is far outside it."""
    frames = _frames(1, 13, 17, 5)
    Wt, bn = _weights(9)
    pads = so.detector_pads(13, 17)
    o = so.stem_conv64(frames, Wt, bn, pads, "detector")
    scale, shift = so.bn_fold(bn)
    xr = so.held(frames, "detector")
    Wf = (Wt.astype(np.float64) * scale).astype(np.float32)
    y32 = np.maximum(torch.nn.functional.conv2d(
        torch.nn.functional.pad(torch.from_numpy(xr.astype(np.float32)).permute(0, 3, 1, 2), (3, pads[3], 3, pads[1])),
        torch.from_numpy(Wf).permute(3, 2, 0, 1), stride=2).permute(0, 2, 3, 1).numpy() + shift.astype(np.float32), 0)
    assert (np.abs(y32 - o["ref"]) <= o["bound"]).all()
    cut = Wt.copy()
    cut[6] = 0
    bad = so.stem_conv64(frames, cut, bn, pads, "detector")["ref"]
    assert (np.abs(bad - o["ref"]) > o["bound"]).any()
