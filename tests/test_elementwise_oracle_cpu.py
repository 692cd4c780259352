"""tests/elementwise_oracle.py pinned against independent implementations: torch's float64 conv2d / pools / interpolate
and unfold, and the project's EfficientDet and EfficientNet oracles, so that the SAME convention and the squeeze-excite the
kernel tests hold the GPU to are the ones the whole-network oracles use.  No GPU needed."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import elementwise_oracle as eo
from oracle import effdet as oeffdet
from oracle import efficientnet as oeffnet
from oracle import frcnn


def _nchw(x):
    return torch.from_numpy(np.ascontiguousarray(x, np.float64)).permute(0, 3, 1, 2)


def _nhwc(t):
    return t.permute(0, 2, 3, 1).numpy()


# ---- the plane format ----------------------------------------------------------------------------------------------
def test_planes_match_torch_half_and_round_trip():
    rng = np.random.default_rng(0)
    x = np.concatenate([rng.standard_normal(20000) * 10.0 ** rng.uniform(-9, 4, 20000),
                        [0.0, -0.0, 1.0, 65504.0, -65504.0, 2.0 ** -24, 2.0 ** -14, 1 + 2.0 ** -11, 1 + 3 * 2.0 ** -12]])
    x = x.astype(np.float32)
    hi, lo = eo.planes(x)
    assert (hi.view(np.uint16) == torch.from_numpy(x).half().numpy().view(np.uint16)).all()
    r = (torch.from_numpy(x) - torch.from_numpy(hi.astype(np.float32))) * 2048.0
    assert (lo.view(np.uint16) == r.half().numpy().view(np.uint16)).all()
    for split in (True, False):
        v = eo.representable(x, split)
        assert (np.abs(v.astype(np.float64) - x) <= eo.store_bound(x, split)).all()
        # a fixed point: its planes hold it exactly, and splitting their value again gives the same planes
        assert np.array_equal(eo.representable(v, split).view(np.uint32), v.view(np.uint32))
        h, l = eo.raw(v, split)
        assert np.array_equal(eo.joined(h, l), v.astype(np.float64))
        h2, l2 = eo.raw(eo.value(h.view(np.float16), None if l is None else l.view(np.float16)), split)
        assert np.array_equal(h2, h) and (l is None or np.array_equal(l2, l))


# ---- depthwise convs -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K,S", [(3, 1), (3, 2), (5, 1), (5, 2)])
@pytest.mark.parametrize("H,W", [(1, 1), (1, 9), (7, 1), (6, 6), (7, 9), (10, 13)])
def test_depthwise_same_matches_torch_and_efficientnet_oracle(K, S, H, W):
    rng = np.random.default_rng(K * 100 + S * 10 + H + W)
    C = 16
    x = rng.standard_normal((1, H, W, C))
    w = rng.standard_normal((K, K, C))
    b = rng.standard_normal(C)
    (Ho, pt), (Wo, pl) = eo.same_pad(H, K, S), eo.same_pad(W, K, S)
    got, Sabs = eo.depthwise(x, w, b, S, (pt, pl), (Ho, Wo))
    # independent: explicit pads, then torch's grouped conv in float64
    ph, pw = max((Ho - 1) * S + K - H, 0), max((Wo - 1) * S + K - W, 0)
    xt = F.pad(_nchw(x), (pl, pw - pl, pt, ph - pt))
    ref = F.conv2d(xt, torch.from_numpy(w).permute(2, 0, 1)[:, None], torch.from_numpy(b), stride=S, groups=C)
    np.testing.assert_allclose(got, _nhwc(ref), rtol=1e-12, atol=1e-12)
    # the EfficientNet oracle's depthwise conv (TF SAME) in float64
    with frcnn.exact():
        t = oeffnet.dwconv(_nchw(x), {"dw/depthwise_kernel": w[:, :, :, None]}, "dw", S)
    np.testing.assert_allclose(got - b, _nhwc(t), rtol=1e-12, atol=1e-12)
    assert (Sabs >= np.abs(got) - 1e-12).all()


def test_depthwise_osnet_matches_torch():
    rng = np.random.default_rng(3)
    x = rng.standard_normal((3, 5, 7, 8))
    w = rng.standard_normal((3, 3, 8))
    b = rng.standard_normal(8)
    got, _ = eo.depthwise(x, w, b, 1, (1, 1))
    ref = F.conv2d(_nchw(x), torch.from_numpy(w).permute(2, 0, 1)[:, None], torch.from_numpy(b), padding=1, groups=8)
    np.testing.assert_allclose(eo.relu(got), _nhwc(torch.relu(ref)), rtol=1e-12, atol=1e-12)


# ---- pools ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H,W", [(1, 1), (2, 3), (5, 6), (8, 8), (9, 7)])
def test_maxpool_stem_matches_torch_and_tf_padding(H, W):
    rng = np.random.default_rng(H * 10 + W)
    x = rng.standard_normal((2, H, W, 8))
    # the ReID stem: nn.MaxPool2d(3, 2, 1)
    ref = F.max_pool2d(_nchw(x), 3, 2, 1)
    np.testing.assert_array_equal(eo.maxpool_stem(x, ref.shape[2:]), _nhwc(ref))
    # the detector stem: TF pad [1, 0] then 3x3/2 VALID (nn.py:896-900), -inf padded
    if H >= 2 and W >= 2:
        ref = F.max_pool2d(F.pad(_nchw(x), (1, 0, 1, 0), value=float("-inf")), 3, 2)
        assert ref.shape[2:] == (H // 2, W // 2)
        np.testing.assert_array_equal(eo.maxpool_stem(x, (H // 2, W // 2)), _nhwc(ref))


@pytest.mark.parametrize("H,W", [(2, 2), (5, 7), (8, 6), (9, 9)])
def test_avgpool2_and_gap_match_torch(H, W):
    rng = np.random.default_rng(H + 7 * W)
    x = rng.standard_normal((2, H, W, 8))
    np.testing.assert_allclose(eo.avgpool2(x), _nhwc(F.avg_pool2d(_nchw(x), 2)), rtol=1e-13, atol=1e-15)
    np.testing.assert_allclose(eo.gap(x), F.adaptive_avg_pool2d(_nchw(x), 1)[:, :, 0, 0].numpy(), rtol=1e-13, atol=1e-15)
    x32 = x.astype(np.float32)
    # three fp32 additions, each off by at most U times the sum of the magnitudes (the * 0.25 is exact)
    assert (np.abs(eo.avgpool2_f32(x32) - eo.avgpool2(x32)) <= 3 * eo.U * eo.avgpool2(np.abs(x32))).all()


# ---- BiFPN ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("src,dst", [((8, 12), (4, 6)), ((7, 9), (4, 5)), ((5, 5), (3, 3)), ((4, 6), (8, 12)),
                                     ((3, 3), (3, 3)), ((2, 3), (1, 2))])
def test_resample_matches_effdet_oracle_and_torch(src, dst):
    rng = np.random.default_rng(src[0] * 31 + dst[1])
    x = rng.standard_normal((2, src[0], src[1], 8))
    mode, pads, got = eo.resample(x, *dst)
    with frcnn.exact():
        ref = oeffdet.resample(_nchw(x), {}, "r", dst[0], dst[1], 8)
    np.testing.assert_array_equal(got, _nhwc(ref))
    if mode == 1:
        odd = (src[0] % 2, src[1] % 2)
        assert pads == odd, (pads, odd)   # an odd map pads one row / column before
    if mode == 2:
        np.testing.assert_array_equal(got, _nhwc(F.interpolate(_nchw(x), scale_factor=2, mode="nearest")))


@pytest.mark.parametrize("weights", [None, (0.7, -0.3, 1.9), (0.2, 0.5)])
def test_bifpn_combine_matches_effdet_oracle_formula(weights):
    rng = np.random.default_rng(5)
    n = 3 if weights is None or len(weights) == 3 else 2
    shapes = [(6, 10), (3, 5), (12, 20)][:n]
    xs = [rng.standard_normal((1, h, w, 8)) for h, w in shapes]
    got, S, pre = eo.bifpn_combine(xs, 6, 10, weights, act=True)
    # the combine as oracle/effdet.py's build_bifpn_layer writes it, in float64 torch
    with frcnn.exact():
        ins = [oeffdet.resample(_nchw(x), {}, "r", 6, 10, 8) for x in xs]
        if weights is None:
            node = ins[0]
            for t in ins[1:]:
                node = node + t
        else:
            ws = [torch.relu(torch.tensor(w, dtype=torch.float64)) for w in weights]
            tot = sum(ws[1:], ws[0])
            node = sum((ins[k] * ws[k] / (tot + 0.0001) for k in range(1, n)), ins[0] * ws[0] / (tot + 0.0001))
        node = oeffdet.swish(node)
    np.testing.assert_allclose(got, _nhwc(node), rtol=1e-12, atol=1e-12)
    f32 = eo.bifpn_combine_f32([x.astype(np.float32) for x in xs], 6, 10, weights)
    assert (np.abs(f32 - pre) <= 8 * eo.U * S + 1e-30).all()


# ---- squeeze-excite ------------------------------------------------------------------------------------------------
def test_mbconv_se_matches_efficientnet_oracle():
    rng = np.random.default_rng(11)
    B, HW, Cp, creal, nr = 2, 35, 128, 96, 6
    x = rng.standard_normal((B, HW, Cp))
    x[..., creal:] = 1e3   # padded channels take no part
    w1, b1 = rng.standard_normal((creal, nr)), rng.standard_normal(nr)
    w2, b2 = rng.standard_normal((nr, creal)), rng.standard_normal(creal)
    gate, _ = eo.mbconv_se(x, creal, w1, b1, w2, b2)
    assert (gate[:, creal:] == 0).all()
    W = {"se/conv2d/kernel": w1[None, None], "se/conv2d/bias": b1,
         "se/conv2d_1/kernel": w2[None, None], "se/conv2d_1/bias": b2}
    with frcnn.exact():   # mbconv's SE lines, with the oracle's own conv and swish
        t = torch.from_numpy(x[..., :creal]).reshape(B, 5, 7, creal).permute(0, 3, 1, 2)
        s = t.mean(dim=(2, 3), keepdim=True)
        s = oeffnet.conv(oeffnet.swish(oeffnet.conv(s, W, "se/conv2d", bias=True)), W, "se/conv2d_1", bias=True)
        ref = torch.sigmoid(s)[:, :, 0, 0].numpy()
    np.testing.assert_allclose(gate[:, :creal], ref, rtol=1e-12, atol=1e-14)


def test_channel_gate_and_gated_sum_match_torch():
    rng = np.random.default_rng(12)
    B, HW, C, creal, cr = 3, 10, 64, 48, 3
    s = rng.standard_normal((4, B, HW, C))
    w1, b1 = rng.standard_normal((cr, creal)), rng.standard_normal(cr)
    w2, b2 = rng.standard_normal((creal, cr)), rng.standard_normal(creal)
    pooled = np.stack([eo.gap(s[k]) for k in range(4)], axis=1)            # [B][4][C]
    gates, _, _, _ = eo.channel_gate(pooled[..., :creal].reshape(B * 4, creal), w1, b1, w2, b2)
    # OSNet's ChannelGate (osnet.py:162-220) as torch modules in float64
    fc1 = torch.nn.Conv2d(creal, cr, 1).double()
    fc2 = torch.nn.Conv2d(cr, creal, 1).double()
    with torch.no_grad():
        fc1.weight.copy_(torch.from_numpy(w1)[:, :, None, None])
        fc1.bias.copy_(torch.from_numpy(b1))
        fc2.weight.copy_(torch.from_numpy(w2)[:, :, None, None])
        fc2.bias.copy_(torch.from_numpy(b2))
        ref = torch.zeros(B, HW, C, dtype=torch.float64)
        for k in range(4):
            xk = torch.from_numpy(s[k][..., :creal]).reshape(B, 2, 5, creal).permute(0, 3, 1, 2)
            g = torch.sigmoid(fc2(torch.relu(fc1(F.adaptive_avg_pool2d(xk, 1)))))
            np.testing.assert_allclose(gates.reshape(B, 4, creal)[:, k], g[:, :, 0, 0].numpy(), rtol=1e-12)
            ref[..., :creal] += (xk * g).permute(0, 2, 3, 1).reshape(B, HW, creal)
    g_full = np.zeros((B, 4, C))
    g_full[..., :creal] = gates.reshape(B, 4, creal)
    out, S = eo.gated_sum4(s, g_full)
    np.testing.assert_allclose(out, ref.numpy(), rtol=1e-12, atol=1e-12)
    f32 = eo.gated_sum4_f32(s.astype(np.float32), g_full.astype(np.float32))
    ref32, S32 = eo.gated_sum4(s.astype(np.float32), g_full.astype(np.float32))
    assert (np.abs(f32 - ref32) <= 8 * eo.U * S32 + 1e-30).all()


# ---- EfficientNet's stem operand -----------------------------------------------------------------------------------
@pytest.mark.parametrize("H,W", [(1, 1), (4, 6), (7, 5), (9, 10)])
def test_stem_im2col_matches_unfold(H, W):
    rng = np.random.default_rng(H * W)
    img = rng.standard_normal((H, W, 3))
    (Ho, pt), (Wo, pl) = eo.same_pad(H, 3, 2), eo.same_pad(W, 3, 2)
    got = eo.stem_im2col(img, (Ho, Wo), (pt, pl))
    ph, pw = max((Ho - 1) * 2 + 3 - H, 0), max((Wo - 1) * 2 + 3 - W, 0)
    t = F.pad(_nchw(img[None]), (pl, pw - pl, pt, ph - pt))
    cols = F.unfold(t, 3, stride=2)                             # [1][c * 9 + r * 3 + s][Ho * Wo]
    ref = cols.reshape(3, 9, Ho, Wo).permute(2, 3, 1, 0).reshape(Ho, Wo, 27).numpy()   # -> (r*3 + s)*3 + c
    np.testing.assert_array_equal(got[..., :27], ref)
    assert (got[..., 27:] == 0).all()
    # the stem conv of the EfficientNet oracle equals this operand times the packed kernel
    w = rng.standard_normal((3, 3, 3, 5))
    with frcnn.exact():
        conv = oeffnet.conv(_nchw(img[None]), {"k/kernel": w}, "k", stride=2)
    np.testing.assert_allclose(got[..., :27] @ w.reshape(27, 5), _nhwc(conv)[0], rtol=1e-12, atol=1e-12)
