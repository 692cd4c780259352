"""The float64 conv oracle (tests/conv_oracle.py) against torch and explicit loops, its plane emulation and error bound,
and the host-side refusals of b2_op_conv2d_view -- all without a GPU."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import conv_oracle as co


def _fp16_exact(rng, shape, scale=1.0):
    return (rng.standard_normal(shape) * scale).astype(np.float16).astype(np.float32)


@pytest.mark.parametrize("R,S,stride,dil,pad,relu", [
    (1, 1, 1, 1, (0, 0, 0, 0), 0), (3, 3, 1, 1, (1, 1, 1, 1), 1), (3, 3, 2, 1, (1, 0, 1, 0), 1),
    (1, 3, 1, 2, (0, 0, 2, 2), 2), (5, 5, 2, 3, (2, 3, 1, 4), 0)])
def test_oracle_equals_torch_float64_on_dense_cases(R, S, stride, dil, pad, relu):
    """Operands that fp16 holds exactly (lo' = 0): the oracle is the float64 conv + bias + activation."""
    rng = np.random.default_rng(R * 10 + S + stride)
    x, w = _fp16_exact(rng, (2, 11, 13, 8)), _fp16_exact(rng, (R, S, 8, 5), 0.3)
    bias = rng.standard_normal(5).astype(np.float32)
    o = co.reference(x, w, bias, stride=stride, dil=dil, pad=pad, relu=relu)
    pt, pb, pl, pr = pad
    t = F.conv2d(F.pad(torch.from_numpy(x).double().permute(0, 3, 1, 2), (pl, pr, pt, pb)),
                 torch.from_numpy(w).double().permute(3, 2, 0, 1), torch.from_numpy(bias).double(), stride=stride,
                 dilation=dil)
    t = torch.relu(t) if relu == 1 else t * torch.sigmoid(t) if relu == 2 else t
    t = t.permute(0, 2, 3, 1).numpy()
    np.testing.assert_allclose(o["ref"][..., :5], t, rtol=1e-12, atol=1e-12)
    assert (o["ref"][..., 5:] == 0).all() if relu != 2 else np.allclose(o["ref"][..., 5:], 0)
    np.testing.assert_allclose(o["S"][..., :5], F.conv2d(
        F.pad(torch.from_numpy(np.abs(x)).double().permute(0, 3, 1, 2), (pl, pr, pt, pb)),
        torch.from_numpy(np.abs(w)).double().permute(3, 2, 0, 1), stride=stride, dilation=dil).permute(0, 2, 3, 1).numpy(),
        rtol=1e-12)
    assert (o["L"] == 0).all()


def _loop_conv(buf, w, bias, res, view, stride, dil, pad, res_shift, off):
    """The ConvDesc contract written out element by element (conv_simt.cu's indexing)."""
    B, PH, PW, ld = buf.shape
    in_H, in_W, Cin = view
    R, S, _, Cout = w.shape
    pt, pb, pl, pr = pad
    Ho, Wo = co.out_size(in_H, pt, pb, R, stride, dil), co.out_size(in_W, pl, pr, S, stride, dil)
    flat = buf.astype(np.float64).reshape(-1)
    out = np.zeros((B, Ho, Wo, Cout))
    for b in range(B):
        for p in range(Ho):
            for q in range(Wo):
                for o in range(Cout):
                    acc = float(bias[o])
                    for r in range(R):
                        ih = p * stride - pt + r * dil
                        if not 0 <= ih < in_H:
                            continue
                        for s in range(S):
                            iw = q * stride - pl + s * dil
                            if not 0 <= iw < in_W:
                                continue
                            base = ((b * PH + ih) * PW + iw) * ld
                            acc += float(np.dot(flat[base:base + Cin], w[r, s, :, o].astype(np.float64)))
                    acc += float(res[b, (p + off[0]) >> res_shift, (q + off[1]) >> res_shift, o])
                    out[b, p, q, o] = acc
    return out


@pytest.mark.parametrize("name,buf_shape,view,R,S,stride,dil,pad,res_shift,off", [
    ("crop_view_s2_remainder", (2, 9, 11, 8), (7, 8, 8), 3, 3, 2, 1, (1, 1, 1, 0), 0, (0, 0)),
    ("channel_slice_1x1", (1, 5, 6, 16), (5, 6, 8), 1, 1, 1, 1, (0, 0, 0, 0), 0, (0, 0)),
    ("stem_overlap_4x1", (2, 7, 9, 4), (7, 6, 16), 4, 1, 1, 1, (0, 0, 0, 0), 0, (0, 0)),
    ("negative_crop_pad", (1, 10, 10, 8), (10, 10, 8), 1, 1, 2, 1, (0, -1, 0, -1), 0, (0, 0)),
    ("placed_upsampled_res", (1, 6, 7, 8), (6, 7, 8), 3, 1, 1, 2, (2, 2, 0, 0), 1, (1, 2)),
    ("dil3_R_ne_S", (1, 12, 9, 8), (11, 9, 8), 3, 2, 1, 3, (3, 2, 0, 3), 0, (2, 0)),
])
def test_view_stride_overlap_placement_match_an_explicit_loop(name, buf_shape, view, R, S, stride, dil, pad, res_shift,
                                                             off):
    rng = np.random.default_rng(len(name))
    buf = _fp16_exact(rng, buf_shape)
    Cin = view[2]
    w, bias = _fp16_exact(rng, (R, S, Cin, 3), 0.3), rng.standard_normal(3).astype(np.float32)
    Ho = co.out_size(view[0], pad[0], pad[1], R, stride, dil)
    Wo = co.out_size(view[1], pad[2], pad[3], S, stride, dil)
    rH, rW = ((Ho + off[0] - 1) >> res_shift) + 1, ((Wo + off[1] - 1) >> res_shift) + 1
    res = _fp16_exact(rng, (1 if buf_shape[0] == 1 else buf_shape[0], rH, rW, 16))
    o = co.reference(buf, w, bias, res, view=view, stride=stride, dil=dil, pad=pad, res_shift=res_shift, off=off)
    exp = _loop_conv(buf, w, bias, res, view, stride, dil, pad, res_shift, off)
    np.testing.assert_allclose(o["ref"][..., :3], exp, rtol=1e-12, atol=1e-12)
    # placement writes the window at the offset and nothing else
    init = np.full((buf_shape[0], Ho + off[0] + 1, Wo + off[1] + 2, 24), -7.0)
    placed = co.place(o["ref"], init, off)
    assert (placed[:, off[0]:off[0] + Ho, off[1]:off[1] + Wo, :16] == o["ref"]).all()
    keep = np.ones(placed.shape, bool)
    keep[:, off[0]:off[0] + Ho, off[1]:off[1] + Wo, :16] = False
    assert (placed[keep] == -7.0).all()


def test_plane_emulation_is_exact_and_holds_22_bits():
    rng = np.random.default_rng(0)
    x = np.concatenate([rng.standard_normal(200000) * 10.0 ** rng.uniform(-4, 4, 200000),
                        [65504.0, -65504.0, 2.0 ** -14, 1.0 + 2.0 ** -23]]).astype(np.float32)
    hi, lo = co.split_planes(x)
    # numpy's float16 cast is round-to-nearest-even, as __float2half_rn; torch's agrees
    assert (hi == torch.from_numpy(x).half().numpy()).all()
    assert (lo == torch.from_numpy((x - hi.astype(np.float32)) * np.float32(2048)).half().numpy()).all()
    xt = co.join(hi, lo)
    normal = np.abs(x) >= 2.0 ** -14
    assert (np.abs(x[normal] - xt[normal]) <= 2.0 ** -22 * np.abs(x[normal])).all()
    assert (np.abs(x - xt) <= 2.0 ** -36 + 2.0 ** -22 * np.abs(x)).all()


@pytest.mark.parametrize("K_taps,Cin,signed", [(1, 64, True), (9, 64, False), (1, 512, False), (9, 256, True)])
def test_bound_holds_for_a_float32_evaluation_of_the_same_sums(K_taps, Cin, signed):
    """A float32 sequential evaluation (the CUDA-core kernel's fmaf chains, with the split's dropped lo.lo product)
    stays inside the simt bound at every element; the bound is not vacuous (it is far below the output's scale)."""
    rng = np.random.default_rng(K_taps + Cin)
    R = 3 if K_taps == 9 else 1
    x = rng.uniform(0, 2, (1, 6, 7, Cin)).astype(np.float32)
    x[..., ::7] = 0
    scale = 10.0 ** np.linspace(-3, 2, 20)
    w = (rng.uniform(0.1, 1, (R, R, Cin, 20)) * scale / (R * R * Cin)).astype(np.float32)
    if signed:
        w *= rng.choice([-1, 1], w.shape).astype(np.float32)
    bias = (rng.standard_normal(20) * scale).astype(np.float32)
    pad = (R // 2,) * 4
    o = co.reference(x, w, bias, pad=pad)
    xh, xl = co.split_planes(x)
    wh, wl = co.split_planes(np.pad(w, ((0, 0), (0, 0), (0, 0), (0, 12))))
    xpad = np.pad(np.stack([xh.astype(np.float32), xl.astype(np.float32)]), ((0, 0), (0, 0), (R // 2,) * 2, (R // 2,) * 2,
                                                                                (0, 0)))
    acc0 = np.zeros((1, 6, 7, 32), np.float32)
    acc1 = np.zeros_like(acc0)
    for r in range(R):
        for s in range(R):
            a_hi, a_lo = xpad[0][:, r:r + 6, s:s + 7], xpad[1][:, r:r + 6, s:s + 7]
            for c in range(Cin):
                bh, bl = wh[r, s, c].astype(np.float32), wl[r, s, c].astype(np.float32)
                acc0 = (acc0 + a_hi[..., c:c + 1] * bh).astype(np.float32)   # products of fp16 values: exact in fp32
                acc1 = (acc1 + a_hi[..., c:c + 1] * bl).astype(np.float32)
                acc1 = (acc1 + a_lo[..., c:c + 1] * bh).astype(np.float32)
    v = acc0 + acc1 * np.float32(1 / 2048)
    bp = np.zeros(32, np.float32)
    bp[:20] = bias
    v = (v + bp).astype(np.float32)
    hi, lo = co.split_planes(v)
    out = co.join(hi, lo)
    bnd = co.bound(o["K"], o["S"], o["b"], o["r"], o["ref"], "split", L=o["L"], impl="simt")
    err = np.abs(out - o["ref"])
    assert (err <= bnd).all(), (err / bnd).max()
    assert (bnd[..., :20] <= 1e-3 * np.abs(o["S"][..., :20]) + 1e-30).all()
    # and the element-wise bound is tighter than a tensor-wide tolerance on the small columns
    assert bnd[..., 0].max() < 1e-4 * np.abs(o["ref"]).max()


def _view_args(**kw):
    a = dict(x=np.zeros((1, 8, 8, 64), np.float32), w=np.zeros((3, 3, 64, 16), np.float32), pad=(1, 1, 1, 1))
    a.update(kw)
    return a


@pytest.mark.parametrize("kw,message", [
    (dict(view=(9, 8, 64)), "view lies outside the input buffer"),
    (dict(x=np.zeros((1, 8, 8, 16), np.float32), view=(8, 8, 64), w=np.zeros((4, 1, 64, 16), np.float32),
          pad=(0, 0, 0, 0)), "run past the input buffer"),
    (dict(out_init=np.zeros((1, 8, 8, 16), np.float32), off=(1, 0)), "does not fit the output buffer"),
    (dict(out_init=np.zeros((1, 8, 8, 8), np.float32)), "ldc must cover Cout_pad"),
    (dict(res=np.zeros((1, 8, 8, 8), np.float32)), "ldr must cover Cout_pad"),
    (dict(res=np.zeros((1, 4, 3, 16), np.float32), res_shift=1), "residual is smaller"),
    (dict(out_init=np.zeros((1, 9, 9, 16), np.float32), off=(1, 1), res=np.zeros((1, 8, 8, 16), np.float32)),
     "residual is smaller"),
    (dict(images=(1, 1)), "image range outside the batch"),
])
def test_conv2d_view_refuses_malformed_cases_before_any_device_work(kw, message):
    from object_detection_tracking_b200 import engine
    with pytest.raises(RuntimeError, match=message):
        engine.op_conv2d_view(**_view_args(**kw))


def test_conv2d_view_valid_case_reaches_the_device():
    if torch.cuda.is_available():
        pytest.skip("GPU present: tests/test_conv_contract_gpu.py runs it")
    from object_detection_tracking_b200 import engine
    with pytest.raises(RuntimeError) as e:
        engine.op_conv2d_view(**_view_args())
    assert "b2_op_conv2d_view" in str(e.value) and "outside" not in str(e.value) and "cover" not in str(e.value)
