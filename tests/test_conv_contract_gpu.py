"""The conv kernels against the float64 oracle (tests/conv_oracle.py) over the whole ConvDesc contract, through
b2_op_conv2d_view: geometry, input views and channel strides, output placement, fp32 outputs, both epilogues, batch parts,
the accumulation chunking and the range monitor.  Every comparison is element-wise against the oracle's bound, so an
error in a column far below the tensor's largest value is not hidden by it."""
import numpy as np
import pytest

import conv_oracle as co

pytestmark = pytest.mark.gpu

SENTINEL = np.float32(-1234.56789)   # fills every output cell the kernel must not write (both planes non-zero)


def _engine():
    from object_detection_tracking_b200 import engine
    return engine


def make_data(rng, B, PH, PW, ld, view, R, S, Cout, res_shape=None, nonneg=False):
    """Input buffer with NaN outside the view and in channels [Cin, ld), every 5th input channel zero; weights, bias and
    residual with a scale of their own per output column, from 1e-3 to 1e2."""
    in_H, in_W, Cin = view
    x = np.full((B, PH, PW, ld), np.nan, np.float32)
    v = rng.uniform(0, 2, (B, in_H, in_W, Cin)) if nonneg else rng.standard_normal((B, in_H, in_W, Cin))
    v[..., 2::5] = 0
    if ld >= Cin:
        x[:, :in_H, :in_W, :Cin] = v
    scale = 10.0 ** rng.permutation(np.linspace(-3, 2, Cout))
    w = (rng.uniform(0.1, 1, (R, S, Cin, Cout)) * rng.choice([-1, 1], (R, S, Cin, Cout)) * scale /
         np.sqrt(R * S * Cin)).astype(np.float32)
    bias = (rng.standard_normal(Cout) * scale).astype(np.float32)
    res = None
    if res_shape is not None:
        res = rng.standard_normal(res_shape).astype(np.float32)
        res[..., :Cout] *= scale
    return x, v.astype(np.float32), w, bias, res


def check_against_oracle(o, out, hi, lo, split, impl="tc", chunk_kb=None, relu=0, out_f32=False):
    """The window's columns [0, Cout_pad) within the element-wise bound."""
    if out_f32:
        got = out.astype(np.float64)
    else:
        got = co.join(hi.view(np.float16), lo.view(np.float16) if split else None)
    B, Ho, Wo, Cp = o["ref"].shape
    bnd = co.bound(o["K"], o["S"], o["b"], o["r"], o["ref"], "split" if split else "fp16", L=o["L"], chunk_kb=chunk_kb,
                   impl=impl, out="f32" if out_f32 else "planes", relu=relu)
    return got, bnd


def assert_window(o, got, bnd, off=(0, 0)):
    B, Ho, Wo, Cp = o["ref"].shape
    win = got[:, off[0]:off[0] + Ho, off[1]:off[1] + Wo, :Cp]
    assert np.isfinite(win).all(), "non-finite output in the written window"
    err = np.abs(win - o["ref"])
    worst = np.unravel_index(np.argmax(err - bnd), err.shape)
    assert (err <= bnd).all(), "element %s: |err| %.3g > bound %.3g (ref %.6g)" % (
        worst, err[worst], bnd[worst], o["ref"][worst])


def assert_sentinel_kept(hi, lo, Ho, Wo, Cp, off, split):
    """Every plane element outside the written window, and every column >= Cout_pad, holds the sentinel's bits."""
    sh, sl = co.split_planes(np.array([SENTINEL]))
    keep = np.ones(hi.shape, bool)
    keep[:, off[0]:off[0] + Ho, off[1]:off[1] + Wo, :Cp] = False
    assert (hi[keep] == sh.view(np.uint16)[0]).all()
    if split:
        assert (lo[keep] == sl.view(np.uint16)[0]).all()


# ------------------------------------------------------------------------------------------------------------------
# Geometry sweep.  name: (B, H, W, Cin, Cout, R, S, stride, dil, pad (t, b, l, r))
GEOMETRY = {
    "1x1_b1":               (1, 16, 24, 64, 48, 1, 1, 1, 1, (0, 0, 0, 0)),
    "1x1_b3_tiles_wrap":    (3, 7, 9, 128, 200, 1, 1, 1, 1, (0, 0, 0, 0)),     # 63-pixel images: a tile spans 2+ images
    "1x1_many_tiles":       (1, 60, 70, 64, 48, 1, 1, 1, 1, (0, 0, 0, 0)),
    "1x1_s2_even":          (1, 10, 12, 64, 80, 1, 1, 2, 1, (0, 0, 0, 0)),
    "1x1_s2_rem_w":         (1, 9, 10, 64, 80, 1, 1, 2, 1, (0, 0, 0, 0)),      # (9-1) % 2 = 0, (10-1) % 2 = 1
    "1x1_s2_crop_rem_hw":   (3, 23, 41, 128, 144, 1, 1, 2, 1, (0, -1, 0, -1)),  # res5 block 0 shortcut, odd c4
    "3x3_b1":               (1, 13, 17, 64, 80, 3, 3, 1, 1, (1, 1, 1, 1)),
    "3x3_b3_wrap":          (3, 7, 11, 64, 48, 3, 3, 1, 1, (1, 1, 1, 1)),
    "3x3_cout200":          (1, 10, 12, 128, 200, 3, 3, 1, 1, (1, 1, 1, 1)),
    "3x3_cout15":           (1, 11, 13, 64, 15, 3, 3, 1, 1, (1, 1, 1, 1)),
    "3x3_s2_rem_h":         (1, 15, 16, 64, 48, 3, 3, 2, 1, (1, 0, 1, 0)),     # H: 15+1-3 = 13 odd; W: 14 even
    "3x3_s2_rem_w":         (1, 16, 15, 64, 48, 3, 3, 2, 1, (1, 0, 1, 0)),
    "3x3_s2_rem_hw_b3":     (3, 23, 41, 64, 144, 3, 3, 2, 1, (1, 0, 1, 0)),    # res5 block 0 conv2 at odd c4 sizes
    "3x3_s2_pad11_rem_h":   (1, 14, 15, 128, 80, 3, 3, 2, 1, (1, 1, 1, 1)),
    "3x3_s2_dil2_rem":      (1, 23, 40, 64, 80, 3, 3, 2, 2, (1, 0, 1, 0)),     # res5 block 0 with dilations
    "3x3_dil2":             (1, 15, 22, 128, 144, 3, 3, 1, 2, (2, 2, 2, 2)),
    "3x3_dil3":             (1, 14, 19, 64, 80, 3, 3, 1, 3, (3, 3, 3, 3)),
    "3x3_dil3_s2_rem":      (1, 19, 20, 64, 15, 3, 3, 2, 3, (3, 3, 3, 3)),
    "3x3_crop_pad":         (2, 12, 13, 64, 48, 3, 3, 1, 1, (1, -1, 1, -1)),
    "1x3":                  (1, 12, 17, 64, 144, 1, 3, 1, 1, (0, 0, 1, 1)),
    "1x3_s2_rem":           (1, 9, 22, 64, 48, 1, 3, 2, 1, (0, 0, 1, 1)),
    "3x1":                  (2, 13, 10, 128, 15, 3, 1, 1, 1, (1, 1, 0, 0)),
    "3x1_dil2":             (1, 16, 9, 64, 80, 3, 1, 1, 2, (2, 2, 0, 0)),
    "5x5":                  (3, 11, 13, 64, 48, 5, 5, 1, 1, (2, 2, 2, 2)),
    "5x5_s2_rem":           (1, 17, 18, 64, 80, 5, 5, 2, 1, (2, 2, 2, 2)),
    "5x5_dil2":             (1, 16, 17, 64, 15, 5, 5, 1, 2, (4, 4, 4, 4)),
    "4x1_valid":            (2, 15, 12, 64, 64, 4, 1, 1, 1, (0, 0, 0, 0)),
    "4x1_s2":               (1, 16, 11, 128, 48, 4, 1, 2, 1, (1, 1, 0, 0)),
    "7x7_s2":               (1, 20, 21, 64, 48, 7, 7, 2, 1, (3, 3, 3, 3)),
    "7x7_s2_rem_hw_b3":     (3, 19, 22, 64, 80, 7, 7, 2, 1, (3, 2, 3, 2)),
    "7x7_s1":               (1, 9, 12, 64, 200, 7, 7, 1, 1, (3, 3, 3, 3)),
    "1x1_cout15_b3":        (3, 12, 20, 128, 15, 1, 1, 1, 1, (0, 0, 0, 0)),
    "1x1_tiny_m":           (1, 3, 5, 64, 144, 1, 1, 1, 1, (0, 0, 0, 0)),
    "3x3_tiny_m":           (1, 2, 3, 128, 48, 3, 3, 1, 1, (1, 1, 1, 1)),
    "3x3_s2_rem_hw_cout200": (1, 11, 13, 128, 200, 3, 3, 2, 1, (1, 1, 1, 1)),
    "3x3_dil2_s2_b3":       (3, 13, 14, 64, 48, 3, 3, 2, 2, (2, 2, 2, 2)),
    "1x3_dil3":             (1, 8, 21, 64, 80, 1, 3, 1, 3, (0, 0, 3, 3)),
    "3x1_s2_rem_h":         (3, 12, 7, 64, 144, 3, 1, 2, 1, (1, 1, 0, 0)),
    "5x5_crop":             (1, 14, 15, 64, 48, 5, 5, 1, 1, (2, -1, 2, -2)),
    "7x7_dil2":             (1, 18, 20, 64, 15, 7, 7, 1, 2, (6, 6, 6, 6)),
}


def _oracle(x, w, bias, res=None, **kw):
    split = kw.pop("split")
    return co.reference(x, w, bias, res, split=split, **kw)


@pytest.mark.parametrize("name", sorted(GEOMETRY))
@pytest.mark.parametrize("split", [True, False], ids=["split", "fp16"])
def test_geometry_sweep_within_elementwise_bound(name, split):
    B, H, W, Cin, Cout, R, S, stride, dil, pad = GEOMETRY[name]
    rng = np.random.default_rng(sum(map(ord, name)))
    x, _, w, bias, _ = make_data(rng, B, H, W, Cin, (H, W, Cin), R, S, Cout)
    o = _oracle(x, w, bias, stride=stride, dil=dil, pad=pad, relu=1, split=split)
    Ho, Wo, Cp = o["Ho"], o["Wo"], o["Cp"]
    assert (Ho, Wo) == (co.out_size(H, pad[0], pad[1], R, stride, dil), co.out_size(W, pad[2], pad[3], S, stride, dil))
    init = np.full((B, Ho, Wo, Cp), SENTINEL, np.float32)
    out, hi, lo, flag = _engine().op_conv2d_view(x, w, bias, stride=stride, dil=dil, pad=pad, relu=1, out_init=init,
                                                 split=split)
    got, bnd = check_against_oracle(o, out, hi, lo, split)
    assert_window(o, got, bnd)
    assert flag == 0


# ------------------------------------------------------------------------------------------------------------------
# Views and channel strides: NaN everywhere the kernel must not read.  name: (B, PH, PW, in_ld, view, R, S, stride,
# pad, Cout)
VIEWS = {
    "crop_im2col_3x3":        (2, 14, 19, 64, (11, 15, 64), 3, 3, 1, (1, 1, 1, 1), 48),
    "crop_slice_3x3_s2":      (1, 17, 20, 128, (13, 16, 64), 3, 3, 2, (1, 0, 1, 0), 80),
    "crop_slice_1x1":         (3, 9, 12, 192, (7, 10, 128), 1, 1, 1, (0, 0, 0, 0), 144),   # crop: im2col map
    "slice_1x1_plain_2d":     (3, 9, 12, 192, (9, 12, 128), 1, 1, 1, (0, 0, 0, 0), 144),   # in_ld > Cin: 2-D map
    "slice_1x1_plain_2d_b1":  (1, 20, 30, 128, (20, 30, 64), 1, 1, 1, (0, 0, 0, 0), 15),
}


@pytest.mark.parametrize("name", sorted(VIEWS))
@pytest.mark.parametrize("impl,split", [("tcgen05", True), ("tcgen05", False), ("simt", True)])
def test_views_and_channel_strides_read_only_the_view(name, impl, split):
    B, PH, PW, ld, view, R, S, stride, pad, Cout = VIEWS[name]
    rng = np.random.default_rng(sum(map(ord, name)))
    x, _, w, bias, _ = make_data(rng, B, PH, PW, ld, view, R, S, Cout)
    o = _oracle(x, w, bias, view=view, stride=stride, pad=pad, split=split)
    init = np.full((B, o["Ho"], o["Wo"], o["Cp"]), SENTINEL, np.float32)
    out, hi, lo, _ = _engine().op_conv2d_view(x, w, bias, view=view, stride=stride, pad=pad, out_init=init, impl=impl,
                                              split=split)
    got, bnd = check_against_oracle(o, out, hi, lo, split, impl="tc" if impl == "tcgen05" else "simt")
    assert_window(o, got, bnd)


def test_plain_2d_map_and_im2col_map_of_a_channel_slice_are_bit_identical():
    B, PH, PW, ld, view, R, S, stride, pad, Cout = VIEWS["slice_1x1_plain_2d"]
    x, _, w, bias, _ = make_data(np.random.default_rng(4), B, PH, PW, ld, view, R, S, Cout)
    a = _engine().op_conv2d_view(x, w, bias, view=view, a_mode=0)
    b = _engine().op_conv2d_view(x, w, bias, view=view, a_mode=1)
    assert (a[1] == b[1]).all() and (a[2] == b[2]).all()


@pytest.mark.parametrize("c1h,c1w", [(96, 128), (50, 75)])
@pytest.mark.parametrize("impl,split", [("tcgen05", True), ("tcgen05", False), ("simt", True)])
def test_stem_overlapping_window_as_the_engine_builds_conv0(c1h, c1w, impl, split):
    """conv0 (engine.cu): a 4x1 VALID conv with Cin 64 over the [B][c1h + 3][c1w + 3][16] operand, pixel stride 16: each
    GEMM pixel reads four consecutive operand pixels, and the last column's window ends at the row's last pixel."""
    rng = np.random.default_rng(c1w)
    B = 2
    x = rng.standard_normal((B, c1h + 3, c1w + 3, 16)).astype(np.float32)
    w = (rng.standard_normal((4, 1, 64, 64)) * 10.0 ** rng.permutation(np.linspace(-3, 2, 64)) / 16).astype(np.float32)
    bias = rng.standard_normal(64).astype(np.float32)
    view = (c1h + 3, c1w, 64)
    o = _oracle(x, w, bias, view=view, relu=1, split=split)
    assert (o["Ho"], o["Wo"]) == (c1h, c1w)
    out, hi, lo, _ = _engine().op_conv2d_view(x, w, bias, view=view, relu=1, impl=impl, split=split)
    got, bnd = check_against_oracle(o, out, hi, lo, split, impl="tc" if impl == "tcgen05" else "simt", relu=1)
    assert_window(o, got, bnd)


# ------------------------------------------------------------------------------------------------------------------
# Placement
@pytest.mark.parametrize("off", [(1, 1), (0, 3), (2, 0)])
@pytest.mark.parametrize("res_shift", [None, 1])
@pytest.mark.parametrize("impl,split", [("tcgen05", True), ("tcgen05", False), ("simt", True)])
def test_placement_writes_only_its_window(off, res_shift, impl, split):
    rng = np.random.default_rng(off[0] * 7 + off[1])
    B, H, W, Cin, Cout = 2, 9, 11, 64, 40   # Cout_pad 48, ldc 64
    Ho, Wo, Cp, ldc = H, W, 48, 64
    res_shape = None
    if res_shift is not None:
        res_shape = (B, (Ho + off[0] + 1) // 2, (Wo + off[1] + 1) // 2, 56)
    x, _, w, bias, res = make_data(rng, B, H, W, Cin, (H, W, Cin), 3, 3, Cout, res_shape)
    o = _oracle(x, w, bias, res, pad=(1, 1, 1, 1), res_shift=res_shift or 0, off=off, relu=1, split=split)
    init = np.full((B, Ho + off[0] + 1, Wo + off[1] + 2, ldc), SENTINEL, np.float32)
    out, hi, lo, _ = _engine().op_conv2d_view(x, w, bias, res, pad=(1, 1, 1, 1), res_shift=res_shift or 0, off=off,
                                              out_init=init, relu=1, impl=impl, split=split)
    got, bnd = check_against_oracle(o, out, hi, lo, split, impl="tc" if impl == "tcgen05" else "simt", relu=1)
    assert_window(o, got, bnd, off)
    assert_sentinel_kept(hi, lo, Ho, Wo, Cp, off, split)


# ------------------------------------------------------------------------------------------------------------------
# fp32 outputs
@pytest.mark.parametrize("Cout,ldc", [(15, 16), (18, 32), (15, 32)])
@pytest.mark.parametrize("relu", [0, 1, 2])
@pytest.mark.parametrize("off", [(0, 0), (1, 2)])
def test_fp32_outputs(Cout, ldc, relu, off):
    rng = np.random.default_rng(Cout + ldc + relu)
    B, H, W, Cin = 2, 10, 13, 128
    x, _, w, bias, _ = make_data(rng, B, H, W, Cin, (H, W, Cin), 3, 3, Cout)
    Cp = (Cout + 15) // 16 * 16
    init = np.full((B, H + off[0] + 1, W + off[1], ldc), np.nan, np.float32)
    for impl, split in [("tcgen05", True), ("tcgen05", False), ("simt", True)]:
        o = _oracle(x, w, bias, pad=(1, 1, 1, 1), off=off, relu=relu, split=split)
        out, hi, _, flag = _engine().op_conv2d_view(x, w, bias, pad=(1, 1, 1, 1), off=off, out_init=init, relu=relu,
                                                    out_f32=True, impl=impl, split=split)
        assert hi is None and flag == 0
        got, bnd = check_against_oracle(o, out, None, None, split, impl="tc" if impl == "tcgen05" else "simt",
                                        relu=relu, out_f32=True)
        assert_window(o, got, bnd, off)
        keep = np.ones(out.shape, bool)
        keep[:, off[0]:off[0] + H, off[1]:off[1] + W, :Cp] = False
        assert np.isnan(out[keep]).all()


@pytest.mark.parametrize("split", [True, False], ids=["split", "fp16"])
@pytest.mark.parametrize("relu", [0, 1, 2])
def test_fp32_output_split_on_the_host_equals_both_plane_epilogues(split, relu):
    """Three paths of one layer: the fp32 output split by the plane rule, the direct epilogue's planes, the staged
    epilogue's planes -- identical bits."""
    rng = np.random.default_rng(relu)
    x, _, w, bias, res = make_data(rng, 2, 12, 14, 128, (12, 14, 128), 3, 3, 80, (2, 12, 14, 80))
    kw = dict(pad=(1, 1, 1, 1), relu=relu, split=split)
    f32, _, _, _ = _engine().op_conv2d_view(x, w, bias, res, out_f32=True, **kw)
    _, dh, dl, _ = _engine().op_conv2d_view(x, w, bias, res, force_epi=0, **kw)
    _, sh, sl, _ = _engine().op_conv2d_view(x, w, bias, res, force_epi=1, **kw)
    hh, ll = co.split_planes(f32)
    assert (dh == hh.view(np.uint16)).all() and (sh == dh).all()
    if split:
        assert (dl == ll.view(np.uint16)).all() and (sl == dl).all()


# ------------------------------------------------------------------------------------------------------------------
# Staged vs direct epilogue: DESIGN.md §4's "same arithmetic, same order, bit-identical outputs"
def _staged_cases():
    from test_conv_staged_epilogue_gpu import CASES
    return CASES


@pytest.mark.parametrize("name", sorted(_staged_cases()))
@pytest.mark.parametrize("split", [True, False], ids=["split", "fp16"])
def test_staged_and_direct_epilogues_are_bit_identical(name, split):
    B, H, W, Cin, Cout, R, relu, use_res = _staged_cases()[name]
    rng = np.random.default_rng(len(name))
    Cp = (Cout + 15) // 16 * 16
    x, _, w, bias, res = make_data(rng, B, H, W, Cin, (H, W, Cin), R, R, Cout, (B, H, W, Cp) if use_res else None)
    kw = dict(pad=(R // 2,) * 4, relu=relu, split=split)
    _, dh, dl, _ = _engine().op_conv2d_view(x, w, bias, res, force_epi=0, **kw)
    _, sh, sl, _ = _engine().op_conv2d_view(x, w, bias, res, force_epi=1, **kw)
    assert (dh == sh).all()
    if split:
        assert (dl == sl).all()
    if name in ("res_cout80", "swish_res", "no_res_3x3"):   # and both are right, not just equal
        o = _oracle(x, w, bias, res, pad=(R // 2,) * 4, relu=relu, split=split)
        got, bnd = check_against_oracle(o, None, sh, sl, split, relu=relu)
        assert_window(o, got, bnd)


def test_force_staged_refuses_an_ineligible_layer():
    x, _, w, bias, _ = make_data(np.random.default_rng(0), 1, 8, 8, 64, (8, 8, 64), 1, 1, 16)
    with pytest.raises(RuntimeError, match="placed inside a larger buffer"):
        _engine().op_conv2d_view(x, w, bias, off=(1, 0), out_init=np.zeros((1, 9, 8, 16), np.float32), force_epi=1)
    with pytest.raises(RuntimeError, match="fp32"):
        _engine().op_conv2d_view(x, w, bias, out_f32=True, force_epi=1)
    with pytest.raises(RuntimeError, match="upsampled"):
        _engine().op_conv2d_view(x, w, bias, np.zeros((1, 4, 4, 16), np.float32), res_shift=1, force_epi=1)


# ------------------------------------------------------------------------------------------------------------------
# Batch parts: an image's result does not depend on the part of the batch it runs in
@pytest.mark.parametrize("force_epi", [0, 1], ids=["direct", "staged"])
@pytest.mark.parametrize("split", [True, False], ids=["split", "fp16"])
def test_batch_parts_are_bit_identical_to_the_full_batch(force_epi, split):
    rng = np.random.default_rng(5)
    B, H, W, Cin, Cout = 5, 9, 13, 64, 80    # 117 pixels per image: every tile is ragged against the images
    x, _, w, bias, res = make_data(rng, B, H, W, Cin, (H, W, Cin), 3, 3, Cout, (B, H, W, 80))
    kw = dict(pad=(1, 1, 1, 1), relu=1, force_epi=force_epi, split=split)
    init = np.full((B, H, W, 80), SENTINEL, np.float32)
    _, fh, fl, _ = _engine().op_conv2d_view(x, w, bias, res, out_init=init, **kw)
    for parts in ([(b, 1) for b in range(B)], [(0, 2), (2, 3)]):
        for b0, nb in parts:
            _, ph, pl, _ = _engine().op_conv2d_view(x, w, bias, res, out_init=init, images=(b0, nb), **kw)
            assert (ph[b0:b0 + nb] == fh[b0:b0 + nb]).all(), (b0, nb)
            if split:
                assert (pl[b0:b0 + nb] == fl[b0:b0 + nb]).all(), (b0, nb)
            others = np.ones(B, bool)
            others[b0:b0 + nb] = False
            assert_sentinel_kept(ph[others], pl[others] if split else None, 0, 0, 0, (0, 0), split)


# ------------------------------------------------------------------------------------------------------------------
# Accumulation (ACC).  Coherent sums (activations >= 0 as after a ReLU, weights > 0) make the tensor cores' truncation
# toward zero a bias of the whole output; fp32 outputs leave the accumulation's error alone.
# K: (Cin, R, H, W, Cout) -- about 2.1 to 2.4 M outputs each
ACC_SHAPES = {64: (64, 1, 128, 128, 128), 576: (64, 3, 128, 128, 128), 2048: (2048, 1, 96, 96, 256),
              4608: (512, 3, 96, 96, 256)}
_ACC_CACHE = {}


def _acc_case(K):
    if K not in _ACC_CACHE:
        Cin, R, H, W, Cout = ACC_SHAPES[K]
        rng = np.random.default_rng(K)
        x = rng.uniform(0, 1, (1, H, W, Cin)).astype(np.float32)
        x[..., 3::8] = 0
        scale = 10.0 ** rng.permutation(np.linspace(-3, 2, Cout))
        w = (rng.uniform(0.1, 1, (R, R, Cin, Cout)) * scale).astype(np.float32)
        o = co.reference(x, w, None, pad=(R // 2,) * 4, split=True)
        _ACC_CACHE[K] = (x, w, o)
    return _ACC_CACHE[K]


def _acc_run(K, acc_kb):
    x, w, o = _acc_case(K)
    R = w.shape[0]
    out, _, _, _ = _engine().op_conv2d_view(x, w, None, pad=(R // 2,) * 4, out_f32=True, acc_kb=acc_kb)
    return out.astype(np.float64), o


def _chunk(K, acc_kb):
    """K-blocks per accumulator chunk the plan uses: acc_kb (0 = 1), or all of K when ACC is off or K is one chunk."""
    nkb = K // 64
    kb = 1 if acc_kb == 0 else acc_kb
    return nkb if acc_kb < 0 or nkb <= kb else kb


@pytest.mark.parametrize("K", sorted(ACC_SHAPES))
@pytest.mark.parametrize("acc_kb", [0, 2, 3, -1], ids=["default", "kb2", "kb3", "off"])
def test_accumulation_statistics(K, acc_kb):
    out, o = _acc_run(K, acc_kb)
    ckb = _chunk(K, acc_kb)
    bnd = co.bound(K, o["S"], o["b"], o["r"], o["ref"], "split", L=o["L"], chunk_kb=ckb, out="f32")
    err = np.abs(out - o["ref"])
    assert (err <= bnd).all(), (err - bnd).max()
    bias, rms, se = co.acc_statistics(out, o["ref"], o["S"])
    print("ACC K=%d acc_kb=%d chunk=%d: bias %.3e rms %.3e (se %.1e)" % (K, acc_kb, ckb, bias, rms, se))
    if ckb < K // 64 or K == 64:   # ACC on (or the single-chunk compensation)
        assert abs(bias) <= co.acc_bias_bound(ckb)
        if K <= 576:
            assert rms <= co.acc_rms_bound(K, ckb, o["L"] / o["S"])
    elif K >= 2048:                 # ACC off: the truncation bias must be visible against the ACC bound
        assert bias < -co.acc_bias_bound(1), bias


def test_accumulation_off_by_environment_fails_the_bias_bound(monkeypatch):
    monkeypatch.setenv("B2_NO_ACC", "1")
    out, o = _acc_run(4608, 0)
    bias, rms, se = co.acc_statistics(out, o["ref"], o["S"])
    print("B2_NO_ACC K=4608: bias %.3e rms %.3e" % (bias, rms))
    assert bias < -co.acc_bias_bound(1)


@pytest.mark.parametrize("K", [64, 576])
def test_accumulation_delta_is_visible(K, monkeypatch):
    """B2_ACC_DELTA=0 drops the truncation compensation: the bias moves toward zero-truncation by about one ulp, far
    outside the statistic's own spread."""
    out, o = _acc_run(K, 0)
    b1, _, s1 = co.acc_statistics(out, o["ref"], o["S"])
    monkeypatch.setenv("B2_ACC_DELTA", "0")
    out0, _ = _acc_run(K, 0)
    b0, _, s0 = co.acc_statistics(out0, o["ref"], o["S"])
    print("ACC delta K=%d: bias %.3e (delta 0: %.3e), spread %.1e" % (K, b1, b0, np.hypot(s1, s0)))
    assert b1 - b0 >= 5 * np.hypot(s1, s0)


# ------------------------------------------------------------------------------------------------------------------
# Range monitor
def _range_case(bias_last, res_value=None, force_epi=-1, split=True, out_f32=False):
    B, H, W, Cin, Cout = 1, 7, 9, 64, 80    # M = 63: one ragged tile; Cout_pad 80 with 128-column tiles
    x = np.random.default_rng(0).standard_normal((B, H, W, Cin)).astype(np.float32)
    w = np.zeros((1, 1, Cin, Cout), np.float32)
    bias = np.zeros(Cout, np.float32)
    bias[Cout - 1] = bias_last
    res = None if res_value is None else np.full((B, H, W, Cout), res_value, np.float32)
    out, _, _, flag = _engine().op_conv2d_view(x, w, bias, res, force_epi=force_epi, split=split, out_f32=out_f32)
    return out, flag


@pytest.mark.parametrize("force_epi", [0, 1], ids=["direct", "staged"])
@pytest.mark.parametrize("split", [True, False], ids=["split", "fp16"])
def test_range_monitor_threshold(force_epi, split):
    out, flag = _range_case(65504.0, force_epi=force_epi, split=split)
    assert flag == 0 and (out[..., -1] == 65504.0).all()
    _, flag = _range_case(65510.0, force_epi=force_epi, split=split)
    assert flag == 1


@pytest.mark.parametrize("force_epi", [0, 1], ids=["direct", "staged"])
def test_range_monitor_ignores_rows_past_m(force_epi):
    """Bias 65510 and residual -10 on every real row: real outputs are 65500; the zero-filled rows past M of the last
    tile would compute 65510 and must not count."""
    out, flag = _range_case(65510.0, res_value=-10.0, force_epi=force_epi)
    assert (out[..., -1] == 65500.0).all()
    assert flag == 0


def test_range_monitor_ignores_fp32_outputs():
    out, flag = _range_case(1e6, out_f32=True)
    assert (out[..., -1] == 1e6).all() and flag == 0
