"""Deformable-conv detector (`use_deformable`) on the host: the oracle's sampler against an independent float64 numpy loop,
a numpy restatement of the reference helper's whole op sequence (bit-exact against the oracle at batch 1, and its
channel-major batch mixing at batch 2), the tap table with zero offsets, the block rule, the weight manifest and the
importer's refusals, the use_dilations refusal, the synthetic weights shared with the plain model, and the offsets'
non-degeneracy."""
import numpy as np
import pytest
import torch

from object_detection_tracking_b200.config import make_config
from object_detection_tracking_b200.synth import deformable_blocks, frcnn_weight_shapes, synth_frame, synth_weights
import deform_oracle
from oracle import frcnn

DF = dict(use_deformable=True, use_dilations=False)
F32 = np.float32


def np_sample_loop(l, off):
    """float64 loop over (image, pixel, tap, corner): l [N, C, H, W], off [N, 18, Ho, Wo] -> [N, 9, C, Ho, Wo].  Tap k's
    base is (2i - 1, 2j - 1) + the k-th pair of the row-major [2, 3, 3] meshgrid stack; each corner weighs
    (1 - |y - yc|) (1 - |x - xc|)."""
    N, C, H, W = l.shape
    Ho, Wo = off.shape[2:]
    grid = np.stack(np.meshgrid(np.arange(3), np.arange(3), indexing="ij")).reshape(-1, 2)
    out = np.zeros((N, 9, C, Ho, Wo))
    for n in range(N):
        for i in range(Ho):
            for j in range(Wo):
                for k in range(9):
                    y = min(max(2 * i - 1 + grid[k][0] + float(off[n, 2 * k, i, j]), 0.0), H - 1.0)
                    x = min(max(2 * j - 1 + grid[k][1] + float(off[n, 2 * k + 1, i, j]), 0.0), W - 1.0)
                    for yc in {int(np.floor(y)), int(np.ceil(y))}:
                        for xc in {int(np.floor(x)), int(np.ceil(x))}:
                            out[n, k, :, i, j] += (1 - abs(y - yc)) * (1 - abs(x - xc)) * l[n, :, yc, xc]
    return out


def np_helper(inputs, offsets):
    """deformable_conv2d's sampling (nn.py:1655-1686) + _tf_batch_map_offsets (deformable_helper.py:99-137) in numpy,
    op for op in float32: inputs [b, h, w, c], offsets [b, h, w, 18] at every input position -> [b, h, w, 9, c]."""
    b, h, w, c = inputs.shape
    initial = np.stack(np.meshgrid(np.arange(3), np.arange(3), indexing="ij")).reshape(-1, 2)      # [9, 2]
    initial = np.tile(initial[None, None], (h, w, 1, 1)).astype(F32)
    grid = np.stack(np.meshgrid(np.arange(-1, h - 1), np.arange(-1, w - 1), indexing="ij"), -1).astype(F32)
    grid_offset = np.tile(grid[:, :, None], (1, 1, 9, 1)) + initial                                  # [h, w, 9, 2]
    x = inputs.transpose(0, 3, 1, 2).reshape(-1, h, w)                                               # _to_bc_h_w: b * c + ch
    off = offsets.reshape(b, h, w, 9, 2)
    coords = np.tile(grid_offset[None], (b, 1, 1, 1, 1)) + off
    coords = np.stack([np.clip(coords[..., 0], F32(0), F32(h - 1)), np.clip(coords[..., 1], F32(0), F32(w - 1))], -1)
    coords = np.tile(coords, (c, 1, 1, 1, 1))                                                        # index ch * b + image
    lt = np.floor(coords).astype(np.int32)
    rb = np.ceil(coords).astype(np.int32)
    lb = np.stack([lt[..., 0], rb[..., 1]], -1)
    rt = np.stack([rb[..., 0], lt[..., 1]], -1)
    idx = np.arange(b * c)[:, None, None, None]
    val = lambda q: x[idx, q[..., 0], q[..., 1]]
    v_lt, v_rb, v_lb, v_rt = val(lt), val(rb), val(lb), val(rt)
    f = (coords - lt.astype(F32)).astype(F32)
    t = v_lt + (v_rt - v_lt) * f[..., 0]
    bt = v_lb + (v_rb - v_lb) * f[..., 0]
    mapped = t + (bt - t) * f[..., 1]                                                                # [b*c, h, w, 9]
    return mapped.reshape(b, c, h, w, 9).transpose(0, 2, 3, 4, 1)


def _inputs(rng, N, C, H, W, scale=1.5):
    l = rng.standard_normal((N, C, H, W)).astype(F32)
    off = (rng.standard_normal((N, 18, H, W)) * scale).astype(F32)
    off[:, :, ::3, ::2] = np.round(off[:, :, ::3, ::2])                     # integers: y0 == y1
    off[:, 0, 1::4, :] = F32(40.0)                                          # beyond the bottom border
    return l, off


@pytest.mark.parametrize("H,W", [(7, 9), (8, 6)])
def test_oracle_sampler_matches_float64_loop(H, W):
    rng = np.random.default_rng(H * 10 + W)
    l, off = _inputs(rng, 2, 5, H, W)
    off = off[:, :, ::2, ::2]
    with frcnn.exact():
        got = deform_oracle.sample(torch.from_numpy(l.astype(np.float64)), torch.from_numpy(off.astype(np.float64)))
    ref = np_sample_loop(l, off)
    assert got.shape == ref.shape == (2, 9, 5, (H + 1) // 2, (W + 1) // 2)
    assert np.abs(got.numpy() - ref).max() < 1e-12


@pytest.mark.parametrize("H,W", [(7, 9), (10, 12)])
def test_helper_restatement_equals_oracle_bit_for_bit_at_batch1(H, W):
    rng = np.random.default_rng(H + W)
    l, off = _inputs(rng, 1, 6, H, W)
    helper = np_helper(l.transpose(0, 2, 3, 1), off.transpose(0, 2, 3, 1))[:, ::2, ::2]          # the conv3d's stride
    s = deform_oracle.sample(torch.from_numpy(l), torch.from_numpy(off[:, :, ::2, ::2])).numpy()
    got = s.transpose(0, 3, 4, 1, 2)
    assert got.dtype == helper.dtype == F32 and got.shape == helper.shape
    assert np.array_equal(got.view(np.uint32), helper.view(np.uint32))


def test_helper_mixes_images_channel_major_at_batch2():
    """The reference's batch graph samples channel c of image b at the offsets of image (b * C + c) mod B; the engine and
    the oracle use image b's own offsets (DESIGN 4)."""
    rng = np.random.default_rng(7)
    B, C, H, W = 2, 5, 7, 8
    l, off = _inputs(rng, B, C, H, W)
    helper = np_helper(l.transpose(0, 2, 3, 1), off.transpose(0, 2, 3, 1))[:, ::2, ::2]
    own = deform_oracle.sample(torch.from_numpy(l), torch.from_numpy(off[:, :, ::2, ::2])).numpy()
    mixed = 0
    for b in range(B):
        for c in range(C):
            src = (b * C + c) % B
            s = deform_oracle.sample(torch.from_numpy(l[b:b + 1, c:c + 1]),
                                     torch.from_numpy(off[src:src + 1, :, ::2, ::2])).numpy()
            assert np.array_equal(helper[b, :, :, :, c], s[0, :, 0].transpose(1, 2, 0))
            if src != b:
                mixed += 1
                assert np.abs(helper[b, :, :, :, c] - own[b, :, c].transpose(1, 2, 0)).max() > 0.1
    assert mixed == 4


def test_zero_offsets_give_the_tap_table_with_border_replication():
    rng = np.random.default_rng(3)
    C, H, W = 4, 8, 10
    l = rng.standard_normal((1, C, H, W)).astype(F32)
    off = np.zeros((1, 18, H // 2, W // 2), F32)
    s = deform_oracle.sample(torch.from_numpy(l), torch.from_numpy(off)).numpy()
    assert deform_oracle.TAP_BASE == ((0, 0), (0, 1), (1, 1), (2, 2), (2, 0), (1, 2), (0, 1), (2, 0), (1, 2))
    for k, (by, bx) in enumerate(deform_oracle.TAP_BASE):
        for i in range(H // 2):
            for j in range(W // 2):
                y, x = min(max(2 * i - 1 + by, 0), H - 1), min(max(2 * j - 1 + bx, 0), W - 1)
                assert np.array_equal(s[0, k, :, i, j], l[0, :, y, x])
    # not the plain stride-2 3x3 conv of the bottleneck (pad [1, 0], VALID), despite the comment at nn.py:477-478
    w = (rng.standard_normal((3, 3, C, 6)) / 6).astype(F32)
    with frcnn.exact():
        d = deform_oracle.deform_conv(torch.from_numpy(s.astype(np.float64)), w)
        plain = frcnn._conv(torch.from_numpy(l.astype(np.float64)), w, stride=2, pad=(1, 0, 1, 0))
    assert d.shape == plain.shape and float((d - plain).abs().max()) > 0.1


@pytest.mark.parametrize("blocks,extra,expect", [
    ((3, 4, 23, 3), dict(), ["group3/block0"]),
    ((3, 4, 6, 3), dict(), ["group3/block0"]),
    ((1, 1, 2, 1), dict(), ["group1/block0", "group2/block0", "group3/block0"]),
    ((1, 1, 2, 1), dict(use_resnext=True), []),
    ((1, 1, 2, 1), dict(use_deformable=False), []),
])
def test_block_rule(blocks, extra, expect):
    cfg = make_config(resnet_num_block=blocks, **dict(DF, **extra))
    assert [p for p, _ in deformable_blocks(cfg)] == expect
    oracle = ["group%d/block%d" % (g, i) for g, n in enumerate(blocks) for i in range(n)
              if deform_oracle.is_deformable(cfg, g, i, n)]
    assert oracle == expect


@pytest.mark.parametrize("extra", [dict(), dict(use_gn=True), dict(use_se=True)])
def test_manifest_lists_the_offset_convs_and_no_conv2_norm(extra):
    cfg = make_config(resnet_num_block=(1, 1, 2, 1), **DF, **extra)
    sh = frcnn_weight_shapes(cfg)
    w = synth_weights(cfg, 11)
    assert sorted(sh) == sorted(w)
    for k, v in w.items():
        assert tuple(v.shape) == tuple(sh[k]), k
    for p, c in (("group1/block0", 128), ("group2/block0", 256), ("group3/block0", 512)):
        assert sh[p + "/conv2_offset/W"] == (3, 3, c, 18) and sh[p + "/conv2_offset/b"] == (18,)
        assert sh[p + "/conv2/W"] == (3, 3, c, c)
        assert not any(k.startswith(p + "/conv2/") and not k.endswith("/W") for k in sh)
        assert (p + "/conv1/" + ("gn/gamma" if extra.get("use_gn") else "bn/gamma")) in sh
    assert "group2/block1/conv2/" + ("gn/gamma" if extra.get("use_gn") else "bn/gamma") in sh
    assert not any("conv2_offset" in k for k in frcnn_weight_shapes(make_config(resnet_num_block=(1, 1, 2, 1))))
    rx = make_config(resnet_num_block=(1, 1, 2, 1), use_resnext=True, **DF, **extra)
    assert not any("conv2_offset" in k for k in frcnn_weight_shapes(rx))


def test_check_weights_refuses_by_name():
    from object_detection_tracking_b200.backend import check_weights
    cfg, plain = make_config(**DF), make_config(use_dilations=False)
    w = synth_weights(cfg, 5)
    check_weights(cfg, w)
    with pytest.raises(ValueError) as e:                      # a plain checkpoint: no offset conv
        check_weights(cfg, synth_weights(plain, 5))
    assert "group3/block0/conv2_offset/W" in str(e.value) and "group3/block0/conv2_offset/b" in str(e.value)
    with pytest.raises(ValueError) as e:                      # a deformable checkpoint in a plain model: no conv2/bn
        check_weights(plain, w)
    assert "group3/block0/conv2/bn/gamma" in str(e.value)
    partial = {k: v for k, v in w.items() if k != "group3/block0/conv2_offset/b"}
    with pytest.raises(ValueError, match="group3/block0/conv2_offset/b"):
        check_weights(cfg, partial)


def test_use_dilations_is_refused_by_the_oracle():
    cfg = make_config(resnet_num_block=(1, 1, 2, 1), max_size=128, short_edge_size=96, use_deformable=True)
    assert cfg.use_dilations
    with pytest.raises(ValueError, match="use_dilations"):
        deform_oracle.forward(cfg, synth_weights(cfg, 2), synth_frame(96, 128, 1).astype(F32), stages=False)


def test_config_and_abi_carry_use_deformable():
    from object_detection_tracking_b200 import _lib
    assert make_config().use_deformable is False
    assert _lib.make_config(make_config(), 1, 192, 256).use_deformable == 0
    assert _lib.make_config(make_config(**DF), 1, 192, 256).use_deformable == 1
    assert _lib.B2Config._fields_[-1] == ("use_deformable", _lib.c_int32)


@pytest.mark.parametrize("extra", [dict(), dict(use_gn=True, use_conv_frcnn_head=True), dict(use_se=True)])
@pytest.mark.parametrize("blocks", [(3, 4, 23, 3), (1, 1, 2, 1)])
def test_seed_arrays_shared_with_the_plain_model_are_unchanged(blocks, extra):
    base = dict(resnet_num_block=blocks, use_dilations=False, **extra)
    a = synth_weights(make_config(**base), 1234)
    b = synth_weights(make_config(use_deformable=True, **base), 1234)
    blk = [p for p, _ in deformable_blocks(make_config(use_deformable=True, **base))]
    norm = "gn" if extra.get("use_gn") else "bn"
    assert sorted(set(a) - set(b)) == sorted(k for k in a if any(k.startswith(p + "/conv2/%s/" % norm) for p in blk))
    assert sorted(set(b) - set(a)) == sorted(p + "/conv2_offset/" + s for p in blk for s in ("W", "b"))
    for k in set(a) & set(b):
        assert a[k].tobytes() == b[k].tobytes(), k


def _offset_stats(cfg, H, W, seed):
    Wt = synth_weights(cfg, 1234)
    x = frcnn.preprocess(synth_frame(H, W, seed).astype(F32))
    deform_oracle.LAST.clear()
    deform_oracle.backbone(x, Wt, cfg)
    stats = {}
    for p, _ in deformable_blocks(cfg):
        off = deform_oracle.LAST[p + "/conv2_offset"][0]                      # [Ho, Wo, 18]
        Ho, Wo = off.shape[:2]
        h, w = 2 * Ho, 2 * Wo                                                 # the even maps the backbone sees
        by = np.array([b[0] for b in deform_oracle.TAP_BASE], F32)
        bx = np.array([b[1] for b in deform_oracle.TAP_BASE], F32)
        y = (2 * np.arange(Ho, dtype=F32)[:, None, None] - 1 + by) + off[..., 0::2]
        x = (2 * np.arange(Wo, dtype=F32)[None, :, None] - 1 + bx) + off[..., 1::2]
        yc, xc = np.clip(y, 0, h - 1), np.clip(x, 0, w - 1)
        stats[p] = dict(fractional=float(((yc != np.floor(yc)) | (xc != np.floor(xc))).mean()),
                        y_low=float((y < 0).mean()), y_high=float((y > h - 1).mean()),
                        x_low=float((x < 0).mean()), x_high=float((x > w - 1).mean()),
                        beyond_one=float((np.abs(off) > 1).mean()), max_abs=float(np.abs(off).max()))
    return stats


@pytest.mark.parametrize("blocks,H,W", [((3, 4, 23, 3), 192, 256), ((1, 1, 2, 1), 192, 256)])
def test_synthetic_offsets_are_not_degenerate(blocks, H, W):
    """Over every deformable block: at least 90 % of the samples fractional, at least 0.5 % of them clamped at each of the
    four borders (only the outer rows / columns can be, about 1 / Ho of the samples), at least 10 % of the offsets beyond
    one pixel and some beyond two."""
    for p, s in _offset_stats(make_config(resnet_num_block=blocks, **DF), H, W, 3).items():
        assert s["fractional"] > 0.9, (p, s)
        for k in ("y_low", "y_high", "x_low", "x_high"):
            assert s[k] > 0.005, (p, k, s)
        assert s["beyond_one"] > 0.1 and s["max_abs"] > 2.0, (p, s)
