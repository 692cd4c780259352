"""torchreid's ResNet family on the GPU: the IBN-a split InstanceNorm kernel against float64 through
b2_op_instance_norm_split, the grouped 3x3 with torch's padding through b2_op_group_conv2d, and the nine models added to
resnet101 against the reference's golden features (tests/golden/resnet_family.npz) and the float64 oracle's stages
(tests/resnet_family_oracle.py)."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import resnet_family_oracle as oracle

pytestmark = pytest.mark.gpu

NEW = ("resnet18", "resnet34", "resnet50", "resnet152", "resnext50_32x4d", "resnext101_32x8d", "resnet50_fc512",
       "resnet50_ibn_a", "resnet50_ibn_b")
VEHICLE = ("resnet50", "resnext50_32x4d", "resnet50_ibn_a")
GOLDEN = [(n, (256, 128)) for n in NEW] + [(n, (128, 256)) for n in VEHICLE]
DEEP = ("resnet152", "resnext101_32x8d")     # ~100-layer nets: resnet101's bound (test_reid_r101_mask_gpu.py)


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(golden_dir + "/resnet_family.npz")


@pytest.fixture(scope="module")
def crops():
    return {size: oracle.golden_crops(size) for size in ((256, 128), (128, 256))}


def _state(name):
    from object_detection_tracking_b200.synth import synth_resnet_family_state
    return synth_resnet_family_state(name, 2468)


def _ref(golden, name, size):
    return golden[name + ("/feats" if size == (256, 128) else "/feats_128x256")]


# ---- the split InstanceNorm kernel alone ---------------------------------------------------------------------------------

def quantize(x, split):
    """The value the engine's planes hold for x: hi = fp16(x), lo' = fp16((x - hi) * 2048) in split precision."""
    x = np.asarray(x, np.float32)
    hi = x.astype(np.float16).astype(np.float32)
    if not split:
        return hi
    lo = ((x - hi) * np.float32(2048)).astype(np.float16).astype(np.float32)
    return (hi + lo / np.float32(2048)).astype(np.float32)


def op_instance_norm_split(x, gamma, beta, c_norm, split=True):
    from object_detection_tracking_b200 import _lib
    x = np.ascontiguousarray(x, np.float32)
    B, H, W, C = x.shape
    out = np.empty_like(x)
    g, b = np.ascontiguousarray(gamma, np.float32), np.ascontiguousarray(beta, np.float32)
    _lib.check(_lib.load().b2_op_instance_norm_split(0, _lib.ptr(x), _lib.ptr(g), _lib.ptr(b), B, H, W, C, c_norm,
                                                     int(split), _lib.ptr(out)), "b2_op_instance_norm_split")
    return out


def ref_split(xq, gamma, beta, c_norm):
    t = torch.from_numpy(xq.astype(np.float64)).permute(0, 3, 1, 2)
    y = t.clone()
    y[:, :c_norm] = oracle.instance_norm(t[:, :c_norm], torch.from_numpy(gamma.astype(np.float64)),
                                         torch.from_numpy(beta.astype(np.float64)))
    return np.maximum(y.permute(0, 2, 3, 1).numpy(), 0)


@pytest.mark.parametrize("split", (True, False))
@pytest.mark.parametrize("hw", ((1, 1), (7, 5), (128, 64)))
@pytest.mark.parametrize("c_norm,C", ((32, 64), (64, 128), (128, 256)))
def test_split_kernel_matches_float64(split, hw, c_norm, C):
    rng = np.random.default_rng(c_norm + hw[0])
    B, (H, W) = 3, hw
    x = (rng.standard_normal((B, H, W, C)) * rng.uniform(0.2, 4, C) + rng.uniform(-3, 3, C)).astype(np.float32)
    gamma = rng.uniform(0.8, 1.2, c_norm).astype(np.float32)
    beta = (rng.standard_normal(c_norm) * 0.05).astype(np.float32)
    got = op_instance_norm_split(x, gamma, beta, c_norm, split)
    xq = quantize(x, split)
    ref = ref_split(xq, gamma, beta, c_norm)
    tol = (4e-6 if split else 2e-3) * max(1.0, np.abs(ref[..., :c_norm]).max())
    assert np.abs(got[..., :c_norm] - ref[..., :c_norm]).max() <= tol
    np.testing.assert_array_equal(got[..., c_norm:], np.maximum(xq[..., c_norm:], 0))   # pass-through: relu(x), bit for bit


@pytest.mark.parametrize("split", (True, False))
def test_split_kernel_ill_conditioned_channel(split):
    rng = np.random.default_rng(12)
    B, H, W, C, c_norm = 2, 16, 8, 64, 32
    x = rng.standard_normal((B, H, W, C)).astype(np.float32)
    x[..., 3] = 2.5                                                       # constant: var 0 -> beta
    x[..., 5] = (1e3 + 1e-2 * rng.standard_normal((B, H, W))).astype(np.float32)   # mean 1e3, std 1e-2
    x[..., 40] = 1e3                                                      # a large pass-through channel
    gamma = rng.uniform(0.8, 1.2, c_norm).astype(np.float32)
    beta = (rng.standard_normal(c_norm) * 0.05).astype(np.float32)
    got = op_instance_norm_split(x, gamma, beta, c_norm, split)
    xq = quantize(x, split)
    ref = ref_split(xq, gamma, beta, c_norm)
    np.testing.assert_array_equal(got[..., 3], np.maximum(quantize(beta[3], split), 0))
    for c in range(c_norm):
        # channel 5: the planes hold x to ~2.4e-4 (split) / 0.5 (fp16) absolute at 1e3, and the float64 reference reads the
        # same quantised values, so only the kernel's own float32 error remains (as test_osnet_family_gpu.py)
        tol = (2e-3 if c == 5 else 4e-6) if split else (0.5 if c == 5 else 2e-3)
        assert np.abs(got[..., c] - ref[..., c]).max() <= tol * max(1.0, np.abs(ref[..., c]).max()), c
    np.testing.assert_array_equal(got[..., c_norm:], np.maximum(xq[..., c_norm:], 0))


def test_split_kernel_refusals():
    from object_detection_tracking_b200 import _lib
    x = np.zeros((1, 2, 2, 64), np.float32)
    g = np.ones(64, np.float32)
    for C, c_norm in ((48, 24), (64, 0), (64, 12), (64, 72)):
        with pytest.raises(RuntimeError, match="c_norm"):
            _lib.check(_lib.load().b2_op_instance_norm_split(0, _lib.ptr(x), _lib.ptr(g), _lib.ptr(g), 1, 2, 2, C, c_norm,
                                                             1, _lib.ptr(x)), "b2_op_instance_norm_split")


# ---- the grouped 3x3 with torch's padding ----------------------------------------------------------------------------------

@pytest.mark.parametrize("C,groups,H,W", ((128, 32, 64, 32), (256, 32, 32, 64), (1024, 32, 16, 8), (2048, 32, 8, 16)))
@pytest.mark.parametrize("stride", (1, 2))
def test_grouped_conv_torch_padding_single_op(C, groups, H, W, stride):
    """ResNeXt's conv2 (groups 32, 4 to 64 channels per group) with torch's pad 1: stride 2 on even extents runs as pads
    (1, 0), the same convolution.  Against torch float64."""
    from object_detection_tracking_b200 import _lib
    rng = np.random.default_rng(C + stride)
    B, cg = 2, C // groups
    x = rng.standard_normal((B, H, W, C)).astype(np.float32)
    w = (rng.standard_normal((C, cg, 3, 3)) / np.sqrt(9 * cg)).astype(np.float32)     # torch OIHW
    bias = (rng.standard_normal(C) * 0.1).astype(np.float32)
    ref = F.conv2d(torch.from_numpy(x.astype(np.float64)).permute(0, 3, 1, 2), torch.from_numpy(w.astype(np.float64)),
                   torch.from_numpy(bias.astype(np.float64)), stride=stride, padding=1, groups=groups)
    ref = ref.permute(0, 2, 3, 1).numpy()
    hwio = np.ascontiguousarray(w.transpose(2, 3, 1, 0))                               # [3][3][C/groups][C]
    pads = (1, 0, 1, 0) if stride == 2 else (1, 1, 1, 1)
    out = np.zeros((B, H // stride, W // stride, C), np.float32)
    _lib.check(_lib.load().b2_op_group_conv2d(0, _lib.ptr(x), _lib.ptr(hwio), _lib.ptr(bias), None, B, H, W, C, 3, 3,
                                              groups, stride, 1, *pads, 0, 0, 1, _lib.ptr(out)), "b2_op_group_conv2d")
    assert np.abs(out - ref).max() <= 2e-5 * np.abs(ref).max()


# ---- the models --------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name,size", GOLDEN)
def test_split_features_match_reference(name, size, golden, crops):
    from object_detection_tracking_b200.reid import ReidEngine
    from object_detection_tracking_b200.synth import resnet_family_in_layers
    eng = ReidEngine(batch=8, precision="split", model=name, image_size=size)
    state = _state(name)
    eng.load_state(state)
    resized = crops[size][1]
    feats = eng.embed(resized)
    ref = _ref(golden, name, size)
    assert feats.shape == ref.shape == (6, eng.feat_dim)
    bound = 3e-5 if name in DEEP else 2e-5
    assert np.abs(feats - ref).max() <= bound * np.abs(ref).max()
    ins = resnet_family_in_layers(name)
    if ins or name.startswith("resnext"):
        o_feats, st = oracle.forward(name, state, resized)
        stages = []
        for scope in ins:   # every InstanceNorm's input and output
            stage = "conv1" if scope == "bn1" else scope[:-3]
            stages += [stage + ".pre_in", stage]
        if name.startswith("resnext"):   # the stride-2 grouped layers (pads (1, 0)); resnext101's layer4 has 64-ch groups
            stages += ["layer2.0", "layer4.0"]
        for s in stages:
            got = eng.get_activation(s)[:6]
            want = st[s]
            assert got.shape == want.shape, (s, got.shape, want.shape)
            err = np.abs(got - want).max()
            assert err <= bound * np.abs(want).max(), (s, err, np.abs(want).max())
    eng.close()


@pytest.mark.parametrize("name,size", GOLDEN)
def test_fp16_features_are_close(name, size, golden, crops):
    from object_detection_tracking_b200.reid import ReidEngine
    eng = ReidEngine(batch=6, precision="fp16", model=name, image_size=size)
    eng.load_state(_state(name))
    feats = eng.embed(crops[size][1])
    ref = _ref(golden, name, size)
    assert np.abs(feats - ref).max() <= 3e-2 * np.abs(ref).max()
    eng.close()


@pytest.mark.parametrize("name", ("resnet50_ibn_a", "resnext50_32x4d", "resnet50_fc512"))
def test_features_do_not_depend_on_batch_composition(name, crops):
    from object_detection_tracking_b200.reid import ReidEngine
    state = _state(name)
    rng = np.random.default_rng(3)
    others = rng.integers(0, 256, (32, 256, 128, 3), dtype=np.uint8)
    img = crops[(256, 128)][1][2]
    got = []
    for batch in (1, 8, 32):
        eng = ReidEngine(batch=batch, precision="split", model=name)
        eng.load_state(state)
        got.append(eng.embed(img[None])[0])                       # alone (zero crops pad the batch)
        if batch > 1:
            for slot in (0, batch - 1):                           # among other crops, at the first and last slot
                crops_b = others[:batch].copy()
                crops_b[slot] = img
                got.append(eng.embed(crops_b)[slot])
        eng.close()
    for g in got[1:]:
        np.testing.assert_array_equal(g, got[0])


@pytest.mark.parametrize("name,size", (("resnet50_ibn_a", (256, 128)), ("resnext50_32x4d", (128, 256))))
def test_extract_boxes_equals_host_crops(name, size):
    from object_detection_tracking_b200.reid import FeatureExtractor
    from object_detection_tracking_b200.synth import synth_frame
    ext = FeatureExtractor(model_name=name, image_size=size, batch=4, state_dict=_state(name))
    frame = synth_frame(360, 640, seed=9)
    tlwhs = [(10, 20, 60, 150), (300.7, 40.2, 33, 90), (500, 100, 120, 250), (0, 0, 640, 360), (200, 200, 17, 41)]
    got = ext.extract_boxes(frame, tlwhs).numpy()
    host = [frame[int(y):int(y) + int(h), int(x):int(x) + int(w), ::-1] for x, y, w, h in tlwhs]
    np.testing.assert_array_equal(got, ext(host).numpy())


def test_feature_extractor_from_torchreid_checkpoint(tmp_path, golden, crops):
    from object_detection_tracking_b200.reid import FeatureExtractor
    name = "resnet50_ibn_b"
    ckpt = {"state_dict": {"module." + k: torch.from_numpy(v) for k, v in _state(name).items()}, "epoch": 3}
    path = str(tmp_path / "model.pth.tar")
    torch.save(ckpt, path)
    ext = FeatureExtractor(model_name=name, model_path=path, device="cuda", batch=4)
    feats = ext(crops[(256, 128)][0])
    assert isinstance(feats, torch.Tensor) and tuple(feats.shape) == (6, 2048)
    ref = golden[name + "/feats"]
    assert np.abs(feats.numpy() - ref).max() <= 2e-5 * np.abs(ref).max()


def test_refusals():
    from object_detection_tracking_b200 import _lib
    from object_detection_tracking_b200.reid import FeatureExtractor, ReidEngine
    state = _state("resnet50_ibn_a")
    del state["layer2.1.bn1.IN.weight"]
    eng = ReidEngine(batch=2, precision="split", model="resnet50_ibn_a")
    with pytest.raises(RuntimeError, match="layer2.1.bn1.IN.weight"):
        eng.load_state(state)
    eng.close()
    with pytest.raises(NotImplementedError):
        FeatureExtractor(model_name="se_resnet50", state_dict=state)
    with pytest.raises(NotImplementedError):
        FeatureExtractor(model_name="resnet50", image_size=(384, 128), state_dict=_state("resnet50"))
    lib = _lib.load()
    for name, h, w in ((b"resnet200", 256, 128), (b"resnet50", 384, 128), (b"resnet101", 256, 128),
                       (b"osnet_x1_0", 128, 256)):
        ctx = ctypes.c_void_p(0)
        assert lib.b2_reid_create_named(ctypes.byref(ctx), 0, 2, 1, name, h, w) != 0
        assert not ctx.value
        err = lib.b2_last_error()
        assert b"is not built" in err and b"resnext101_32x8d at 256x128 or 128x256" in err, err


def test_existing_plans_are_unchanged(golden_dir):
    """The family's builder leaves every existing model's plan as the parent's (launch counts measured there), and the
    named entry point builds resnet101 exactly as model id 1 does."""
    from object_detection_tracking_b200 import _lib
    from object_detection_tracking_b200.reid import ReidEngine
    from object_detection_tracking_b200.synth import synth_resnet101_reid_state
    parent = {"osnet_x1_0": 182, "resnet101": 107, "osnet_x0_75": 182, "osnet_x0_5": 182, "osnet_x0_25": 182,
              "osnet_ibn_x1_0": 185, "osnet_ain_x1_0": 187}
    for name, n in parent.items():
        eng = ReidEngine(batch=2, precision="split", model=name)
        assert eng.num_launches() == n, (name, eng.num_launches())
        eng.close()
    r101 = np.load(golden_dir + "/resnet101_reid.npz")
    lib = _lib.load()
    ctx = ctypes.c_void_p(0)
    _lib.check(lib.b2_reid_create_model(ctypes.byref(ctx), 0, 4, 1, 1), "b2_reid_create_model")
    by_id = ReidEngine.__new__(ReidEngine)
    by_id.lib, by_id._ctx, by_id.batch, by_id.image_size, by_id.feat_dim = lib, ctx, 4, (128, 256), 2048
    named = ReidEngine(batch=4, precision="split", model="resnet101")
    state = synth_resnet101_reid_state(2468)
    feats = []
    for eng in (by_id, named):
        eng.load_state(state)
        feats.append(eng.embed(r101["resized"]))
        assert eng.num_launches() == parent["resnet101"]
        eng.close()
    np.testing.assert_array_equal(feats[0], feats[1])
    assert np.abs(feats[1] - r101["feats"]).max() <= 3e-5 * np.abs(r101["feats"]).max()


def test_new_models_launch_counts():
    """One launch per conv, plus one per InstanceNorm: IBN-a adds the 13 split norms of layer1-3, IBN-b three."""
    from object_detection_tracking_b200.reid import ReidEngine
    n = {}
    for name in ("resnet50", "resnet50_ibn_a", "resnet50_ibn_b", "resnext50_32x4d", "resnet50_fc512"):
        eng = ReidEngine(batch=2, precision="split", model=name)
        n[name] = eng.num_launches()
        eng.close()
    assert n["resnet50_ibn_a"] == n["resnet50"] + 13
    assert n["resnet50_ibn_b"] == n["resnet50"] + 3
    assert n["resnext50_32x4d"] == n["resnet50"]
    assert n["resnet50_fc512"] == n["resnet50"] + 2        # gap + row conversion as two launches, then the fc
