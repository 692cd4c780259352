"""torchreid's OSNet family on the GPU: the InstanceNorm kernel against float64 through b2_op_instance_norm, and the five
models added to osnet_x1_0 (x0.75 / x0.5 / x0.25 widths, osnet_ibn_x1_0, osnet_ain_x1_0) against the reference's golden
features (tests/golden/osnet_family.npz) and the float64 oracle's InstanceNorm stages (tests/osnet_family_oracle.py)."""
import ctypes
import os

import numpy as np
import pytest
import torch

import osnet_family_oracle as oracle

pytestmark = pytest.mark.gpu

NEW = ("osnet_x0_75", "osnet_x0_5", "osnet_x0_25", "osnet_ibn_x1_0", "osnet_ain_x1_0")
PADDED = {"osnet_x0_75": {"conv1": 48, "conv3.0.x1": 72, "conv3.1": 288}, "osnet_x0_25": {"conv1": 16, "conv2.0.x2": 16,
                                                                             "conv3": 96, "conv3.1.x1": 24}}


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "osnet_family.npz"))


@pytest.fixture(scope="module")
def resized(golden_dir):
    return np.load(os.path.join(golden_dir, "osnet.npz"))["resized"]


def _state(name):
    from object_detection_tracking_b200.synth import synth_osnet_family_state
    return synth_osnet_family_state(name, 4321)


# ---- the kernel alone ---------------------------------------------------------------------------------------------------

def op_instance_norm(x, gamma, beta, res=None, relu=False, split=True):
    from object_detection_tracking_b200 import _lib
    lib = _lib.load()
    x = np.ascontiguousarray(x, np.float32)
    B, H, W, C = x.shape
    out = np.empty_like(x)
    r = None if res is None else np.ascontiguousarray(res, np.float32)
    g, b = np.ascontiguousarray(gamma, np.float32), np.ascontiguousarray(beta, np.float32)
    _lib.check(lib.b2_op_instance_norm(0, _lib.ptr(x), None if r is None else _lib.ptr(r), _lib.ptr(g), _lib.ptr(b),
                                       B, H, W, C, int(relu), int(split), _lib.ptr(out)), "b2_op_instance_norm")
    return out


def quantize(x, split):
    """The value the engine's planes hold for x: hi = fp16(x), lo' = fp16((x - hi) * 2048) in split precision."""
    x = np.asarray(x, np.float32)
    hi = x.astype(np.float16).astype(np.float32)
    if not split:
        return hi
    lo = ((x - hi) * np.float32(2048)).astype(np.float16).astype(np.float32)
    return (hi + lo / np.float32(2048)).astype(np.float32)


def ref_instance_norm(x, gamma, beta, res, relu):
    t = torch.from_numpy(x.astype(np.float64)).permute(0, 3, 1, 2)
    y = oracle.instance_norm(t, torch.from_numpy(gamma.astype(np.float64)), torch.from_numpy(beta.astype(np.float64)))
    y = y.permute(0, 2, 3, 1).numpy()
    if res is not None:
        y = y + res.astype(np.float64)
    return np.maximum(y, 0) if relu else y


@pytest.mark.parametrize("split", (True, False))
@pytest.mark.parametrize("hw", ((1, 1), (16, 8), (128, 64)))
@pytest.mark.parametrize("creal", (16, 48, 64, 288))
def test_kernel_matches_float64(split, hw, creal):
    rng = np.random.default_rng(creal * 7 + hw[0])
    C = (creal + 63) // 64 * 64
    B, (H, W) = 3, hw
    x = np.zeros((B, H, W, C), np.float32)
    x[..., :creal] = rng.standard_normal((B, H, W, creal)) * rng.uniform(0.2, 4, creal) + rng.uniform(-3, 3, creal)
    gamma, beta = np.zeros(C, np.float32), np.zeros(C, np.float32)
    gamma[:creal] = rng.uniform(0.8, 1.2, creal)
    beta[:creal] = rng.standard_normal(creal) * 0.05
    res = np.zeros_like(x)
    res[..., :creal] = rng.standard_normal((B, H, W, creal))
    xq, rq = quantize(x, split), quantize(res, split)
    for r, relu in ((None, False), (res, False), (None, True), (res, True)):
        got = op_instance_norm(x, gamma, beta, r, relu, split)
        ref = ref_instance_norm(xq, gamma, beta, None if r is None else rq, relu)
        # output planes round to 2^-22 (split) / 2^-11 (fp16) of the value; float32 statistics add a few ulp
        tol = (4e-6 if split else 2e-3) * max(1.0, np.abs(ref).max())
        assert np.abs(got - ref).max() <= tol, (r is not None, relu, np.abs(got - ref).max())
        assert not got[..., creal:].any()                        # padded channels stay exactly 0


@pytest.mark.parametrize("split", (True, False))
def test_kernel_ill_conditioned_channels(split):
    rng = np.random.default_rng(11)
    B, H, W, C = 2, 16, 8, 64
    x = rng.standard_normal((B, H, W, C)).astype(np.float32)
    x[:, :, :, 3] = 2.5                                          # constant: var 0
    x[..., 5] = (1e3 + 1e-2 * rng.standard_normal((B, H, W))).astype(np.float32)   # mean 1e3, std 1e-2
    x[1, 4, 2, 9] = np.nan                                      # NaN in (image 1, channel 9)
    x[0, 7, 1, 11] = np.inf                                     # inf in (image 0, channel 11)
    gamma = rng.uniform(0.8, 1.2, C).astype(np.float32)
    beta = (rng.standard_normal(C) * 0.05).astype(np.float32)
    got = op_instance_norm(x, gamma, beta, None, False, split)
    with np.errstate(invalid="ignore"):
        xq = quantize(x, split)
        ref = ref_instance_norm(xq, gamma, beta, None, False)
    np.testing.assert_array_equal(got[..., 3], quantize(beta[3], split))                  # finite: beta, as stored
    assert np.isnan(got[1, ..., 9]).all() and np.isfinite(got[0, ..., 9]).all()
    assert not np.isfinite(got[0, ..., 11]).any() and np.isfinite(got[1, ..., 11]).all()
    ok = np.ones((B, C), bool)
    ok[1, 9] = ok[0, 11] = False
    for b in range(B):
        for c in range(C):
            if ok[b, c]:
                # channel 5: the planes hold x to ~2.4e-4 (split) / 0.5 (fp16) absolute at 1e3; the float64 reference
                # reads the same quantised values, so only the kernel's own float32 error remains
                tol = (2e-3 if c == 5 else 4e-6) if split else (0.5 if c == 5 else 2e-3)
                err = np.abs(got[b, ..., c] - ref[b, ..., c]).max()
                assert err <= tol * max(1.0, np.abs(ref[b, ..., c]).max()), (b, c, err)


def test_kernel_refuses_bad_channel_count():
    from object_detection_tracking_b200 import _lib
    x = np.zeros((1, 2, 2, 48), np.float32)
    g = np.ones(48, np.float32)
    with pytest.raises(RuntimeError, match="multiple of 64"):
        _lib.check(_lib.load().b2_op_instance_norm(0, _lib.ptr(x), None, _lib.ptr(g), _lib.ptr(g), 1, 2, 2, 48, 0, 1,
                                                   _lib.ptr(x)), "b2_op_instance_norm")


# ---- the models ---------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", NEW)
def test_split_features_match_reference_and_in_stages_match_oracle(name, golden, resized):
    from object_detection_tracking_b200.reid import ReidEngine
    from object_detection_tracking_b200.synth import osnet_family_in_layers
    eng = ReidEngine(batch=8, precision="split", model=name)
    state = _state(name)
    eng.load_state(state)
    feats = eng.embed(resized)
    ref = golden[name + "/feats"]
    assert feats.shape == ref.shape == (6, 512)
    assert np.abs(feats - ref).max() <= 2e-5 * np.abs(ref).max()
    for stage, creal in PADDED.get(name, {}).items():               # channels past the model's count stay 0
        a = eng.get_activation(stage)
        assert a.shape[-1] == (creal + 63) // 64 * 64 and not a[..., creal:].any() and a[..., :creal].any(), stage
    ins = osnet_family_in_layers(name)
    if ins:
        o_feats, st = oracle.forward(name, state, resized)
        assert np.abs(feats - o_feats).max() <= 2e-5 * np.abs(o_feats).max()
        for scope in ins:
            stage = "conv1" if scope == "conv1.bn" else scope[:-3]
            for s in (stage + ".pre_in", stage):
                got = eng.get_activation(s)[:6]
                want = st[s]
                got = got[..., :want.shape[-1]]
                assert got.shape == want.shape, (s, got.shape, want.shape)
                err = np.abs(got - want).max()
                assert err <= 2e-5 * np.abs(want).max(), (s, err, np.abs(want).max())
    eng.close()


@pytest.mark.parametrize("name", NEW)
def test_fp16_features_are_close(name, golden, resized):
    from object_detection_tracking_b200.reid import ReidEngine
    eng = ReidEngine(batch=6, precision="fp16", model=name)
    eng.load_state(_state(name))
    feats = eng.embed(resized)
    ref = golden[name + "/feats"]
    assert np.abs(feats - ref).max() <= 3e-2 * np.abs(ref).max()
    eng.close()


@pytest.mark.parametrize("name", ("osnet_ibn_x1_0", "osnet_ain_x1_0", "osnet_x0_25"))
def test_features_do_not_depend_on_batch_composition(name, resized):
    from object_detection_tracking_b200.reid import ReidEngine
    state = _state(name)
    rng = np.random.default_rng(3)
    others = rng.integers(0, 256, (32, 256, 128, 3), dtype=np.uint8)
    img = resized[2]
    got = []
    for batch in (1, 8, 32):
        eng = ReidEngine(batch=batch, precision="split", model=name)
        eng.load_state(state)
        got.append(eng.embed(img[None])[0])                       # alone (zero crops pad the batch)
        if batch > 1:
            for slot in (0, batch - 1):                           # among other crops, at the first and last slot
                crops = others[:batch].copy()
                crops[slot] = img
                got.append(eng.embed(crops)[slot])
        eng.close()
    for g in got[1:]:
        np.testing.assert_array_equal(g, got[0])


@pytest.mark.parametrize("name", ("osnet_ain_x1_0", "osnet_x0_25"))
def test_extract_boxes_equals_host_crops(name):
    from object_detection_tracking_b200.reid import FeatureExtractor
    from object_detection_tracking_b200.synth import synth_frame
    ext = FeatureExtractor(model_name=name, batch=4, state_dict=_state(name))
    frame = synth_frame(360, 640, seed=9)
    tlwhs = [(10, 20, 60, 150), (300.7, 40.2, 33, 90), (500, 100, 120, 250), (0, 0, 640, 360), (200, 200, 17, 41)]
    got = ext.extract_boxes(frame, tlwhs).numpy()
    crops = [frame[int(y):int(y) + int(h), int(x):int(x) + int(w), ::-1] for x, y, w, h in tlwhs]
    np.testing.assert_array_equal(got, ext(crops).numpy())


def test_feature_extractor_from_torchreid_checkpoint(tmp_path, golden):
    from object_detection_tracking_b200.reid import FeatureExtractor
    name = "osnet_ain_x1_0"
    ckpt = {"state_dict": {"module." + k: torch.from_numpy(v) for k, v in _state(name).items()}, "epoch": 3}
    path = str(tmp_path / "model.pth.tar")
    torch.save(ckpt, path)
    ext = FeatureExtractor(model_name=name, model_path=path, device="cuda", batch=4)
    rng = np.random.default_rng(5)                                # make_golden.py's crops
    crops = [rng.integers(0, 256, (int(rng.integers(60, 300)), int(rng.integers(30, 160)), 3), dtype=np.uint8)
             for _ in range(6)]
    feats = ext(crops)
    assert isinstance(feats, torch.Tensor) and tuple(feats.shape) == (6, 512)
    ref = golden[name + "/feats"]
    assert np.abs(feats.numpy() - ref).max() <= 2e-5 * np.abs(ref).max()


def test_refusals():
    from object_detection_tracking_b200 import _lib
    from object_detection_tracking_b200.reid import FeatureExtractor, ReidEngine
    state = _state("osnet_ibn_x1_0")
    del state["conv2.0.IN.weight"]
    eng = ReidEngine(batch=2, precision="split", model="osnet_ibn_x1_0")
    with pytest.raises(RuntimeError, match="conv2.0.IN.weight"):
        eng.load_state(state)
    eng.close()
    with pytest.raises(NotImplementedError):
        FeatureExtractor(model_name="osnet_x0_25", image_size=(128, 64), state_dict=_state("osnet_x0_25"))
    with pytest.raises(NotImplementedError):
        FeatureExtractor(model_name="osnet_x2_0", state_dict=_state("osnet_x0_25"))
    lib = _lib.load()
    ctx = ctypes.c_void_p(0)
    assert lib.b2_reid_create_model(ctypes.byref(ctx), 0, 2, 1, 7) != 0
    assert not ctx.value
    assert b"model must be" in lib.b2_last_error()


def test_existing_models_keep_their_launch_counts():
    """The family's builder leaves osnet_x1_0's and resnet101's plans as they were; the IN models add one launch per
    InstanceNorm."""
    from object_detection_tracking_b200.reid import ReidEngine
    n = {}
    for name in ("osnet_x1_0", "osnet_ibn_x1_0", "osnet_ain_x1_0", "osnet_x0_25"):
        eng = ReidEngine(batch=2, precision="split", model=name)
        n[name] = eng.num_launches()
        eng.close()
    assert n["osnet_ibn_x1_0"] == n["osnet_x1_0"] + 3
    assert n["osnet_ain_x1_0"] == n["osnet_x1_0"] + 5
    assert n["osnet_x0_25"] == n["osnet_x1_0"]
