"""CPU checks of torchreid's OSNet family support: the float64 oracle (tests/osnet_family_oracle.py) against the reference's
golden features (tests/golden/make_golden_osnet_family.py), the synthetic state dicts against the reference model's
state_dict shapes, and where InstanceNorm and the bare conv3 sit."""
import json
import os

import numpy as np
import pytest
import torch

from object_detection_tracking_b200.synth import (OSNET_FAMILY, osnet_family_in_layers, osnet_family_param_shapes,
                                                  osnet_param_shapes, synth_osnet_family_state)

import osnet_family_oracle as oracle

NEW = ("osnet_x0_75", "osnet_x0_5", "osnet_x0_25", "osnet_ibn_x1_0", "osnet_ain_x1_0")


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "osnet_family.npz"))


@pytest.fixture(scope="module")
def resized(golden_dir):
    return np.load(os.path.join(golden_dir, "osnet.npz"))["resized"]


@pytest.mark.parametrize("name", NEW)
def test_oracle_float32_matches_reference_features(name, golden, resized):
    feats, _ = oracle.forward(name, synth_osnet_family_state(name, 4321), resized, dtype=torch.float32)
    ref = golden[name + "/feats"]
    assert feats.shape == ref.shape == (6, 512)
    assert np.abs(feats - ref).max() <= 2e-5 * np.abs(ref).max()


def test_oracle_reproduces_osnet_x1_0_golden(golden_dir, resized):
    from object_detection_tracking_b200.synth import synth_osnet_state
    feats, _ = oracle.forward("osnet_x1_0", synth_osnet_state(4321), resized, dtype=torch.float32)
    ref = np.load(os.path.join(golden_dir, "osnet.npz"))["feats"]
    assert np.abs(feats - ref).max() <= 2e-5 * np.abs(ref).max()


@pytest.mark.parametrize("name", NEW)
def test_synth_shapes_match_reference_model(name, golden_dir):
    with open(os.path.join(golden_dir, "osnet_family_state_shapes.json")) as f:
        ref = {k: tuple(v) for k, v in json.load(f)[name].items()}
    assert ref == osnet_family_param_shapes(name)
    assert set(synth_osnet_family_state(name, 1)) == set(ref)


def test_family_table_restates_osnet_x1_0():
    assert osnet_family_param_shapes("osnet_x1_0") == osnet_param_shapes()


@pytest.mark.parametrize("name", NEW)
def test_states_are_seeded_and_deterministic(name):
    a, b, c = synth_osnet_family_state(name, 7), synth_osnet_family_state(name, 7), synth_osnet_family_state(name, 8)
    assert all(v.dtype == np.float32 for v in a.values())
    for k in a:
        np.testing.assert_array_equal(a[k], b[k])
    assert any(not np.array_equal(a[k], c[k]) for k in a)
    for scope in osnet_family_in_layers(name):          # gamma ~ U(0.8, 1.2), beta ~ N(0, 0.05)
        g, bt = a[scope + ".weight"], a[scope + ".bias"]
        assert g.min() >= 0.8 and g.max() <= 1.2 and np.abs(bt).max() < 0.5


def test_instance_norm_and_bare_conv3_placement():
    shapes = {n: osnet_family_param_shapes(n) for n in OSNET_FAMILY}
    for n in ("osnet_x1_0", "osnet_x0_75", "osnet_x0_5", "osnet_x0_25"):
        assert osnet_family_in_layers(n) == []
    assert osnet_family_in_layers("osnet_ibn_x1_0") == ["conv1.bn", "conv2.0.IN", "conv2.1.IN"]
    assert osnet_family_in_layers("osnet_ain_x1_0") == ["conv1.bn", "conv2.0.IN", "conv2.1.IN", "conv3.1.IN",
                                                        "conv4.0.IN"]
    ain = shapes["osnet_ain_x1_0"]
    for blk, bare in (("conv2.0", True), ("conv2.1", True), ("conv3.0", False), ("conv3.1", True), ("conv4.0", True),
                      ("conv4.1", False)):
        assert (blk + ".conv3.bn.weight" not in ain) == bare         # OSBlockINin's conv3 has no BN
        assert (blk + ".IN.weight" in ain) == bare
        assert blk + ".conv2.3.layers.3.conv1.weight" in ain
    assert "pool2.0.conv.weight" in ain and "conv2.2.0.conv.weight" not in ain
    ibn = shapes["osnet_ibn_x1_0"]
    assert all(k + ".conv3.bn.weight" in ibn for k in ("conv2.0", "conv2.1"))   # IBN keeps conv3's BN
    assert "conv1.bn.running_mean" not in ibn and "conv1.bn.running_mean" in shapes["osnet_x1_0"]
    # widths: mid = cout / 4, gate reduction mid // 16 (1 for mid 16 and 24), conv5 / fc from channels[3]
    q = shapes["osnet_x0_25"]
    assert q["conv2.0.gate.fc1.weight"] == (1, 16, 1, 1) and q["conv3.0.gate.fc1.weight"] == (1, 24, 1, 1)
    assert q["conv5.conv.weight"] == (128, 128, 1, 1) and q["fc.0.weight"] == (512, 128)
    assert shapes["osnet_x0_75"]["conv3.1.conv3.conv.weight"] == (288, 72, 1, 1)


@pytest.mark.parametrize("name", ("osnet_ibn_x1_0", "osnet_ain_x1_0"))
def test_oracle_stage_names_and_in_stages(name, resized):
    _, st = oracle.forward(name, synth_osnet_family_state(name, 4321), resized[:1])
    ins = [s for s in osnet_family_in_layers(name)]
    pre = sorted(k for k in st if k.endswith(".pre_in"))
    assert pre == sorted(("conv1" if s == "conv1.bn" else s[:-3]) + ".pre_in" for s in ins)
    assert st["conv1"].shape == (1, 128, 64, 64) and st["conv5"].shape == (1, 16, 8, 512)
    assert {"maxpool", "conv2.0", "conv2.1", "conv2.t", "conv2", "conv3", "conv4.1"} <= set(st)


def test_instance_norm_restatement_matches_torch():
    rng = np.random.default_rng(0)
    x = torch.from_numpy(rng.standard_normal((2, 5, 7, 3)) * 3 + 10)
    w, b = torch.from_numpy(rng.uniform(0.8, 1.2, 5)), torch.from_numpy(rng.standard_normal(5) * 0.05)
    m = torch.nn.InstanceNorm2d(5, affine=True).double().eval()
    with torch.no_grad():
        m.weight.copy_(w)
        m.bias.copy_(b)
        ref = m(x)
    assert torch.allclose(oracle.instance_norm(x, w, b), ref, rtol=0, atol=1e-12)
