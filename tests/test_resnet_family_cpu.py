"""CPU checks of torchreid's ResNet family support: the synthetic state dicts against the reference model's state_dict
shapes (tests/golden/make_golden_resnet_family.py), the float32 oracle (tests/resnet_family_oracle.py) against the
reference's golden features at both crop sizes, and the oracle's IBN-a / IBN-b norms against torch's modules."""
import json
import os

import numpy as np
import pytest
import torch

from object_detection_tracking_b200.synth import (RESNET_FAMILY, resnet101_reid_param_shapes, resnet_family_in_layers,
                                                  resnet_family_param_shapes, synth_resnet_family_state)

import resnet_family_oracle as oracle

NEW = ("resnet18", "resnet34", "resnet50", "resnet152", "resnext50_32x4d", "resnext101_32x8d", "resnet50_fc512",
       "resnet50_ibn_a", "resnet50_ibn_b")
VEHICLE = ("resnet50", "resnext50_32x4d", "resnet50_ibn_a")


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "resnet_family.npz"))


@pytest.fixture(scope="module")
def resized(golden_dir):
    return np.load(os.path.join(golden_dir, "osnet.npz"))["resized"]


@pytest.mark.parametrize("name", NEW)
def test_synth_shapes_match_reference_model(name, golden_dir):
    with open(os.path.join(golden_dir, "resnet_family_state_shapes.json")) as f:
        ref = {k: tuple(v) for k, v in json.load(f)[name].items()}
    assert ref == resnet_family_param_shapes(name)
    assert set(synth_resnet_family_state(name, 1)) == set(ref)


def test_family_table_restates_resnet101():
    assert resnet_family_param_shapes("resnet101") == resnet101_reid_param_shapes()
    assert set(RESNET_FAMILY) == set(NEW) | {"resnet101"}


@pytest.mark.parametrize("name", NEW)
def test_states_are_seeded_and_deterministic(name):
    a, b, c = synth_resnet_family_state(name, 7), synth_resnet_family_state(name, 7), synth_resnet_family_state(name, 8)
    assert all(v.dtype == np.float32 for v in a.values())
    for k in a:
        np.testing.assert_array_equal(a[k], b[k])
    assert any(not np.array_equal(a[k], c[k]) for k in a)
    for scope in resnet_family_in_layers(name):          # gamma ~ U(0.8, 1.2), well away from 0; beta ~ N(0, 0.05)
        g, bt = a[scope + ".weight"], a[scope + ".bias"]
        assert g.min() >= 0.8 and g.max() <= 1.2 and np.abs(bt).max() < 0.5


@pytest.mark.parametrize("name", NEW)
def test_oracle_float32_matches_reference_features(name, golden, resized):
    state = synth_resnet_family_state(name, 2468)
    feats, _ = oracle.forward(name, state, resized, dtype=torch.float32)
    ref = golden[name + "/feats"]
    assert feats.shape == ref.shape == (6, 512 if name in ("resnet18", "resnet34", "resnet50_fc512") else 2048)
    assert np.abs(feats - ref).max() <= 2e-5 * np.abs(ref).max()
    if name in VEHICLE:
        feats, _ = oracle.forward(name, state, oracle.golden_crops((128, 256))[1], dtype=torch.float32)
        ref = golden[name + "/feats_128x256"]
        assert np.abs(feats - ref).max() <= 2e-5 * np.abs(ref).max()


def test_in_placement():
    a = resnet_family_in_layers("resnet50_ibn_a")
    assert a == ["layer%d.%d.bn1.IN" % (li, bi) for li, n in ((1, 3), (2, 4), (3, 6)) for bi in range(n)]
    assert resnet_family_in_layers("resnet50_ibn_b") == ["bn1", "layer1.2.IN", "layer2.3.IN"]
    sa = resnet_family_param_shapes("resnet50_ibn_a")
    assert sa["layer1.0.bn1.IN.weight"] == (32,) and sa["layer1.0.bn1.BN.running_var"] == (32,)
    assert sa["layer3.5.bn1.IN.weight"] == (128,) and "layer4.0.bn1.running_mean" in sa
    sb = resnet_family_param_shapes("resnet50_ibn_b")
    assert "bn1.running_mean" not in sb and sb["layer2.3.IN.weight"] == (512,)
    x = resnet_family_param_shapes("resnext101_32x8d")
    assert x["layer1.0.conv2.weight"] == (256, 8, 3, 3) and x["layer4.2.conv2.weight"] == (2048, 64, 3, 3)
    assert resnet_family_param_shapes("resnet50_fc512")["fc.0.weight"] == (512, 2048)
    assert "layer1.0.downsample.0.weight" not in resnet_family_param_shapes("resnet18")


@pytest.mark.parametrize("name", ("resnet50_ibn_a", "resnet50_ibn_b"))
def test_oracle_in_stage_names(name, resized):
    _, st = oracle.forward(name, synth_resnet_family_state(name, 2468), resized[:1])
    pre = sorted(k for k in st if k.endswith(".pre_in"))
    if name == "resnet50_ibn_a":
        assert pre == sorted(s[:-3] + ".pre_in" for s in resnet_family_in_layers(name))
        assert st["layer1.0.bn1"].shape == (1, 64, 32, 64) and st["layer3.5.bn1.pre_in"].shape == (1, 16, 8, 256)
    else:
        assert pre == ["conv1.pre_in", "layer1.2.pre_in", "layer2.3.pre_in"]
    assert st["conv1"].shape == (1, 128, 64, 64) and st["layer4"].shape == (1, 8, 4, 2048)
    assert {"maxpool", "layer1.0", "layer1", "layer2.3", "layer3", "layer4.2"} <= set(st)


def test_ibn_a_split_matches_torch_modules():
    """IBN (resnet_ibn_a.py:63-79) is InstanceNorm2d(affine) of the first half, BatchNorm2d (eval) of the rest."""
    rng = np.random.default_rng(0)
    C = 8
    x = torch.from_numpy(rng.standard_normal((2, C, 5, 7)) * 3 + 10)
    sd = {"p.IN.weight": rng.uniform(0.8, 1.2, C // 2), "p.IN.bias": rng.standard_normal(C // 2) * 0.05,
          "p.BN.weight": rng.uniform(0.7, 1.3, C // 2), "p.BN.bias": rng.standard_normal(C // 2) * 0.05,
          "p.BN.running_mean": rng.standard_normal(C // 2), "p.BN.running_var": rng.uniform(0.6, 1.4, C // 2)}
    sd = {k: torch.from_numpy(v) for k, v in sd.items()}
    inm = torch.nn.InstanceNorm2d(C // 2, affine=True).double().eval()
    bnm = torch.nn.BatchNorm2d(C // 2).double().eval()
    with torch.no_grad():
        inm.weight.copy_(sd["p.IN.weight"])
        inm.bias.copy_(sd["p.IN.bias"])
        for k in ("weight", "bias", "running_mean", "running_var"):
            getattr(bnm, k).copy_(sd["p.BN." + k])
        ref = torch.cat((inm(x[:, :C // 2].contiguous()), bnm(x[:, C // 2:].contiguous())), 1)
    assert torch.allclose(oracle.ibn_a(x, sd, "p"), ref, rtol=0, atol=1e-12)


def test_ibn_b_block_matches_torch_modules():
    """resnet_ibn_b.py's IN block: relu(IN(bn3(conv3(.)) + residual)); the oracle's block against torch modules."""
    rng = np.random.default_rng(1)
    cin, planes = 16, 4
    spec = dict(RESNET_FAMILY["resnet50_ibn_b"])
    sd = {"p.conv1.weight": rng.standard_normal((planes, cin, 1, 1)) * 0.3,
          "p.conv2.weight": rng.standard_normal((planes, planes, 3, 3)) * 0.3,
          "p.conv3.weight": rng.standard_normal((cin, planes, 1, 1)) * 0.3,
          "p.IN.weight": rng.uniform(0.8, 1.2, cin), "p.IN.bias": rng.standard_normal(cin) * 0.05}
    for bn, c in (("bn1", planes), ("bn2", planes), ("bn3", cin)):
        sd.update({"p.%s.weight" % bn: rng.uniform(0.7, 1.3, c), "p.%s.bias" % bn: rng.standard_normal(c) * 0.05,
                   "p.%s.running_mean" % bn: rng.standard_normal(c) * 0.1,
                   "p.%s.running_var" % bn: rng.uniform(0.6, 1.4, c)})
    sd = {k: torch.from_numpy(v) for k, v in sd.items()}
    x = torch.from_numpy(np.abs(rng.standard_normal((2, cin, 6, 5))))
    mods = {"conv1": torch.nn.Conv2d(cin, planes, 1, bias=False), "conv2": torch.nn.Conv2d(planes, planes, 3, padding=1,
                                                                                          bias=False),
            "conv3": torch.nn.Conv2d(planes, cin, 1, bias=False), "bn1": torch.nn.BatchNorm2d(planes),
            "bn2": torch.nn.BatchNorm2d(planes), "bn3": torch.nn.BatchNorm2d(cin),
            "IN": torch.nn.InstanceNorm2d(cin, affine=True)}
    mods = {k: m.double().eval() for k, m in mods.items()}
    with torch.no_grad():
        for k, v in sd.items():
            _, mod, param = k.split(".")
            getattr(mods[mod], param).copy_(v)
        r = torch.relu
        out = r(mods["bn2"](mods["conv2"](r(mods["bn1"](mods["conv1"](x))))))
        ref = r(mods["IN"](mods["bn3"](mods["conv3"](out)) + x))
    stages = {}
    got = oracle._block(x, sd, "p", 1, False, spec, True, stages)
    assert torch.allclose(got, ref, rtol=0, atol=1e-12)
    assert set(stages) == {"p.pre_in"}
