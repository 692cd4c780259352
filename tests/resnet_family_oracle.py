"""Functional restatement of torchreid's ResNet family (resnet.py:52-366, resnet_ibn_a.py:63-264,
resnet_ibn_b.py:62-249) from a state_dict, in float64 (or float32) torch on the CPU, without importing torchreid.
`forward` returns the eval features and the intermediate maps under the ReID engine's stage names (NHWC): "conv1",
"maxpool", "layerN.M", "layerN"; IBN-a adds "layerN.M.bn1.pre_in" (conv1's output, raw in the channels the
InstanceNorm takes and batch-normalised in the rest) and "layerN.M.bn1" (after the split norm and ReLU), IBN-b
"conv1.pre_in" and "layerN.M.pre_in" for each InstanceNorm's input."""
import numpy as np
import torch
import torch.nn.functional as F

from object_detection_tracking_b200.synth import RESNET_FAMILY, resnet_family_blocks
from osnet_family_oracle import _bn, instance_norm, normalize


def golden_crops(size=(256, 128)):
    """make_golden.py's six osnet() crops, PIL-resized to `size` (h, w) as FeatureExtractor resizes them."""
    from PIL import Image
    rng = np.random.default_rng(5)
    cs = [rng.integers(0, 256, (int(rng.integers(60, 300)), int(rng.integers(30, 160)), 3), dtype=np.uint8)
          for _ in range(6)]
    return cs, np.stack([np.asarray(Image.fromarray(c).resize(size[::-1], Image.BILINEAR)) for c in cs])


def ibn_a(x, sd, p):
    """IBN (resnet_ibn_a.py:63-79): InstanceNorm2d of the first C // 2 channels, BatchNorm2d of the rest, concatenated."""
    half = x.shape[1] // 2
    return torch.cat((instance_norm(x[:, :half], sd[p + ".IN.weight"], sd[p + ".IN.bias"]), _bn(x[:, half:], sd, p + ".BN")),
                     1)


def _block(x, sd, p, stride, down, spec, in_after, stages):
    identity = x
    if spec["block"] == "basic":                                   # resnet.py:86-102
        out = F.relu(_bn(F.conv2d(x, sd[p + ".conv1.weight"], stride=stride, padding=1), sd, p + ".bn1"))
        out = _bn(F.conv2d(out, sd[p + ".conv2.weight"], padding=1), sd, p + ".bn2")
    else:                                                          # resnet.py:134-154
        out = F.conv2d(x, sd[p + ".conv1.weight"])
        if p + ".bn1.IN.weight" in sd:
            half = out.shape[1] // 2                               # the split step's input: conv1's raw first half
            stages[p + ".bn1.pre_in"] = torch.cat((out[:, :half], _bn(out[:, half:], sd, p + ".bn1.BN")), 1)
            out = F.relu(ibn_a(out, sd, p + ".bn1"))
            stages[p + ".bn1"] = out
        else:
            out = F.relu(_bn(out, sd, p + ".bn1"))
        out = F.conv2d(out, sd[p + ".conv2.weight"], stride=stride, padding=1, groups=spec["groups"])
        out = F.relu(_bn(out, sd, p + ".bn2"))
        out = _bn(F.conv2d(out, sd[p + ".conv3.weight"]), sd, p + ".bn3")
    if down:
        identity = _bn(F.conv2d(x, sd[p + ".downsample.0.weight"], stride=stride), sd, p + ".downsample.1")
    out = out + identity
    if in_after:                                                   # resnet_ibn_b.py:106-109
        stages[p + ".pre_in"] = out
        out = instance_norm(out, sd[p + ".IN.weight"], sd[p + ".IN.bias"])
    return F.relu(out)


def forward(name, state, crops_u8, dtype=torch.float64):
    """-> (features [n, D] numpy, {engine stage name: NHWC numpy})."""
    spec = RESNET_FAMILY[name]
    sd = {k: torch.from_numpy(v).to(dtype) for k, v in state.items()}
    stages = {}
    x = F.conv2d(normalize(crops_u8, dtype), sd["conv1.weight"], stride=2, padding=3)
    if spec["ibn"] == "b":                                         # resnet_ibn_b.py:142
        stages["conv1.pre_in"] = x
        x = F.relu(instance_norm(x, sd["bn1.weight"], sd["bn1.bias"]))
    else:
        x = F.relu(_bn(x, sd, "bn1"))
    stages["conv1"] = x
    x = F.max_pool2d(x, 3, 2, 1)
    stages["maxpool"] = x
    blocks = resnet_family_blocks(name)
    for i, (p, stride, _, _, _, down) in enumerate(blocks):
        x = _block(x, sd, p, stride, down, spec, p + ".IN.weight" in sd, stages)
        stages[p] = x
        if i + 1 == len(blocks) or blocks[i + 1][0].split(".")[0] != p.split(".")[0]:
            stages[p.split(".")[0]] = x
    v = x.mean(dim=(2, 3))
    if spec["fc"]:                                                 # resnet.py:292-320, 358-359
        v = F.relu(_bn(F.linear(v, sd["fc.0.weight"], sd["fc.0.bias"]), sd, "fc.1"))
    return v.numpy(), {k: t.permute(0, 2, 3, 1).contiguous().numpy() for k, t in stages.items()}
