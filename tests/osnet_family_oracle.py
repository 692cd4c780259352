"""Functional restatement of torchreid's OSNet family (osnet.py:223-438, :522-598; osnet_ain.py:230-541) from a
state_dict, in float64 (or float32) torch on the CPU, without importing torchreid.  `forward` returns the 512-d eval
features and the intermediate maps under the ReID engine's stage names (NHWC, the model's own channel counts):
"conv1.pre_in", "conv1", "maxpool", "conv2.0.pre_in", "conv2.0", ..., "conv2.t", "conv2", ..., "conv5"."""
import numpy as np
import torch
import torch.nn.functional as F

from object_detection_tracking_b200.synth import OSNET_FAMILY

MEAN = (0.485, 0.456, 0.406)
STD = (0.229, 0.224, 0.225)


def _bn(x, sd, p, eps=1e-5):
    sh = (1, -1, 1, 1) if x.dim() == 4 else (1, -1)
    return (x - sd[p + ".running_mean"].view(sh)) / torch.sqrt(sd[p + ".running_var"].view(sh) + eps) \
        * sd[p + ".weight"].view(sh) + sd[p + ".bias"].view(sh)


def instance_norm(x, w, b, eps=1e-5):
    """InstanceNorm2d(affine=True, track_running_stats=False): per (image, channel) statistics, biased variance."""
    m = x.mean(dim=(2, 3), keepdim=True)
    v = ((x - m) ** 2).mean(dim=(2, 3), keepdim=True)
    return (x - m) / torch.sqrt(v + eps) * w.view(1, -1, 1, 1) + b.view(1, -1, 1, 1)


def _in(x, sd, p):
    return instance_norm(x, sd[p + ".weight"], sd[p + ".bias"])


def _light(x, sd, p):
    x = F.conv2d(x, sd[p + ".conv1.weight"])
    x = F.conv2d(x, sd[p + ".conv2.weight"], padding=1, groups=x.shape[1])
    return F.relu(_bn(x, sd, p + ".bn"))


def _gate(x, sd, p):
    g = x.mean(dim=(2, 3), keepdim=True)
    g = F.relu(F.conv2d(g, sd[p + ".fc1.weight"], sd[p + ".fc1.bias"]))
    return x * torch.sigmoid(F.conv2d(g, sd[p + ".fc2.weight"], sd[p + ".fc2.bias"]))


def _block(x, sd, p, kind, ain, stages):
    identity = x
    x1 = F.relu(_bn(F.conv2d(x, sd[p + ".conv1.conv.weight"]), sd, p + ".conv1.bn"))
    x2 = 0
    for t in range(4):
        s = x1
        for j in range(t + 1):
            s = _light(s, sd, ("%s.conv2.%d.layers.%d" % (p, t, j)) if ain
                       else ("%s.conv2%s" % (p, "abcd"[t]) + ("" if t == 0 else ".%d" % j)))
        x2 = x2 + _gate(s, sd, p + ".gate")
    x3 = F.conv2d(x2, sd[p + ".conv3.conv.weight"])
    if p + ".downsample.conv.weight" in sd:
        identity = _bn(F.conv2d(x, sd[p + ".downsample.conv.weight"]), sd, p + ".downsample.bn")
    if kind == "inin":                                   # osnet_ain.py:283-295
        stages[p + ".pre_in"] = x3
        return F.relu(_in(x3, sd, p + ".IN") + identity)
    out = _bn(x3, sd, p + ".conv3.bn") + identity
    if kind == "ibn":                                    # osnet.py:270-276
        stages[p + ".pre_in"] = out
        out = _in(out, sd, p + ".IN")
    return F.relu(out)


def normalize(crops_u8, dtype=torch.float64):
    """ToTensor + Normalize of [n, 256, 128, 3] RGB uint8 crops -> [n, 3, 256, 128]."""
    x = torch.from_numpy(np.ascontiguousarray(crops_u8)).to(dtype).permute(0, 3, 1, 2) / 255.0
    return (x - torch.tensor(MEAN, dtype=dtype).view(1, 3, 1, 1)) / torch.tensor(STD, dtype=dtype).view(1, 3, 1, 1)


def forward(name, state, crops_u8, dtype=torch.float64):
    """-> (features [n, 512] numpy, {engine stage name: NHWC numpy})."""
    spec = OSNET_FAMILY[name]
    sd = {k: torch.from_numpy(np.asarray(v)).to(dtype) for k, v in state.items()}
    stages = {}
    x = F.conv2d(normalize(crops_u8, dtype), sd["conv1.conv.weight"], stride=2, padding=3)
    if spec["stem_in"]:
        stages["conv1.pre_in"] = x
        x = F.relu(_in(x, sd, "conv1.bn"))
    else:
        x = F.relu(_bn(x, sd, "conv1.bn"))
    stages["conv1"] = x
    x = F.max_pool2d(x, 3, 2, 1)
    stages["maxpool"] = x
    for s in range(3):
        sn = "conv%d" % (s + 2)
        for i in range(2):
            x = _block(x, sd, "%s.%d" % (sn, i), spec["kinds"][s][i], spec["ain"], stages)
            stages["%s.%d" % (sn, i)] = x
        if s < 2:
            tn = "pool%d.0" % (s + 2) if spec["ain"] else sn + ".2.0"
            x = F.relu(_bn(F.conv2d(x, sd[tn + ".conv.weight"]), sd, tn + ".bn"))
            stages[sn + ".t"] = x
            x = F.avg_pool2d(x, 2, 2)
            stages[sn] = x
    x = F.relu(_bn(F.conv2d(x, sd["conv5.conv.weight"]), sd, "conv5.bn"))
    stages["conv5"] = x
    v = x.mean(dim=(2, 3))
    v = F.relu(_bn(F.linear(v, sd["fc.0.weight"], sd["fc.0.bias"]), sd, "fc.1"))
    return v.numpy(), {k: t.permute(0, 2, 3, 1).contiguous().numpy() for k, t in stages.items()}
