"""Generates tests/golden/resnet_family.npz and tests/golden/resnet_family_state_shapes.json by running the REFERENCE's own
torchreid (/root/reference/torchreid) on the CPU for resnet18, resnet34, resnet50, resnet152, resnext50_32x4d,
resnext101_32x8d, resnet50_fc512, resnet50_ibn_a and resnet50_ibn_b, each with its seeded synthetic state_dict
(synth_resnet_family_state(name, 2468)), on the six crops of make_golden.py's osnet() recipe.  Run once in the authoring
container:
    python tests/golden/make_golden_resnet_family.py
The npz holds, per model, "<name>/feats" (FeatureExtractor at 256x128 on the raw crops) and, for the models of VEHICLE,
"<name>/feats_128x256" (at 128x256).  The 256x128 crops PIL-resized are osnet.npz's "resized", which this script checks
it reproduces; the tests resize the crops to 128x256 with PIL as FeatureExtractor does.
Every InstanceNorm input channel of these crops is asserted well conditioned (std >= MIN_STD_OVER_MEAN * |mean| over
H x W), so the engine's float32 statistics are compared where they are meaningful; ill-conditioned channels are the
kernel tests' business (tests/test_resnet_family_gpu.py)."""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, "/root/reference")
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from object_detection_tracking_b200.synth import synth_resnet_family_state  # noqa: E402
from torchreid.feature_extractor import FeatureExtractor  # noqa: E402

MODELS = ("resnet18", "resnet34", "resnet50", "resnet152", "resnext50_32x4d", "resnext101_32x8d", "resnet50_fc512",
          "resnet50_ibn_a", "resnet50_ibn_b")
VEHICLE = ("resnet50", "resnext50_32x4d", "resnet50_ibn_a")     # also stored at the drivers' vehicle size 128x256
SEED = 2468
MIN_STD_OVER_MEAN = 0.05


def crops():
    rng = np.random.default_rng(5)          # make_golden.py osnet()
    return [rng.integers(0, 256, (int(rng.integers(60, 300)), int(rng.integers(30, 160)), 3), dtype=np.uint8)
            for _ in range(6)]


def main():
    out, shapes, worst = {}, {}, {}
    cs = crops()
    for name in MODELS:
        state = synth_resnet_family_state(name, SEED)
        ratios = []

        def hook(mod, inp, _out):
            x = inp[0].double()
            m = x.mean(dim=(2, 3)).abs()
            s = x.std(dim=(2, 3), unbiased=False)
            ratios.append(float((s / m.clamp_min(1e-30)).min()))

        for size in ((256, 128),) + (((128, 256),) if name in VEHICLE else ()):
            ext = FeatureExtractor(name, model_path="", image_size=size, device="cpu", verbose=False)
            sd = ext.model.state_dict()
            ref_keys = {k for k in sd if not k.startswith("classifier") and not k.endswith("num_batches_tracked")}
            assert ref_keys == set(state), (name, ref_keys ^ set(state))
            for k, v in state.items():
                assert tuple(sd[k].shape) == v.shape, (k, sd[k].shape, v.shape)
                sd[k].copy_(torch.from_numpy(v))
            ext.model.load_state_dict(sd)
            ext.model.eval()
            shapes[name] = {k: list(sd[k].shape) for k in sorted(ref_keys)}
            hs = [m.register_forward_hook(hook) for m in ext.model.modules() if isinstance(m, torch.nn.InstanceNorm2d)]
            feats = ext(cs).numpy()
            for h in hs:
                h.remove()
            if size == (256, 128):
                out[name + "/feats"] = feats
                resized = np.stack([np.asarray(ext.to_pil(c).resize((128, 256), 2)) for c in cs])   # 2 = PIL BILINEAR
                np.testing.assert_array_equal(resized, np.load(os.path.join(HERE, "osnet.npz"))["resized"])
            else:
                out[name + "/feats_128x256"] = feats
        if ratios:
            worst[name] = min(ratios)
            assert worst[name] >= MIN_STD_OVER_MEAN, (name, ratios)
    np.savez_compressed(os.path.join(HERE, "resnet_family.npz"), **out)
    with open(os.path.join(HERE, "resnet_family_state_shapes.json"), "w") as f:
        json.dump(shapes, f, indent=0, sort_keys=True)
    print("min std / |mean| over the InstanceNorm inputs:", worst)


if __name__ == "__main__":
    main()
