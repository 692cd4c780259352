"""Wall-clock timings of the two other engines through their host-facing calls (host buffers in, host results out):
EfficientDet-D7 1536x1536 single-frame detect (BASELINE configs[2]) and OSNet-x1.0 ReID embedding (configs[4]).
Prints one JSON line per engine; redirect it to a file."""
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from gpu_effnet_probe import synth_frame  # noqa: E402
from object_detection_tracking_b200.effdet import EffdetEngine  # noqa: E402
from object_detection_tracking_b200.effdet_config import BACKBONE_OF, make_effdet_config  # noqa: E402
from object_detection_tracking_b200.reid import ReidEngine  # noqa: E402
from object_detection_tracking_b200.synth import synth_effdet_weights, synth_efficientnet_weights, synth_osnet_state  # noqa: E402


def effdet(det="efficientdet-d7", H=1536, W=1536, reps=10):
    for prec in ("split", "fp16"):
        cfg = make_effdet_config(det, H, W)
        Wt = dict(synth_effdet_weights(cfg))
        Wt.update(synth_efficientnet_weights(BACKBONE_OF[det]))
        eng = EffdetEngine(cfg, Wt, precision=prec, backbone=BACKBONE_OF[det])
        frame = synth_frame(1080, 1920)
        for _ in range(3):
            eng.detect(frame)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(reps):
            out = eng.detect(frame)
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t0) / reps * 1e3
        print(json.dumps({"engine": det, "input": [1080, 1920, 3], "network_input": [H, W], "precision": prec,
                          "ms_per_frame_host_call": ms, "frames_per_s": 1e3 / ms, "launches_per_frame": eng.num_launches,
                          "detections": int(len(out["final_probs"]))}), flush=True)
        eng.close()


def osnet(batch=64, reps=10):
    for prec in ("split", "fp16"):
        eng = ReidEngine(batch=batch, precision=prec)
        eng.load_state(synth_osnet_state(4321))
        crops = np.random.default_rng(0).integers(0, 256, (batch, 256, 128, 3), dtype=np.uint8)
        for _ in range(3):
            eng.embed(crops)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(reps):
            eng.embed(crops)
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t0) / reps * 1e3
        print(json.dumps({"engine": "osnet_x1_0", "batch": batch, "precision": prec, "ms_per_batch_host_call": ms,
                          "crops_per_s": batch / ms * 1e3, "launches_per_batch": eng.num_launches()}), flush=True)
        eng.close()


if __name__ == "__main__":
    effdet()
    osnet()
