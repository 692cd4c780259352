"""EfficientDet-D7 at 1536x1536 on batches of synthetic 1080x1920 frames: batch 1 against batch B in one run.

For every (precision, batch) case, one context at a time (each is closed before the next is created), prints one JSON line:
  host_fps    frames/s through the whole host call (upload, pre-processing, graph, download): detect_batch()
  replay_fps  frames/s of the captured graph replayed alone (no host copies): b2_effdet_replay
  launches    kernels per batched call
  context_mib device memory the context holds (free memory before creation minus free memory after its first call)
Each rate is given as the median, min and max over --repeats windows of --steps calls: the GPU is shared, so the spread
is part of the result.  The GPU's name and power limit are read in the same run and printed with every line.

    python tools/bench_effdet_batch.py [--batches 1,2,4] [--precisions split,fp16] [--steps 10] [--repeats 5]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def frames(n, h=1080, w=1920):
    """n textured BGR frames, one seed per camera."""
    out = []
    for seed in range(n):
        rng = np.random.default_rng(100 + seed)
        base = rng.integers(0, 256, (h // 8 + 1, w // 8 + 1, 3)).astype(np.float32)
        img = np.kron(base, np.ones((8, 8, 1), np.float32))[:h, :w]
        out.append(np.clip(img + rng.standard_normal((h, w, 3)) * 12, 0, 255).astype(np.uint8))
    return out


def gpu_info():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30)
        power = float(r.stdout.strip().splitlines()[0])
    except Exception:
        power = None
    return name, power


def spread(v):
    return {"median": round(statistics.median(v), 2), "min": round(min(v), 2), "max": round(max(v), 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,2,4")
    ap.add_argument("--precisions", default="split,fp16")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_effdet_batch needs a GPU")
    from object_detection_tracking_b200.effdet import EffdetEngine
    from object_detection_tracking_b200.effdet_config import BACKBONE_OF, make_effdet_config
    from object_detection_tracking_b200.synth import synth_effdet_weights, synth_efficientnet_weights
    det = "efficientdet-d7"
    cfg = make_effdet_config(det, 1536, 1536)
    Wt = dict(synth_effdet_weights(cfg))
    Wt.update(synth_efficientnet_weights(BACKBONE_OF[det]))
    # the seeded predict layers are conditioned for shallow nets: bring D7's deep heads to a trained detector's range
    Wt["class_net/class-predict/pointwise_kernel"] = Wt["class_net/class-predict/pointwise_kernel"] * np.float32(0.03)
    Wt["box_net/box-predict/pointwise_kernel"] = Wt["box_net/box-predict/pointwise_kernel"] * np.float32(0.08)
    batches = [int(b) for b in args.batches.split(",")]
    fr = frames(max(batches))
    name, power = gpu_info()
    for precision in args.precisions.split(","):
        for B in batches:
            torch.cuda.synchronize()
            free0 = torch.cuda.mem_get_info(0)[0]
            eng = EffdetEngine(cfg, Wt, precision=precision, backbone=BACKBONE_OF[det], batch=B)
            try:
                batch = fr[:B]
                outs = eng.detect_batch(batch)
                context = free0 - torch.cuda.mem_get_info(0)[0]
                for _ in range(args.warmup):
                    eng.detect_batch(batch)
                host, replay = [], []
                for _ in range(args.repeats):
                    t0 = time.perf_counter()
                    for _ in range(args.steps):
                        eng.detect_batch(batch)
                    host.append(B * args.steps / (time.perf_counter() - t0))
                    replay.append(B * 1000.0 / eng.replay_ms(args.steps))
                rec = {"config": "%s %dx%d" % (det, 1536, 1536), "frames": "1080x1920", "batch": B,
                       "precision": precision, "host_fps": spread(host), "replay_fps": spread(replay),
                       "launches": eng.num_launches, "context_mib": round(context / 2 ** 20),
                       "detections": [len(o["final_probs"]) for o in outs], "steps": args.steps,
                       "repeats": args.repeats, "gpu": name, "power_limit_w": power}
                print(json.dumps(rec), flush=True)
            finally:
                eng.close()


if __name__ == "__main__":
    main()
