"""Throughput of the COCO partial-class detector ("Object COCO partial": --is_coco_model --use_partial_classes --resnet50,
version 2): R50-FPN, an 81-class checkpoint whose box head keeps person / car / bus / truck / bicycle, 1280x720, rpn300,
CUDA graph -- at batch 8 (batch-graph semantics) and batch 1, with the same loop and clock record as bench.py's
device-resident leg.  --full runs the same checkpoint as the 80-class model, the baseline the partial head is read
against; run the two interleaved.

  python tools/bench_partial_classes.py [--full --steps 50 --warmup 5 --precision split --batches 8,1 --profile-json FILE]

Prints one JSON line per batch size: frames/s (host clock around synchronised graph replays), SM clocks, the board's name
and power limit, and from one eager per-step profile (CUDA events, three passes averaged) the time of the box head's
output layer (fastrcnn/outputs, N = 30 partial or 405 full columns) and of the post-processing step (head_post: softmax
and decode, per-class NMS, final top-k)."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

H, W = 720, 1280
MODEL = dict(resnet_num_block=(3, 4, 6, 3), num_class=81, use_dilations=False, version=2)


def run(batch, args, cfg, weights):
    import torch
    from bench import ClockSampler
    from object_detection_tracking_b200.engine import Detector
    from object_detection_tracking_b200.synth import synth_frame
    det = Detector(cfg, batch, H, W, device=0, precision=args.precision, use_cuda_graph=True,
                   multi_semantics=batch > 1)
    det.load_weights(weights)
    dev = [torch.from_numpy(np.stack([synth_frame(H, W, seed=8 * j + i) for i in range(batch)]).astype(np.float32)).cuda()
           for j in range(4)]                    # a rotating input set larger than the 50 MB L2 at batch 8
    for i in range(max(args.warmup, 3)):
        det.detect_device(dev[i % 4], None, sync=True)
    sampler = ClockSampler(0)
    sampler.start()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(args.steps):
        det.detect_device(dev[i % 4], None, sync=(i == args.steps - 1))
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    sampler.stop.set()
    sampler.join(timeout=2)
    prof = det.profile_steps(reps=3)
    det.close()
    head = [p for p in prof if "fastrcnn/outputs" in p["name"]]
    post = [p for p in prof if "head_post" in p["name"]]
    return prof, {"value": args.steps * batch / dt, "unit": "frames/s", "steps": args.steps,
                  "ms_per_step": dt / args.steps * 1e3, "batch": batch, "clocks": sampler.summary(),
                  "profile": {"total_ms": sum(p["ms"] for p in prof),
                              "box_head_output_ms": sum(p["ms"] for p in head),
                              "head_post_ms": sum(p["ms"] for p in post),
                              "steps": [p["name"] for p in head + post]}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--full", action="store_true", help="the same checkpoint as the full 80-class model")
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--precision", default="split", choices=["split", "fp16"])
    ap.add_argument("--batches", default="8,1")
    ap.add_argument("--profile-json", default="", help="write the per-step profiles here")
    args = ap.parse_args()

    import torch
    from bench_gn import board
    from object_detection_tracking_b200.config import make_config
    from object_detection_tracking_b200.synth import synth_weights
    if not torch.cuda.is_available():
        raise RuntimeError("bench_partial_classes.py needs an H100: no CUDA device")
    torch.cuda.set_device(0)
    cfg = make_config(use_partial_classes=not args.full, **MODEL)
    weights = synth_weights(make_config(**MODEL), 4321)
    profiles = {}
    for batch in (int(b) for b in args.batches.split(",")):
        prof, res = run(batch, args, cfg, weights)
        profiles[batch] = prof
        line = {"metric": "detector FPS @1280x720 rpn300 (ResNet-50-FPN Faster-RCNN, COCO %s)"
                          % ("80 classes" if args.full else "partial: person/car/bus/truck/bicycle"),
                "classes": list(cfg.partial_classes) if not args.full else "all 80", "precision": args.precision,
                "weights": "seeded synthetic (synth.py, seed 4321)", "board": board(0), **res}
        print(json.dumps(line), flush=True)
    if args.profile_json:
        with open(args.profile_json, "w") as f:
            json.dump({"precision": args.precision, "full": args.full, "steps": profiles}, f, indent=1)


if __name__ == "__main__":
    main()
