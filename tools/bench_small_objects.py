"""Throughput of the small-object detector: the ActEV merge-prop model (ResNet-101 FPN, dilated res5, 17 classes,
class-specific 2fc head) with the small-object branch (use_small_object_head, models.py:590-692, 845-897) over its four
default classes, 1280x720, batch 1 (the branch exists in the single-image graph only), CUDA graph -- the same loop and
clock record as bench.py's device-resident leg.  --no-so runs the same model without the branch and --association adds
person_object_relation, for interleaved A/B runs; --rpn-topk 1000 is main.py's rpn_test_post_nms_topk.

  python tools/bench_small_objects.py [--no-so] [--association] [--rpn-topk 1000] [--steps 200 --warmup 10
                                       --precision split --profile-json FILE]

Prints one JSON line: frames/s (host clock around synchronised graph replays), SM clocks, the board's name and power limit,
and from one eager per-step profile (CUDA events, three passes averaged) the branch's steps (kinds 20-24 and its dense
layers, all named so_* or fastrcnn/small_objects/*) with each one's time, FLOPs and bytes as b2_step_info computes them
from the shapes, and their share of the pass."""
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
MODEL = dict(resnet_num_block=(3, 4, 23, 3), num_class=17, use_dilations=True, use_frcnn_class_agnostic=False)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--no-so", action="store_true", help="the same model without the small-object branch")
    ap.add_argument("--association", action="store_true", help="with use_so_association")
    ap.add_argument("--rpn-topk", type=int, default=300)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--precision", default="split", choices=["split", "fp16"])
    ap.add_argument("--profile-json", default="", help="write the per-step profile here")
    args = ap.parse_args()

    import torch
    from bench import ClockSampler
    from bench_gn import board
    from object_detection_tracking_b200.config import make_config
    from object_detection_tracking_b200.engine import Detector
    from object_detection_tracking_b200.synth import synth_frame, synth_weights
    if not torch.cuda.is_available():
        raise RuntimeError("bench_small_objects.py needs an H100: no CUDA device")
    torch.cuda.set_device(0)
    model = dict(MODEL, rpn_test_post_nms_topk=args.rpn_topk, use_small_object_head=not args.no_so,
                 use_so_association=args.association and not args.no_so)
    cfg = make_config(**model)
    det = Detector(cfg, 1, H, W, device=0, precision=args.precision, use_cuda_graph=True)
    det.load_weights(synth_weights(cfg, 1234))
    dev = [torch.from_numpy(synth_frame(H, W, seed=j)[None].astype(np.float32)).cuda() for j in range(8)]

    for i in range(max(args.warmup, 3)):
        det.detect_device(dev[i % 8], None, sync=True)
    sampler = ClockSampler(0)
    sampler.start()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(args.steps):
        det.detect_device(dev[i % 8], None, sync=(i == args.steps - 1))
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    sampler.stop.set()
    sampler.join(timeout=2)

    prof = det.profile_steps(reps=3)
    if args.profile_json:
        with open(args.profile_json, "w") as f:
            json.dump({"precision": args.precision, "model": model, "steps": prof}, f, indent=1)
    total = sum(p["ms"] for p in prof)
    branch = [dict(name=p["name"], ms=p["ms"], gflop=p["flops"] / 1e9, gb=p["bytes"] / 1e9) for p in prof
              if p["kind"] in (20, 21, 22, 23, 24) or p["name"].startswith("fastrcnn/small_objects/")]
    so_ms = sum(p["ms"] for p in branch)
    line = {"metric": "detector FPS @1280x720 rpn%d batch 1 (ResNet-101-FPN merge-prop, 17 classes%s)"
                      % (args.rpn_topk, "" if args.no_so else " + small-object head" +
                         (" + association" if args.association else "")),
            "value": args.steps / dt, "unit": "frames/s", "steps": args.steps, "ms_per_step": dt / args.steps * 1e3,
            "batch": 1, "precision": args.precision, "use_small_object_head": not args.no_so,
            "use_so_association": bool(model["use_so_association"]),
            "weights": "seeded synthetic (synth.py, seed 1234)", "board": board(0), "clocks": sampler.summary(),
            "profile": {"total_ms": total, "so_ms": so_ms, "so_share": so_ms / total if total else None,
                        "so_gflop": sum(p["gflop"] for p in branch), "so_steps": branch}}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
