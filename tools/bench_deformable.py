"""Throughput of the deformable-conv detector: ResNet-101 FPN with use_deformable (--version 2 flags: no dilation, 15
classes; res5 block 0 deformable), 1280x720, rpn300, batch 8, batch-graph semantics, CUDA graph -- the same loop and clock
record as bench.py's device-resident leg.  --no-deformable runs the same seed as the plain model, for interleaved A/B runs.

  python tools/bench_deformable.py [--no-deformable --steps 50 --warmup 5 --precision split --sustained-seconds 5
                                    --profile-json FILE]

Prints one JSON line: frames/s (host clock around synchronised graph replays), a sustained record, SM clocks, the board's
name and power limit, and from one eager per-step profile (CUDA events, three passes averaged) the time, algorithmic
GFLOP, HBM bytes and achieved rates of the deformable block's three steps (conv2_offset, conv2_sample, conv2) -- or, with
--no-deformable, of the dense conv2 they replace."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

H, W, BATCH = 720, 1280, 8
MODEL = dict(resnet_num_block=(3, 4, 23, 3), num_class=15, use_dilations=False, version=2, use_deformable=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--no-deformable", action="store_true", help="the plain ResNet-101 with the same configuration")
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--precision", default="split", choices=["split", "fp16"])
    ap.add_argument("--sustained-seconds", type=float, default=5.0)
    ap.add_argument("--profile-json", default="", help="write the per-step profile here")
    args = ap.parse_args()

    import torch
    from bench import ClockSampler
    from bench_gn import board
    from object_detection_tracking_b200.config import make_config
    from object_detection_tracking_b200.engine import Detector
    from object_detection_tracking_b200.synth import synth_frame, synth_weights
    if not torch.cuda.is_available():
        raise RuntimeError("bench_deformable.py needs an H100: no CUDA device")
    torch.cuda.set_device(0)
    model = dict(MODEL, use_deformable=not args.no_deformable)
    cfg = make_config(**model)
    det = Detector(cfg, BATCH, H, W, device=0, precision=args.precision, use_cuda_graph=True, multi_semantics=True)
    det.load_weights(synth_weights(cfg, 1234))
    dev = [torch.from_numpy(np.stack([synth_frame(H, W, seed=8 * j + i) for i in range(BATCH)]).astype(np.float32)).cuda()
           for j in range(4)]                    # 4 x 88 MB: the rotating input set exceeds the 50 MB L2

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

    sustained = None
    if args.sustained_seconds > 0:
        s2 = ClockSampler(0)
        s2.start()
        n, ts = 0, time.perf_counter()
        while time.perf_counter() - ts < args.sustained_seconds:
            for _ in range(16):
                det.detect_device(dev[n % 4], None, sync=False)
                n += 1
            det.detect_device(dev[n % 4], None, sync=True)
            n += 1
        dts = time.perf_counter() - ts
        s2.stop.set()
        s2.join(timeout=2)
        sustained = {"value": n * BATCH / dts, "unit": "frames/s", "seconds": dts, "clocks": s2.summary()}

    prof = det.profile_steps(reps=3)
    if args.profile_json:
        with open(args.profile_json, "w") as f:
            json.dump({"precision": args.precision, "batch": BATCH, "model": model, "steps": prof}, f, indent=1)
    total = sum(p["ms"] for p in prof)
    block = [p for p in prof if p["name"].startswith(("group3/block0/conv2 ", "group3/block0/conv2_offset ",
                                                       "group3/block0/conv2_sample "))]
    rows = [{"name": p["name"], "ms": p["ms"], "gflop": p["flops"] / 1e9, "mbytes": p["bytes"] / 1e6,
             "tflops": p["flops"] / (p["ms"] * 1e-3) / 1e12 if p["ms"] > 0 else None,
             "gbytes_per_s": p["bytes"] / (p["ms"] * 1e-3) / 1e9 if p["ms"] > 0 else None} for p in block]
    block_ms = sum(p["ms"] for p in block)
    line = {"metric": "detector FPS @1280x720 rpn300 (ResNet-101-FPN Faster-RCNN%s, no dilation, 15 classes)"
                      % ("" if args.no_deformable else ", deformable res5 block 0"),
            "value": args.steps * BATCH / dt, "unit": "frames/s", "steps": args.steps, "ms_per_step": dt / args.steps * 1e3,
            "batch": BATCH, "precision": args.precision, "use_deformable": not args.no_deformable,
            "weights": "seeded synthetic (synth.py, seed 1234)", "board": board(0), "clocks": sampler.summary(),
            "sustained": sustained,
            "profile": {"total_ms": total, "block_conv2_ms": block_ms, "block_conv2_share": block_ms / total if total else None,
                        "block_conv2_steps": rows}}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
