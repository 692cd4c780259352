"""Throughput of the attention-head detector: ResNet-101 FPN with the attention box head (use_att_frcnn_head,
models.py:1064-1089), --version 3 flags (dilated res5, 15 classes, class-specific head), 1280x720, rpn300, batch 8,
batch-graph semantics, CUDA graph -- the same loop and clock record as bench.py's device-resident leg.  --no-att runs the
same model without the attention branch, for interleaved A/B runs.

  python tools/bench_att_head.py [--no-att --steps 50 --warmup 5 --precision split --sustained-seconds 5
                                  --profile-json FILE]

Prints one JSON line: frames/s (host clock around synchronised graph replays), a sustained record, SM clocks, the board's
name and power limit, and from one eager per-step profile (CUDA events, three passes averaged) the share of the pass spent
in the att_* steps, with each step's time and achieved GB/s over the bytes b2_step_info computes from the shapes (each
operand read once, each output written once, at the stored precision)."""
import argparse
import json
import os
import re
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

H, W, BATCH = 720, 1280, 8
MODEL = dict(resnet_num_block=(3, 4, 23, 3), num_class=15, use_dilations=True, use_frcnn_class_agnostic=False,
             use_att_frcnn_head=True)
STEPS = ("att_pool", "att_trans", "att_sum")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--no-att", action="store_true", help="the same model without the attention branch")
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
        raise RuntimeError("bench_att_head.py needs an H100: no CUDA device")
    torch.cuda.set_device(0)
    model = dict(MODEL, use_att_frcnn_head=not args.no_att)
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
    steps = {}
    for name in STEPS:
        sel = [p for p in prof if re.match(r"fastrcnn/%s\b" % name, p["name"])]
        ms = sum(p["ms"] for p in sel)
        gb = sum(p["bytes"] for p in sel) / 1e9
        gflop = sum(p["flops"] for p in sel) / 1e9
        steps[name] = {"steps": len(sel), "ms": ms, "gb": gb, "gflop": gflop, "gb_per_s": gb / ms * 1e3 if ms > 0 else None}
    att_ms = sum(v["ms"] for v in steps.values())
    line = {"metric": "detector FPS @1280x720 rpn300 (ResNet-101-FPN Faster-RCNN%s, dilated, 15 classes)"
                      % ("" if args.no_att else " + attention head"),
            "value": args.steps * BATCH / dt, "unit": "frames/s", "steps": args.steps, "ms_per_step": dt / args.steps * 1e3,
            "batch": BATCH, "precision": args.precision, "use_att_frcnn_head": not args.no_att,
            "weights": "seeded synthetic (synth.py, seed 1234)", "board": board(0), "clocks": sampler.summary(),
            "sustained": sustained,
            "profile": {"total_ms": total, "att_ms": att_ms, "att_share": att_ms / total if total else None,
                        "att_steps": steps}}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
