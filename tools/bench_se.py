"""Throughput of the SE-ResNet detector ("Object v6": --version 6 = use_se + use_frcnn_class_agnostic, no dilation):
R101-FPN with squeeze-excite bottlenecks, 15 classes, 1280x720, rpn300, batch 8, batch-graph semantics, CUDA graph -- the
same loop and clock record as bench.py's device-resident leg.  --no-se runs the same model with use_se off (the plain
class-agnostic R101), the baseline the SE cost is read against.

  python tools/bench_se.py [--no-se --steps 50 --warmup 5 --precision split --sustained-seconds 5 --profile-json FILE]

Prints one JSON line: frames/s (host clock around synchronised graph replays), a sustained record, SM clocks, the board's
name and power limit, and from one eager per-step profile (CUDA events, three passes averaged) the share of the pass spent
in the squeeze-excite steps and the achieved bandwidth of every SE step from b2_step_info's byte counts."""
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
MODEL = dict(resnet_num_block=(3, 4, 23, 3), num_class=15, use_frcnn_class_agnostic=True, use_dilations=False, version=6,
             use_se=True)
SE_KINDS = {13: "squeeze", 14: "excite", 15: "apply"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--no-se", action="store_true", help="the same model with use_se off")
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
        raise RuntimeError("bench_se.py needs an H100: no CUDA device")
    torch.cuda.set_device(0)
    model = dict(MODEL, use_se=not args.no_se)
    cfg = make_config(**model)
    det = Detector(cfg, BATCH, H, W, device=0, precision=args.precision, use_cuda_graph=True, multi_semantics=True)
    det.load_weights(synth_weights(make_config(**MODEL), 1234))   # the v6 checkpoint; without use_se its SE arrays are unused
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
    se = [p for p in prof if p["kind"] in SE_KINDS]
    by_kind = {SE_KINDS[k]: {"steps": sum(1 for p in se if p["kind"] == k),
                             "ms": sum(p["ms"] for p in se if p["kind"] == k),
                             "gb": sum(p["bytes"] for p in se if p["kind"] == k) / 1e9} for k in SE_KINDS}
    line = {"metric": "detector FPS @1280x720 rpn300 (ResNet-101-FPN Faster-RCNN, %s, class-agnostic, 15 classes)"
                      % ("no SE" if args.no_se else "squeeze-excite (v6)"),
            "value": args.steps * BATCH / dt, "unit": "frames/s", "steps": args.steps, "ms_per_step": dt / args.steps * 1e3,
            "batch": BATCH, "precision": args.precision, "use_se": not args.no_se,
            "weights": "seeded synthetic (synth.py, seed 1234)", "board": board(0), "clocks": sampler.summary(),
            "sustained": sustained,
            "profile": {"total_ms": total, "se_ms": sum(p["ms"] for p in se),
                        "se_share": sum(p["ms"] for p in se) / total, "se_by_kind": by_kind,
                        "se_steps_gbs": [{"name": p["name"], "ms": p["ms"], "gb": p["bytes"] / 1e9,
                                          "gbs": p["bytes"] / (p["ms"] * 1e-3) / 1e9 if p["ms"] > 0 else None}
                                         for p in se]}}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
