"""Throughput of the ResNet-34 / ResNet-18 detectors (use_basic_block; --version 4 flags: dilated res5 -- which the basic
block ignores --, class-agnostic box head, 15 classes), 1280x720, rpn300, batch 8, batch-graph semantics, CUDA graph -- the
same loop and clock record as bench.py's device-resident leg.  --bottleneck runs ResNet-50 with the same configuration,
for interleaved A/B runs.

  python tools/bench_basic_block.py [--depth 34|18 --bottleneck --steps 50 --warmup 5 --precision split
                                     --sustained-seconds 5 --profile-json FILE]

Prints one JSON line: frames/s (host clock around synchronised graph replays), a sustained record, SM clocks, the board's
name and power limit, and from one eager per-step profile (CUDA events, three passes averaged) the backbone's conv1 and
conv2 times per group.  In every basic block after a group's first, conv1 and conv2 are the same GEMM (3x3, ch -> ch, same
M); only conv2 has the shortcut in its epilogue, on a staged epilogue with a residual slot ring.  Per group the line gives
both means over those blocks, their difference, the residual's bytes and the rate at which the difference would read
them (residual bytes / difference): a rate at or above the stream rate of the residual 1x1 layers says the ring costs
nothing beyond the extra read."""
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
MODEL = dict(num_class=15, version=4, use_dilations=True, use_frcnn_class_agnostic=True)


def conv_rows(prof, esz):
    """Per group: conv1 / conv2 of the blocks after the first (mean ms), and block 0's."""
    steps = {}
    for p in prof:
        m = re.match(r"(group(\d)/block(\d+))/(conv1|conv2) ", p["name"])
        if p["kind"] == 0 and m:
            steps[(int(m.group(2)), int(m.group(3)), m.group(4))] = p
    rows = []
    for g in range(4):
        blocks = sorted({b for (gg, b, _) in steps if gg == g})
        later = [b for b in blocks if b > 0]
        row = {"group": g, "blocks": len(blocks),
               "block0_conv1_ms": steps[(g, 0, "conv1")]["ms"], "block0_conv2_ms": steps[(g, 0, "conv2")]["ms"]}
        if later:
            c1 = float(np.mean([steps[(g, b, "conv1")]["ms"] for b in later]))
            c2 = float(np.mean([steps[(g, b, "conv2")]["ms"] for b in later]))
            s2 = steps[(g, later[0], "conv2")]
            flops = s2["flops"]
            cout = int(re.search(r"->(\d+)\]", s2["name"]).group(1))
            res_bytes = flops / (2.0 * 9 * cout) * esz                   # M * Cout planes: one read of the shortcut
            row.update({"conv1_ms": c1, "conv2_ms": c2, "conv2_minus_conv1_ms": c2 - c1,
                        "conv_tflops": flops / (c1 * 1e-3) / 1e12, "residual_mb": res_bytes / 1e6,
                        "residual_rate_tbs": res_bytes / ((c2 - c1) * 1e-3) / 1e12 if c2 > c1 else None})
        rows.append(row)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--depth", type=int, default=34, choices=[34, 18])
    ap.add_argument("--bottleneck", action="store_true", help="ResNet-50 with the same configuration")
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
        raise RuntimeError("bench_basic_block.py needs an H100: no CUDA device")
    torch.cuda.set_device(0)
    model = dict(MODEL, **({"resnet50": True} if args.bottleneck else {"resnet%d" % args.depth: True}))
    cfg = make_config(**model)
    name = "ResNet-50" if args.bottleneck else "ResNet-%d" % args.depth
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
    backbone = sum(p["ms"] for p in prof if p["name"].startswith(("conv0", "maxpool", "group")))
    line = {"metric": "detector FPS @1280x720 rpn300 (%s-FPN Faster-RCNN, --version 4 flags, 15 classes)" % name,
            "value": args.steps * BATCH / dt, "unit": "frames/s", "steps": args.steps, "ms_per_step": dt / args.steps * 1e3,
            "batch": BATCH, "precision": args.precision, "backbone": name, "use_basic_block": bool(cfg.use_basic_block),
            "weights": "seeded synthetic (synth.py, seed 1234)", "board": board(0), "clocks": sampler.summary(),
            "sustained": sustained, "launches": det.kernel_launches(),
            "profile": {"total_ms": total, "backbone_ms": backbone}}
    if cfg.use_basic_block:
        line["profile"]["groups"] = conv_rows(prof, 4.0 if args.precision == "split" else 2.0)
    det.close()
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
