"""Throughput of the relation-network detector: ResNet-101 FPN with the relation box head (add_relation_nn: RM_r1 / RM_r2,
nn.py:115-190), --version 3 flags (dilated res5, 15 classes), 1280x720, rpn300, batch 8, batch-graph semantics, CUDA
graph -- the same loop and clock record as bench.py's device-resident leg.  --no-relation runs the same model without the
relation modules, for interleaved A/B runs.

  python tools/bench_relation.py [--no-relation --steps 50 --warmup 5 --precision split --sustained-seconds 5
                                  --profile-json FILE]

Prints one JSON line: frames/s (host clock around synchronised graph replays), a sustained record, SM clocks, the board's
name and power limit, and from one eager per-step profile (CUDA events, three passes averaged) the share of the pass spent
in the relation steps, with each kind's time and achieved TFLOP/s.  The FLOP counts are computed here from the shapes
(at the full K = rpn300 rows per image): query|key 2 * BK * D * 2D, attend 2 * B * K^2 * (4*64 + 64*16 + D) (geometry
net and the 16 head dots per pair), P.V 2 * 16K * K * D per image, output_linear 2 * BK * 16D * D."""
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
MODEL = dict(resnet_num_block=(3, 4, 23, 3), num_class=15, use_dilations=True, add_relation_nn=True)
KINDS = ("query_key", "attend", "attention_value", "output_linear")


def step_flops(kind, B, K, D):
    """Algorithmic FLOPs of one relation module's steps of `kind` over the batch, from the shapes."""
    return {"query_key": 2.0 * B * K * D * 2 * D,
            "attend": 2.0 * B * K * K * (4 * 64 + 64 * 16 + D),
            "attention_value": 2.0 * B * 16 * K * K * D,
            "output_linear": 2.0 * B * K * 16 * D * D}[kind]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--no-relation", action="store_true", help="the same model without the relation modules")
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
        raise RuntimeError("bench_relation.py needs an H100: no CUDA device")
    torch.cuda.set_device(0)
    model = dict(MODEL, add_relation_nn=not args.no_relation)
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
    K, D = cfg.rpn_test_post_nms_topk, cfg.fpn_frcnn_fc_head_dim
    kinds = {}
    for kind in KINDS:
        steps = [p for p in prof if re.match(r"fastrcnn/RM_r\d/%s\b" % kind, p["name"])]
        ms = sum(p["ms"] for p in steps)
        gflop = 2 * step_flops(kind, BATCH, K, D) / 1e9 if steps else 0.0        # both modules
        kinds[kind] = {"steps": len(steps), "ms": ms, "gflop": gflop, "tflops": gflop / ms if ms > 0 else None}
    rel_ms = sum(v["ms"] for v in kinds.values())
    line = {"metric": "detector FPS @1280x720 rpn300 (ResNet-101-FPN Faster-RCNN%s, dilated, 15 classes)"
                      % ("" if args.no_relation else " + relation head"),
            "value": args.steps * BATCH / dt, "unit": "frames/s", "steps": args.steps, "ms_per_step": dt / args.steps * 1e3,
            "batch": BATCH, "precision": args.precision, "add_relation_nn": not args.no_relation,
            "weights": "seeded synthetic (synth.py, seed 1234)", "board": board(0), "clocks": sampler.summary(),
            "sustained": sustained,
            "profile": {"total_ms": total, "relation_ms": rel_ms, "relation_share": rel_ms / total if total else None,
                        "relation_steps": kinds}}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
