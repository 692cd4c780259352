"""main.py --mode forward's scene feature: the backbone-only pass (--just_feat: b2_fpn_feature with frames, backbone + FPN
+ the 7x7 resize of p5) against the full detect (b2_detect_host) on the same context, at main.py's documented size
(1080x1920, SPEED.md / TRAINING.md: ResNet-101 FPN, dilated res5, rpn_test_post_nms_topk 1000, batch 1) and at 720x1280.
Both are host-in / host-out calls as the driver makes them (the float32 frame is uploaded every call), with the CUDA graph.
The two run alternately, `--steps` calls each per round over `--rounds` rounds, so that clock and neighbour drift hits both
alike; the host clock is read around the synchronous calls.

  python tools/bench_forward_feat.py [--steps 30 --rounds 5 --warmup 5 --precision split]

Prints one JSON line per size: ms per call of each pass (median and range over the rounds), kernels per pass, the board's
name and power limit."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

SIZES = ((1080, 1920), (720, 1280))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--precision", default="split", choices=["split", "fp16"])
    args = ap.parse_args()

    import torch
    from bench_gn import board
    from object_detection_tracking_b200.config import make_config
    from object_detection_tracking_b200.engine import Detector
    from object_detection_tracking_b200.synth import synth_frame, synth_weights
    if not torch.cuda.is_available():
        raise RuntimeError("bench_forward_feat.py needs an H100: no CUDA device")
    info = board(0)
    for H, W in SIZES:
        cfg = make_config(rpn_test_post_nms_topk=1000, short_edge_size=H, max_size=W)   # R101, dilated res5
        det = Detector(cfg, 1, H, W, device=0, precision=args.precision, use_cuda_graph=True)
        det.load_weights(synth_weights(cfg, 1234))
        frames = [synth_frame(H, W, seed=j)[None].astype(np.float32) for j in range(4)]
        out = det.alloc_outputs()
        passes = {"detect": lambda f: det.detect_host(f, out, want_feat=True),
                  "feature_only": lambda f: det.fpn_feature(f)}
        for run in passes.values():
            for i in range(args.warmup):
                run(frames[i % 4])
        ms = {k: [] for k in passes}
        for _ in range(args.rounds):
            for k, run in passes.items():
                t0 = time.perf_counter()
                for i in range(args.steps):
                    run(frames[i % 4])
                ms[k].append((time.perf_counter() - t0) * 1e3 / args.steps)
        line = {"metric": "main.py forward: ms per call, %dx%d, ResNet-101 FPN dilated, rpn 1000, batch 1, %s"
                          % (W, H, args.precision),
                "kernels": {"detect": det.kernel_launches(), "feature_only": det.fpn_feature_launches()},
                "steps": args.steps, "rounds": args.rounds, "gpu": info["name"], "power_limit_w": info["power_limit_w"]}
        for k, v in ms.items():
            line[k + "_ms"] = {"median": round(float(np.median(v)), 3), "min": round(min(v), 3), "max": round(max(v), 3)}
        print(json.dumps(line), flush=True)
        det.close()


if __name__ == "__main__":
    main()
