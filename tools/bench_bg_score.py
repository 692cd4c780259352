"""Cost of --use_bg_score on the BASELINE config-1 detector: R101-FPN dilated, 15 classes, 720x1280, rpn300, the
single-image graph at batch 1, CUDA graph, split precision.  The option adds one kernel (bg_filter_kernel: one read of the
[rpn300][15] probabilities per image) ahead of the class NMS, which then skips the dropped rows.

  python tools/bench_bg_score.py [--runs 5 --steps 200 --warmup 20]

Builds the model with the option off and on, from the same weights, and times them alternately (off, on, off, on, ...)
in one process: each run is `steps` synchronised graph replays under a host clock.  Prints one JSON line: the median
ms/frame of each, their difference, the share of ROIs the filter dropped on the timed frames, the post-processing step's
device time from one eager per-step profile (CUDA events), SM clocks, and the board's name and power limit."""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

H, W = 720, 1280


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()

    import torch
    from bench import ClockSampler
    from bench_gn import board
    from object_detection_tracking_b200.config import make_config
    from object_detection_tracking_b200.engine import Detector
    from object_detection_tracking_b200.synth import synth_frame, synth_weights
    if not torch.cuda.is_available():
        raise RuntimeError("bench_bg_score.py needs an H100: no CUDA device")
    torch.cuda.set_device(0)
    weights = synth_weights(make_config(), 1234)
    dets = {}
    for flag in (False, True):
        cfg = make_config(use_bg_score=flag)
        assert cfg.resnet_num_block == (3, 4, 23, 3) and cfg.rpn_test_post_nms_topk == 300
        dets[flag] = Detector(cfg, 1, H, W, device=0, precision="split", use_cuda_graph=True)
        dets[flag].load_weights(weights)
    frames = [torch.from_numpy(synth_frame(H, W, seed=s)[None].astype(np.float32)).cuda() for s in range(4)]
    for d in dets.values():
        for i in range(max(args.warmup, 3)):
            d.detect_device(frames[i % 4], None, sync=True)
    ms = {False: [], True: []}
    sampler = ClockSampler(0)
    sampler.start()
    for _ in range(args.runs):
        for flag in (False, True):
            d = dets[flag]
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for i in range(args.steps):
                d.detect_device(frames[i % 4], None, sync=(i == args.steps - 1))
            torch.cuda.synchronize()
            ms[flag].append((time.perf_counter() - t0) / args.steps * 1e3)
    sampler.stop.set()
    sampler.join(timeout=2)
    dropped = []
    for f in frames:
        dets[True].detect_device(f, None, sync=True)
        n = int(dets[True].get_stage("proposal_count").reshape(-1)[0])
        dropped.append(float((dets[True].get_stage("bg_rank").reshape(-1)[:n] < 0).mean()) if n else 0.0)
    post = {}
    for flag, d in dets.items():
        prof = d.profile_steps(reps=3)
        post["on" if flag else "off"] = sum(p["ms"] for p in prof if "head_post" in p["name"])
        d.close()
    off, on = statistics.median(ms[False]), statistics.median(ms[True])
    print(json.dumps({
        "model": "BASELINE config 1: R101-FPN dilated, 15 classes, 720x1280, rpn300, batch 1, single-image graph",
        "ms_per_frame_off": off, "ms_per_frame_on": on, "delta_ms": on - off,
        "runs_off": ms[False], "runs_on": ms[True], "steps": args.steps,
        "dropped_share": dropped, "head_post_ms": post,
        "clocks": sampler.summary(), "board": board(0)}))


if __name__ == "__main__":
    main()
