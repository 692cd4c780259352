"""Crops/s of torchreid's six OSNet person models on the GPU (osnet_x1_0, osnet_x0_75, osnet_x0_5, osnet_x0_25,
osnet_ibn_x1_0, osnet_ain_x1_0; 256x128 crops, 512-d features, seeded synthetic weights), or of any model ReidEngine
builds named in --models (torchreid's ResNets draw synth_resnet_family_state(name, 2468)), each at its first crop size.

  python tools/bench_reid_models.py [--batches 32,128] [--rounds 5] [--reps 10] [--precision split] [--models a,b]

For every batch size, the models alternate within each of `rounds` rounds (so clock and thermal drift spread over all of
them).  Each model times `reps` calls of ReidEngine.embed (resized crops in, features out) and of ReidEngine.embed_boxes
(one seeded 1080p BGR frame with `batch` person-shaped boxes, cut and resized on the GPU).  The median over the rounds is
reported as crops/s, one JSON line per (model, batch).  Then one pass per model runs under torch.profiler (CUDA activities)
and the device time of its kernels is summed by kernel name: the InstanceNorm kernel's share of the pass is reported for
the IBN / AIN models (both IN kernels: the plain one and IBN-a's split one).  The card's name and power limit are printed in the same run."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_reid_boxes import card, person_boxes  # noqa: E402

MODELS = ("osnet_x1_0", "osnet_x0_75", "osnet_x0_5", "osnet_x0_25", "osnet_ibn_x1_0", "osnet_ain_x1_0")


def kernel_profile(eng, crops):
    """{kernel name: device ms} of one embed pass (torch.profiler, CUDA activities)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    eng.embed(crops)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        eng.embed(crops)
        torch.cuda.synchronize()
    out = {}
    for e in prof.events():
        if e.device_time_total > 0 and "memcpy" not in e.name.lower() and "memset" not in e.name.lower():
            out[e.name] = out.get(e.name, 0.0) + e.device_time_total / 1e3
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="32,128")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--precision", default="split")
    ap.add_argument("--models", default=",".join(MODELS))
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_reid_models needs a GPU"
    from object_detection_tracking_b200.reid import ReidEngine
    from object_detection_tracking_b200.synth import (RESNET_FAMILY, synth_frame, synth_osnet_family_state,
                                                      synth_osnet_state, synth_resnet_family_state)

    name, power = card()
    print(json.dumps({"gpu": name, "power_limit": power}), flush=True)
    models = args.models.split(",")
    states = {m: synth_osnet_state(4321) if m == "osnet_x1_0" else synth_resnet_family_state(m, 2468)
              if m in RESNET_FAMILY else synth_osnet_family_state(m, 4321) for m in models}
    frame = np.ascontiguousarray(synth_frame(1080, 1920, seed=1))
    rng = np.random.default_rng(0)
    for batch in (int(b) for b in args.batches.split(",")):
        boxes = person_boxes(np.random.default_rng(batch), batch, 1080, 1920)
        engs, crops = {}, {}
        for m in models:
            engs[m] = ReidEngine(batch, 0, args.precision, m)
            engs[m].load_state(states[m])
            size = engs[m].image_size
            if size not in crops:
                crops[size] = rng.integers(0, 256, (batch,) + size + (3,), dtype=np.uint8)
            engs[m].embed(crops[size])                 # captures the graph
            engs[m].embed_boxes(frame, boxes)
        t_embed = {m: [] for m in models}
        t_boxes = {m: [] for m in models}
        for _ in range(args.rounds):
            for m in models:
                e = engs[m]
                t0 = time.perf_counter()
                for _ in range(args.reps):
                    e.embed(crops[e.image_size])
                t1 = time.perf_counter()
                for _ in range(args.reps):
                    e.embed_boxes(frame, boxes)
                t2 = time.perf_counter()
                t_embed[m].append((t1 - t0) / args.reps)
                t_boxes[m].append((t2 - t1) / args.reps)
        for m in models:
            prof = kernel_profile(engs[m], crops[engs[m].image_size])
            total = sum(prof.values())
            inorm = sum(v for k, v in prof.items() if "instnorm_kernel" in k)
            print(json.dumps({
                "model": m, "image_size": list(engs[m].image_size), "batch": batch, "precision": args.precision, "rounds": args.rounds, "reps": args.reps,
                "embed_crops_per_s": round(batch / float(np.median(t_embed[m])), 1),
                "embed_boxes_1080p_crops_per_s": round(batch / float(np.median(t_boxes[m])), 1),
                "embed_ms_median": round(1e3 * float(np.median(t_embed[m])), 3),
                "kernel_ms_per_pass": round(total, 3),
                "instnorm_ms_per_pass": round(inorm, 3),
                "instnorm_share": round(inorm / total, 4) if total else None,
                "launches": engs[m].num_launches()}), flush=True)
        for e in engs.values():
            e.close()


if __name__ == "__main__":
    main()
