"""ReID input step, host against device: seeded 1080p uint8 BGR frames with N person-shaped track boxes each, embedded
by OSNet-x1.0 (256x128) and ResNet-101 (128x256).

  python tools/bench_reid_boxes.py [--per-frame 8,32,64] [--models osnet_x1_0,resnet101] [--frames 12] [--precision split]

  host path:   numpy slice, [..., ::-1] (BGR -> RGB), FeatureExtractor._resize (Pillow, one crop at a time), then
               ReidEngine.embed of the stacked crops -- what FeatureExtractor.__call__ does after the drivers' crop loop;
  device path: ReidEngine.embed_boxes(frame, boxes) -- the frame and the box table go to the GPU, the crop-resize kernel
               cuts and resizes, the same captured pass embeds.

Per (model, N) one JSON line: end-to-end crops/s of each path (host clock around calls that end in a device
synchronise), the host path's slice + convert + resize milliseconds per crop, and the crop-resize kernel's mean time
(torch.profiler with CUDA activities, in a pass of its own after the timed ones).  Every frame's features of the two paths
must be bit-identical, or the script stops.  The card's name and power limit are printed in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def person_boxes(rng, n, H, W, frame_index=0):
    """n person-shaped boxes (h = 1.8..3 w, w 24..220 px) inside an H x W frame -> int32 [n, 5]."""
    b = np.zeros((n, 5), np.int32)
    for i in range(n):
        w = int(rng.integers(24, 221))
        h = min(H, int(w * rng.uniform(1.8, 3.0)))
        b[i] = (frame_index, rng.integers(0, W - w + 1), rng.integers(0, H - h + 1), w, h)
    return b


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, check=True).stdout.strip()
        name, power = (s.strip() for s in out.split(","))
        return name, power
    except (OSError, subprocess.CalledProcessError, ValueError):
        import torch
        return torch.cuda.get_device_name(0), "unknown"


def kernel_ms(eng, frame, boxes, reps):
    """Mean device time of reid_crop_resize_kernel over `reps` embed_boxes calls (torch.profiler, CUDA activities)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            eng.embed_boxes(frame, boxes)
        torch.cuda.synchronize()
    times = [e.device_time_total for e in prof.events() if "reid_crop_resize_kernel" in e.name]
    return (sum(times) / len(times) / 1e3) if times else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--per-frame", default="8,32,64")
    ap.add_argument("--models", default="osnet_x1_0,resnet101")
    ap.add_argument("--frames", type=int, default=12, help="timed frames per path and configuration")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--precision", default="split")
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_reid_boxes needs a GPU"
    from object_detection_tracking_b200.reid import FeatureExtractor
    from object_detection_tracking_b200.synth import synth_frame, synth_osnet_state, synth_resnet101_reid_state

    name, power = card()
    print(json.dumps({"gpu": name, "power_limit": power}), flush=True)
    H, W = 1080, 1920
    frames = [np.ascontiguousarray(synth_frame(H, W, seed=k)) for k in range(4)]   # decoded frames are contiguous
    states = {"osnet_x1_0": synth_osnet_state(4321), "resnet101": synth_resnet101_reid_state(2468)}
    sizes = {"osnet_x1_0": (256, 128), "resnet101": (128, 256)}
    for model in args.models.split(","):
        for n in (int(v) for v in args.per_frame.split(",")):
            ext = FeatureExtractor(model_name=model, image_size=sizes[model], batch=n, precision=args.precision,
                                   state_dict=states[model])
            eng = ext.engine
            rng = np.random.default_rng(1000 + n)
            boxes = [person_boxes(rng, n, H, W) for _ in frames]

            def host(k):
                t0 = time.perf_counter()
                crops = [ext._resize(frames[k][y:y + h, x:x + w][..., ::-1]) for _, x, y, w, h in boxes[k]]
                t1 = time.perf_counter()
                return eng.embed(np.stack(crops)), t1 - t0

            def device(k):
                return eng.embed_boxes(frames[k], boxes[k])

            for k in range(args.warmup):
                j = k % len(frames)
                fh, _ = host(j)
                if not np.array_equal(fh, device(j)):
                    raise SystemExit("%s N=%d frame %d: device-path features differ from the host path" % (model, n, j))
            t_prep = 0.0
            t0 = time.perf_counter()
            host_feats = []
            for k in range(args.frames):
                f, dt = host(k % len(frames))
                host_feats.append(f)
                t_prep += dt
            t_host = time.perf_counter() - t0
            t0 = time.perf_counter()
            dev_feats = [device(k % len(frames)) for k in range(args.frames)]
            t_dev = time.perf_counter() - t0
            for k, (a, b) in enumerate(zip(host_feats, dev_feats)):
                if not np.array_equal(a, b):
                    raise SystemExit("%s N=%d frame %d: device-path features differ from the host path" % (model, n, k))
            kms = kernel_ms(eng, frames[0], boxes[0], 20)
            crops = n * args.frames
            print(json.dumps({
                "model": model, "boxes_per_frame": n, "precision": args.precision, "frames": args.frames,
                "host_crops_per_s": round(crops / t_host, 1), "device_crops_per_s": round(crops / t_dev, 1),
                "host_prep_ms_per_crop": round(1e3 * t_prep / crops, 4),
                "crop_resize_kernel_ms": None if kms is None else round(kms, 4),
                "crop_resize_kernel_us_per_crop": None if kms is None else round(1e3 * kms / n, 3),
                "bit_identical": True, "gpu": name, "power_limit": power}), flush=True)
            eng.close()


if __name__ == "__main__":
    main()
