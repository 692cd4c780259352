"""Mask paste + COCO RLE, host against device: what the drivers do with final_masks (obj_detect_tracking.py:716-739).

  python tools/bench_mask_rle.py [--counts 10,100] [--frames 1080x1920,2160x3840] [--reps 20] [--host-reps 2]

  host path:   per box fill_full_mask (cv2.resize when cv2 imports, else the NumPy restatement tests/mask_rle_oracle.py),
               np.array(full[:, :, None], order="F"), and pycocotools' encode when it imports, else the restated
               encoder of tests/mask_rle_oracle.py;
  device path: masks.encode_masks(boxes, masks, im_shape) with the masks already on the GPU (a CUDA tensor), and once
               with NumPy masks (uploaded per call).

Seeded boxes: widths and heights drawn from 2-40 % of the frame's sides, seeded 28x28 blob masks.  Then one --add_mask
COCO-81 ResNet-50 detector (synthetic weights, 1080p uint8 frames resized on the GPU to 720 x 1280): detect + engine
encode (Detector.encode_masks, masks never leave the GPU) against detect + fetch final_masks + host path.

One JSON line per case: milliseconds per frame of each path (host clock around calls that end in a device synchronise)
and `match`, true when every RLE string of every timed frame equalled the host path's; the script stops on a mismatch.
The card's name and power limit are printed in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, check=True).stdout.strip()
        name, power = (s.strip() for s in out.split(","))
        return name, power
    except (OSError, subprocess.CalledProcessError, ValueError):
        import torch
        return torch.cuda.get_device_name(0), "unknown"


def seeded(rng, n, H, W):
    boxes = []
    for _ in range(n):
        w, h = rng.uniform(0.02, 0.4) * W, rng.uniform(0.02, 0.4) * H
        x, y = rng.uniform(0, W - w - 1), rng.uniform(0, H - h - 1)
        boxes.append((x, y, x + w, y + h))
    yy, xx = np.mgrid[0:28, 0:28].astype(np.float32)
    masks = []
    for _ in range(n):
        cx, cy, r = rng.uniform(6, 22), rng.uniform(6, 22), rng.uniform(20, 120)
        masks.append(1.0 / (1.0 + np.exp(((xx - cx) ** 2 + (yy - cy) ** 2) / r - 1.0)))
    return np.array(boxes, np.float32).reshape(-1, 4), np.array(masks, np.float32).reshape(-1, 28, 28)


def host_path():
    """The drivers' per-box loop, with the libraries they call where they import."""
    import mask_rle_oracle as oracle
    try:
        import cv2
        resize = cv2.resize
        which = "cv2 %s" % cv2.__version__
    except ImportError:
        resize = None
        which = "numpy restatement"
    try:
        from pycocotools import mask as cocomask
        enc = "pycocotools"
    except ImportError:
        cocomask = None
        enc = "restated encoder"

    def fill(box, mask, im_shape):
        if resize is None:
            return oracle.fill_full_mask(box, mask, im_shape)
        x0, y0 = list(map(int, box[:2] + 0.5))
        x1, y1 = list(map(int, box[2:] - 0.5))
        x1, y1 = max(x0, x1), max(y0, y1)
        w, h = x1 + 1 - x0, y1 + 1 - y0
        patch = (resize(mask, (w, h)) > 0.5).astype("uint8")
        ret = np.zeros(im_shape, dtype="uint8")
        ret[y0:y1 + 1, x0:x1 + 1] = patch
        return ret

    def run(boxes, masks, im_shape):
        out = []
        for box, mask in zip(boxes, masks):
            full = np.array(fill(box, mask, im_shape)[:, :, None], order="F")
            if cocomask is not None:
                rle = cocomask.encode(full)[0]
                rle["counts"] = rle["counts"].decode("ascii")
            else:
                rle = oracle.encode(full[:, :, 0])
            out.append({"size": [int(s) for s in rle["size"]], "counts": rle["counts"]})
        return out

    return run, "%s + %s" % (which, enc)


def timed(fn, reps):
    t = time.perf_counter()
    for _ in range(reps):
        out = fn()
    return (time.perf_counter() - t) * 1e3 / reps, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--counts", default="10,100")
    ap.add_argument("--frames", default="1080x1920,2160x3840")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--host-reps", type=int, default=2)
    ap.add_argument("--skip-detector", action="store_true")
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_mask_rle.py measures the GPU path: it needs cuda:0"
    from object_detection_tracking_b200 import masks as gm
    name, power = card()
    host, host_desc = host_path()
    print("# card: %s, power limit %s; host path: %s" % (name, power, host_desc), flush=True)
    rng = np.random.default_rng(2024)
    for fr in a.frames.split(","):
        H, W = (int(v) for v in fr.split("x"))
        for n in (int(v) for v in a.counts.split(",")):
            boxes, masks = seeded(rng, n, H, W)
            dev = torch.from_numpy(masks).cuda()
            gm.encode_masks(boxes, dev, (H, W))                              # warm-up: workspaces, module load
            gpu_ms, got = timed(lambda: gm.encode_masks(boxes, dev, (H, W)), a.reps)
            up_ms, got_up = timed(lambda: gm.encode_masks(boxes, masks, (H, W)), a.reps)
            host_ms, ref = timed(lambda: host(boxes, masks, (H, W)), a.host_reps)
            match = got == ref and got_up == ref
            print(json.dumps(dict(case="seeded", frame=[H, W], boxes=n, gpu_ms=round(gpu_ms, 3),
                                  gpu_upload_ms=round(up_ms, 3), host_ms=round(host_ms, 2),
                                  speedup=round(host_ms / gpu_ms, 1), match=match)), flush=True)
            if not match:
                sys.exit("RLE strings differ from the host path (%dx%d, %d boxes)" % (H, W, n))
    if a.skip_detector:
        return
    from object_detection_tracking_b200.config import make_config
    from object_detection_tracking_b200.engine import Detector
    from object_detection_tracking_b200.synth import synth_frame, synth_weights
    SH, SW, H, W = 1080, 1920, 720, 1280
    cfg = make_config(num_class=81, add_mask=True, max_size=W, short_edge_size=H, result_score_thres=0.0001)
    det = Detector(cfg, 1, H, W, device=0, precision="split", use_cuda_graph=True)
    det.load_weights(synth_weights(cfg, 7))
    frames = [synth_frame(SH, SW, s).astype(np.uint8)[None] for s in range(4)]
    scale = H / SH

    def detect(f):
        out = det.detect_host_resize(f, want_feat=False)
        r = int(out["valid"][0])
        return out["boxes"][0, :r] / scale

    def device(f):
        b = detect(f)
        return det.encode_masks(b, (SH, SW))

    def host_side(f):
        b = detect(f)
        return host(b, det.get_masks()[0, :len(b)], (SH, SW))

    for f in frames:
        device(f)
    dev_ms = host_ms = 0.0
    match, nboxes = True, []
    for f in frames:
        t, got = timed(lambda: device(f), a.reps)
        dev_ms += t / len(frames)
        t, ref = timed(lambda: host_side(f), a.host_reps)
        host_ms += t / len(frames)
        nboxes.append(len(got))
        match &= got == ref
    det_ms, _ = timed(lambda: detect(frames[0]), a.reps)
    print(json.dumps(dict(case="detector", model="COCO-81 R50 add_mask", source=[SH, SW], input=[H, W], boxes=nboxes,
                          detect_ms=round(det_ms, 3), detect_encode_gpu_ms=round(dev_ms, 3),
                          detect_host_path_ms=round(host_ms, 2), match=match)), flush=True)
    if not match:
        sys.exit("RLE strings differ from the host path (detector)")


if __name__ == "__main__":
    main()
