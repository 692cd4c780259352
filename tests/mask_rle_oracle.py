"""NumPy restatement of the drivers' mask post-processing (obj_detect_tracking.py:716-739): nn.fill_full_mask
(nn.py:1565-1584) with cv2.resize as OpenCV 4.13 computes it for a float32 28x28 mask (default dispatch), then
pycocotools' encode / rleToString (csrc/mask_rle_math.h states the arithmetic).  The checker of csrc/mask_rle.cu."""
import numpy as np

SIDE = 28


def fmaf(a, b, c):
    """float32 a * b + c with one rounding.  a * b is exact in float64; the float64 sum s rounds once, and TwoSum's error
    term e decides the one case where rounding s again to float32 differs from rounding the exact value: s exactly halfway
    between two float32 values while e != 0."""
    a, b, c = (np.asarray(v, np.float32).astype(np.float64) for v in (a, b, c))
    p = a * b
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)
    r = s.astype(np.float32)
    r64 = r.astype(np.float64)
    toward = np.where(s > r64, np.float32(np.inf), np.float32(-np.inf)).astype(np.float32)
    other = np.nextafter(r, toward)
    mid = (s != r64) & ((r64 + other.astype(np.float64)) * 0.5 == s) & (e != 0)
    up = np.maximum(r, other)
    down = np.minimum(r, other)
    return np.where(mid, np.where(e > 0, up, down), r).astype(np.float32)


def taps(n):
    """Source taps s0, s1 and float32 weights f of the n output indices of an axis resized from 28."""
    d = np.arange(n, dtype=np.float64)
    f = (d + 0.5) * (SIDE / n) - 0.5
    s = np.floor(f)
    f = f - s
    s = s.astype(np.int64)
    lo = s < 0
    s[lo], f[lo] = 0, 0.0
    hi = s >= SIDE - 1
    s[hi], f[hi] = SIDE - 1, 0.0
    return s, np.minimum(s + 1, SIDE - 1), f.astype(np.float32)


def resize(mask, w, h):
    """cv2.resize(mask, (w, h)) of a float32 [28, 28] mask, INTER_LINEAR: horizontal pass first, float32 fmaf lerps."""
    m = np.asarray(mask, np.float32)
    assert m.shape == (SIDE, SIDE)
    x0, x1, fx = taps(w)
    y0, y1, fy = taps(h)
    a, b = m[:, x0], m[:, x1]
    t = fmaf(b - a, np.broadcast_to(fx, a.shape), a)
    a, b = t[y0], t[y1]
    return fmaf(b - a, np.broadcast_to(fy[:, None], a.shape), a)


def geometry(box):
    """nn.py:1566-1575 as written: (x0, y0, x1, y1, w, h) of a float32 box."""
    box = np.asarray(box, np.float32)
    x0, y0 = list(map(int, box[:2] + 0.5))
    x1, y1 = list(map(int, box[2:] - 0.5))
    x1 = max(x0, x1)
    y1 = max(y0, y1)
    return x0, y0, x1, y1, x1 + 1 - x0, y1 + 1 - y0


def fill_full_mask(box, mask, im_shape):
    """nn.fill_full_mask with the resize above; NumPy's slice assignment raises ValueError where it cannot broadcast.
    Negative corners (which NumPy would wrap) raise ValueError as the GPU path does."""
    x0, y0, x1, y1, w, h = geometry(box)
    if x0 < 0 or y0 < 0:
        raise ValueError("negative corner")
    patch = (resize(mask, w, h) > 0.5).astype("uint8")
    ret = np.zeros(im_shape, dtype="uint8")
    ret[y0:y1 + 1, x0:x1 + 1] = patch
    return ret


def rle_counts(full):
    """pycocotools rleEncode of one H x W uint8 mask: run lengths of the column-major flattening, zeros first."""
    flat = np.asarray(full, np.uint8).ravel(order="F")
    change = np.flatnonzero(flat[1:] != flat[:-1]) + 1
    bounds = np.concatenate([[0], change, [flat.size]])
    counts = np.diff(bounds)
    if flat.size and flat[0]:
        counts = np.concatenate([[0], counts])
    return [int(c) for c in counts]


def rle_string(counts):
    """pycocotools rleToString."""
    out = []
    for i, c in enumerate(counts):
        x = int(c)
        if i > 2:
            x -= int(counts[i - 2])
        more = True
        while more:
            ch = x & 0x1f
            x >>= 5
            more = (x != -1) if (ch & 0x10) else (x != 0)
            if more:
                ch |= 0x20
            out.append(chr(ch + 48))
    return "".join(out)


def rle_parse(s):
    """pycocotools rleFrString: the counts of a string."""
    counts, p = [], 0
    while p < len(s):
        x, k, more = 0, 0, True
        while more:
            ch = ord(s[p]) - 48
            x |= (ch & 0x1f) << (5 * k)
            more = bool(ch & 0x20)
            p += 1
            k += 1
            if not more and (ch & 0x10):
                x |= -1 << (5 * k)
        if len(counts) > 2:
            x += counts[-2]
        counts.append(x)
    return counts


def rle_decode(counts, H, W):
    flat = np.zeros(H * W, np.uint8)
    at, v = 0, 0
    for c in counts:
        flat[at:at + c] = v
        at += c
        v ^= 1
    return flat.reshape((H, W), order="F")


def encode(full):
    H, W = full.shape
    return {"size": [H, W], "counts": rle_string(rle_counts(full))}
