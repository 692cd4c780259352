// Arithmetic of the mask paste and RLE kernels (mask_rle.cu): the drivers' per-detection post-processing of final_masks
// (obj_detect_tracking.py:716-739, nn.py:1565-1584), i.e. fill_full_mask followed by pycocotools' encode / rleToString.
//   - geometry (host): x0, y0 = int(box[:2] + 0.5), x1, y1 = int(box[2:] - 0.5) in float32 with int() truncating toward
//     zero, x1 = max(x0, x1), y1 = max(y0, y1), w = x1 + 1 - x0, h = y1 + 1 - y0; the paste ret[y0:y1+1, x0:x1+1] = patch
//     follows NumPy's slice and broadcast rules (mask_geometry);
//   - resize: cv2.resize(mask, (w, h)) of a float32 28x28 mask, INTER_LINEAR, as OpenCV 4.13 computes it with its default
//     (optimised) dispatch: per axis in double f = (d + 0.5) * (28 / n) - 0.5, s = floor(f), f -= s, clamped to the
//     source (s < 0: s = 0, f = 0; s >= 27: s = 27, f = 0), f rounded to float32, second tap min(s + 1, 27); then the
//     horizontal pass t = fmaf(src[s1] - src[s0], fx, src[s0]) and the vertical out = fmaf(t[y1] - t[y0], fy, t[y0]), both
//     float32 with one rounding per fmaf; the pixel is set when out > 0.5f;
//   - RLE string (pycocotools rleToString): each count x (x -= cnts[i - 2] for i > 2, as a signed 64-bit value) is sent
//     as 5-bit groups, low first, c = x & 0x1f, x >>= 5 (arithmetic), more = (c & 0x10) ? x != -1 : x != 0, c |= 0x20 when
//     more, character c + 48.
// Shared by the CUDA kernels and a host harness the CPU tests compile (tests/test_mask_rle_cpu.py), so the kernels'
// arithmetic is checked against the cv2-pinned oracle without a GPU.
#pragma once
#include <math.h>
#include <stdint.h>

#include "resize_math.h"   // B2_HD, B2_DMUL, B2_DSUB

#if defined(__CUDA_ARCH__)
#define B2_FSUB(a, b) __fsub_rn((a), (b))
#define B2_FMAF(a, b, c) __fmaf_rn((a), (b), (c))
#else
#define B2_FSUB(a, b) ((a) - (b))
#define B2_FMAF(a, b, c) fmaf((a), (b), (c))
#endif

namespace b2 {

constexpr int kMaskSide = 28;   // the mask head's output (models.py:958-961)

// One output index d of an axis resized from kMaskSide to n samples.
struct MaskTap {
  int s0, s1;
  float f;
};

B2_HD MaskTap mask_tap(int d, int n) {
  double f = B2_DSUB(B2_DMUL(static_cast<double>(d) + 0.5, static_cast<double>(kMaskSide) / n), 0.5);
  const double s = floor(f);
  f = B2_DSUB(f, s);
  MaskTap t;
  t.s0 = static_cast<int>(s);
  if (t.s0 < 0) {
    t.s0 = 0;
    f = 0.0;
  }
  if (t.s0 >= kMaskSide - 1) {
    t.s0 = kMaskSide - 1;
    f = 0.0;
  }
  t.s1 = t.s0 + 1 < kMaskSide - 1 ? t.s0 + 1 : kMaskSide - 1;
  t.f = static_cast<float>(f);
  return t;
}

B2_HD float mask_lerp(float a, float b, float f) { return B2_FMAF(B2_FSUB(b, a), f, a); }

// The resized value at (tx, ty) of a row-major kMaskSide x kMaskSide source.
B2_HD float mask_resize_at(const float* src, MaskTap tx, MaskTap ty) {
  const float* r0 = src + ty.s0 * kMaskSide;
  const float* r1 = src + ty.s1 * kMaskSide;
  const float t0 = mask_lerp(r0[tx.s0], r0[tx.s1], tx.f);
  const float t1 = mask_lerp(r1[tx.s0], r1[tx.s1], tx.f);
  return mask_lerp(t0, t1, ty.f);
}

B2_HD bool mask_on(float v) { return v > 0.5f; }

// Where fill_full_mask puts a box's patch in an H x W frame.
enum MaskGeomStatus {
  kMaskGeomOk = 0,
  kMaskGeomNegative = 1,   // a corner int(box[:2] + 0.5) below 0: NumPy would index from the far edge
  kMaskGeomOverhang = 2,   // the frame cuts the slice short and the patch cannot broadcast to it: NumPy's ValueError
  kMaskGeomRange = 3,      // a coordinate that is not finite or not below 2^30
};

struct MaskPlace {
  int x0, y0, w, h;   // the patch cv2.resize makes: w x h at (x0, y0)
  bool pasted;        // false when the slice is empty (x0 >= W or y0 >= H with a size-1 patch side): nothing lands
};

B2_HD int mask_trunc(float v, int* out) {
  if (!(v > -1073741824.0f && v < 1073741824.0f)) return kMaskGeomRange;
  *out = static_cast<int>(v);   // truncates toward zero, as int()
  return kMaskGeomOk;
}

B2_HD int mask_geometry(const float box[4], int H, int W, MaskPlace* p) {
  int x0, y0, x1, y1;
  if (mask_trunc(box[0] + 0.5f, &x0) || mask_trunc(box[1] + 0.5f, &y0) || mask_trunc(box[2] - 0.5f, &x1) ||
      mask_trunc(box[3] - 0.5f, &y1))
    return kMaskGeomRange;
  if (x0 < 0 || y0 < 0) return kMaskGeomNegative;
  if (x1 < x0) x1 = x0;
  if (y1 < y0) y1 = y0;
  p->x0 = x0;
  p->y0 = y0;
  p->w = x1 + 1 - x0;
  p->h = y1 + 1 - y0;
  // ret[y0:y1+1, x0:x1+1]: the slice stops at the frame's edge, and the patch must equal it or be 1 along each axis
  const int sh = y0 >= H ? 0 : (y1 + 1 < H ? y1 + 1 : H) - y0;
  const int sw = x0 >= W ? 0 : (x1 + 1 < W ? x1 + 1 : W) - x0;
  if ((sh != p->h && p->h != 1) || (sw != p->w && p->w != 1)) return kMaskGeomOverhang;
  p->pasted = sh > 0 && sw > 0;   // then sh == h and sw == w
  return kMaskGeomOk;
}

// Characters rleToString writes for the value x.
B2_HD int rle_char_len(long long x) {
  int n = 0;
  for (bool more = true; more; ++n) {
    const long long c = x & 0x1f;
    x >>= 5;
    more = (c & 0x10) ? x != -1 : x != 0;
  }
  return n;
}

B2_HD int rle_emit(long long x, char* out) {
  int n = 0;
  for (bool more = true; more;) {
    long long c = x & 0x1f;
    x >>= 5;
    more = (c & 0x10) ? x != -1 : x != 0;
    if (more) c |= 0x20;
    out[n++] = static_cast<char>(c + 48);
  }
  return n;
}

}  // namespace b2
