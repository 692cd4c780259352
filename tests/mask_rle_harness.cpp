// Host harness around csrc/mask_rle_math.h (the arithmetic of mask_rle.cu): lets the CPU tests check the kernels' box
// geometry, resize, threshold and RLE characters against the cv2-pinned oracle without a GPU, and the oracle's fmaf
// against C's.  Test infrastructure only -- never part of libb200det.so.
#include <math.h>
#include <stdint.h>

#include "../object_detection_tracking_b200/csrc/mask_rle_math.h"

// out[0..5] = status, x0, y0, w, h, pasted
extern "C" void mask_geometry_harness(const float* box, int H, int W, int* out) {
  b2::MaskPlace p = {0, 0, 0, 0, false};
  out[0] = b2::mask_geometry(box, H, W, &p);
  out[1] = p.x0;
  out[2] = p.y0;
  out[3] = p.w;
  out[4] = p.h;
  out[5] = p.pasted ? 1 : 0;
}

// src [28][28] -> out [h][w] float32, the values before the threshold; on [h][w] uint8 the thresholded patch
extern "C" void mask_resize_harness(const float* src, int w, int h, float* out, uint8_t* on) {
  for (int y = 0; y < h; ++y) {
    const b2::MaskTap ty = b2::mask_tap(y, h);
    for (int x = 0; x < w; ++x) {
      const float v = b2::mask_resize_at(src, b2::mask_tap(x, w), ty);
      out[y * w + x] = v;
      on[y * w + x] = b2::mask_on(v) ? 1 : 0;
    }
  }
}

// rleToString of counts [n] (uint32 values held in int64) into out; returns the length
extern "C" int64_t rle_string_harness(const int64_t* counts, int n, char* out) {
  int64_t len = 0;
  for (int i = 0; i < n; ++i) {
    long long x = counts[i];
    if (i > 2) x -= counts[i - 2];
    const int k = b2::rle_char_len(x);
    if (b2::rle_emit(x, out + len) != k) return -1;
    len += k;
  }
  return len;
}

extern "C" void fmaf_harness(const float* a, const float* b, const float* c, float* out, int n) {
  for (int i = 0; i < n; ++i) out[i] = fmaf(a[i], b[i], c[i]);
}
