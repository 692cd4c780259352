// Host harness around csrc/pil_resize_math.h (the arithmetic of reid_crop_resize_kernel): lets the CPU tests check the
// kernel's coefficients, fixed-point sums and pass order against the Pillow-pinned oracle without a GPU.  Like the kernel
// it runs both passes even where a size does not change.  Test infrastructure only -- never part of libb200det.so.
#include <stddef.h>
#include <stdint.h>

#include <vector>

#include "../object_detection_tracking_b200/csrc/pil_resize_math.h"

namespace {

// one pass over uint8 [h][w][3]: along x (horizontal, w -> out) or y (vertical, h -> out)
void pil_pass(const uint8_t* src, int h, int w, uint8_t* dst, int out, bool horizontal) {
  const b2::PilAxis a = b2::pil_axis(horizontal ? w : h, out);
  std::vector<int> k(a.ksize);
  const int ow = horizontal ? out : w;
  for (int o = 0; o < out; ++o) {
    int first = 0;
    const int n = b2::pil_coeffs(a, o, k.data(), &first);
    for (int p = 0; p < (horizontal ? h : w); ++p)
      for (int c = 0; c < 3; ++c) {
        int acc = b2::pil_round();
        for (int t = 0; t < n; ++t) {
          const size_t at = horizontal ? (static_cast<size_t>(p) * w + first + t) * 3 + c
                                       : (static_cast<size_t>(first + t) * w + p) * 3 + c;
          acc += src[at] * k[t];
        }
        const size_t to = horizontal ? (static_cast<size_t>(p) * ow + o) * 3 + c : (static_cast<size_t>(o) * ow + p) * 3 + c;
        dst[to] = b2::pil_clip8(acc);
      }
  }
}

}  // namespace

// src: RGB uint8 [sh][sw][3] -> dst [dh][dw][3]
extern "C" void pil_resize_harness(const uint8_t* src, int sh, int sw, uint8_t* dst, int dh, int dw) {
  if (b2::pil_vertical_first(sw, sh, dh)) {
    std::vector<uint8_t> tmp(static_cast<size_t>(dh) * sw * 3);
    pil_pass(src, sh, sw, tmp.data(), dh, false);
    pil_pass(tmp.data(), dh, sw, dst, dw, true);
  } else {
    std::vector<uint8_t> tmp(static_cast<size_t>(sh) * dw * 3);
    pil_pass(src, sh, sw, tmp.data(), dw, true);
    pil_pass(tmp.data(), sh, dw, dst, dh, false);
  }
}
