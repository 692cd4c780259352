// Arithmetic of the ReID crop-resize kernel (reid_ingest.cu): Pillow's Image.resize(size, BILINEAR) on an 8-bit RGB image,
// the torchvision T.Resize step of torchreid's FeatureExtractor (feature_extractor.py:190-196).  Pillow is a third-party
// dependency; its published algorithm (libImaging/Resample.c, 8 bits per channel, and Image.resize in PIL/Image.py) is
// restated here:
//   - per axis of size `in` resized to `out`, coefficients in double: scale = in / out, fs = max(scale, 1), support = fs
//     (the bilinear filter's support is 1), ksize = 2 * ceil(support) + 1; output index xx has centre (xx + 0.5) * scale,
//     first tap xmin = max((int)(centre - support + 0.5), 0), tap count xmax = min((int)(centre + support + 0.5), in) - xmin
//     and weights tri((x + xmin - centre + 0.5) * (1 / fs)), tri(t) = max(0, 1 - |t|), divided by their sum when it is
//     not 0;
//   - fixed point: each weight becomes (int)(w * 2^22 +- 0.5) (sign of w); a sample starts from 2^21, sums the products
//     in int32, and is shifted right by 22 and clamped to 0..255;
//   - horizontal pass first into a uint8 intermediate, then the vertical pass, except when in_h > 100 * in_w and
//     out_h < in_h (Image.resize): vertical first, then horizontal.  A pass whose size does not change is the identity
//     (the weights are exactly 1 and 0 then), so Pillow skipping it and the kernel running it agree.
// Shared by the CUDA kernel and a host harness the CPU tests compile (tests/test_reid_crop_resize_cpu.py), so the
// kernel's coefficients and sums are checked against the Pillow-pinned oracle without a GPU.
#pragma once
#include <math.h>
#include <stdint.h>

#include "resize_math.h"   // B2_HD, B2_DMUL, B2_DSUB

#if defined(__CUDA_ARCH__)
#define B2_DADD(a, b) __dadd_rn((a), (b))
#define B2_DDIV(a, b) __ddiv_rn((a), (b))
#else
#define B2_DADD(a, b) ((a) + (b))
#define B2_DDIV(a, b) ((a) / (b))
#endif

namespace b2 {

constexpr int kPilPrecisionBits = 22;   // 32 - 8 - 2: 8-bit samples times 22-bit weights fit int32 with 2 spare bits

// One axis of a resize: `in` samples to `out`.
struct PilAxis {
  int in, out, ksize;
  double scale, support, ss;   // ss = 1 / fs: Pillow multiplies by the reciprocal
};

B2_HD PilAxis pil_axis(int in, int out) {
  PilAxis a;
  a.in = in;
  a.out = out;
  a.scale = B2_DDIV(static_cast<double>(in), static_cast<double>(out));
  const double fs = a.scale < 1.0 ? 1.0 : a.scale;
  a.support = fs;                                   // bilinear support 1.0 times fs
  a.ksize = static_cast<int>(ceil(a.support)) * 2 + 1;
  a.ss = B2_DDIV(1.0, fs);
  return a;
}

// Taps of output index xx: writes the first source index to *xmin and returns the tap count (Pillow's xmax).
B2_HD int pil_bounds(const PilAxis& a, int xx, int* xmin, double* centre) {
  const double c = B2_DMUL(B2_DADD(static_cast<double>(xx), 0.5), a.scale);
  int lo = static_cast<int>(B2_DADD(B2_DSUB(c, a.support), 0.5));
  if (lo < 0) lo = 0;
  int hi = static_cast<int>(B2_DADD(B2_DADD(c, a.support), 0.5));
  if (hi > a.in) hi = a.in;
  *xmin = lo;
  *centre = c;
  return hi - lo;
}

B2_HD double pil_tap_weight(const PilAxis& a, int src, double centre) {
  double t = B2_DMUL(B2_DADD(B2_DSUB(static_cast<double>(src), centre), 0.5), a.ss);
  if (t < 0.0) t = -t;
  return t < 1.0 ? B2_DSUB(1.0, t) : 0.0;
}

// Fixed-point weights of output index xx into k[0, return value) (at most a.ksize entries); *xmin = first source index.
B2_HD int pil_coeffs(const PilAxis& a, int xx, int* k, int* xmin) {
  double centre;
  const int n = pil_bounds(a, xx, xmin, &centre);
  double ww = 0.0;
  for (int x = 0; x < n; ++x) ww = B2_DADD(ww, pil_tap_weight(a, x + *xmin, centre));
  for (int x = 0; x < n; ++x) {
    double w = pil_tap_weight(a, x + *xmin, centre);
    if (ww != 0.0) w = B2_DDIV(w, ww);
    const double f = B2_DMUL(w, static_cast<double>(1 << kPilPrecisionBits));
    k[x] = static_cast<int>(w < 0 ? B2_DADD(-0.5, f) : B2_DADD(0.5, f));
  }
  return n;
}

// A sum started from pil_round() and shifted back to a clamped uint8 (Pillow's clip8).
B2_HD int pil_round() { return 1 << (kPilPrecisionBits - 1); }
B2_HD uint8_t pil_clip8(int acc) {
  const int v = acc >> kPilPrecisionBits;
  return static_cast<uint8_t>(v < 0 ? 0 : (v > 255 ? 255 : v));
}

// Image.resize's pass order: vertical first for a crop more than 100 times taller than wide that shrinks in height.
B2_HD bool pil_vertical_first(int in_w, int in_h, int out_h) {
  return in_h > 100 * in_w && out_h < in_h;
}

}  // namespace b2
