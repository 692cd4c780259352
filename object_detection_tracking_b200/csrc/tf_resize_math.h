// Per-pixel arithmetic of TF1's legacy ResizeBilinear (tf.image.resize_images(..., BILINEAR) with align_corners=False,
// half_pixel_centers=False; tensorflow/core/kernels/resize_bilinear_op.cc LegacyScaler + compute_lerp):
//   scale = float(in_size) / out_size            (float32, computed once per axis by the caller)
//   in    = out * scale,  lo = floor(in),  hi = min(ceil(in), in_size - 1),  lerp = in - lo
//   top   = tl + (tr - tl) * lx,  bot = bl + (br - bl) * lx,  out = top + (bot - top) * ly
// every step rounded on its own (no FMA contraction).  Shared by EfficientDet's input pre-processing (effnet.cu) and the
// detector's scene feature, p5 resized to 7 x 7 (engine.cu, models.py:517-518); oracle/efficientnet.py
// resize_bilinear_legacy restates it in NumPy.
#pragma once
#include <math.h>

#ifdef __CUDACC__
#define B2_TF_HD __host__ __device__ __forceinline__
#else
#define B2_TF_HD inline
#endif

namespace b2 {

B2_TF_HD float tf_rn_mul(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}
B2_TF_HD float tf_rn_add(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fadd_rn(a, b);
#else
  return a + b;
#endif
}
B2_TF_HD float tf_rn_sub(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fsub_rn(a, b);
#else
  return a - b;
#endif
}

// The scale of one axis: in_size / out_size in float32.
inline float tf_resize_scale(int in_size, int out_size) {
  return static_cast<float>(in_size) / static_cast<float>(out_size);
}

struct TfResizeTap {
  int lo, hi;      // source indices
  float lerp;      // weight of hi
};

B2_TF_HD TfResizeTap tf_resize_tap(int out, float scale, int in_size) {
  const float in = tf_rn_mul(static_cast<float>(out), scale);
  const float fl = floorf(in);
  TfResizeTap t;
  t.lo = static_cast<int>(fl);
  const int c = static_cast<int>(ceilf(in));
  t.hi = c < in_size - 1 ? c : in_size - 1;
  t.lerp = tf_rn_sub(in, fl);
  return t;
}

B2_TF_HD float tf_resize_lerp(float tl, float tr, float bl, float br, float lx, float ly) {
  const float top = tf_rn_add(tl, tf_rn_mul(tf_rn_sub(tr, tl), lx));
  const float bot = tf_rn_add(bl, tf_rn_mul(tf_rn_sub(br, bl), lx));
  return tf_rn_add(top, tf_rn_mul(tf_rn_sub(bot, top), ly));
}

}  // namespace b2
