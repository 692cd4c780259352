// Device helpers shared by the proposal / NMS / post-processing kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace b2 {

// Monotone map float -> uint32 (larger float => larger key).  -0.0 and +0.0 give one key, so that equal scores of either
// sign tie by index as in tf.nn.top_k (a bare f + 0.f could be folded away, so the select is explicit).
__device__ __forceinline__ uint32_t float_key(float f) {
  const uint32_t u = f == 0.f ? 0u : __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// Composite sort key: ascending order of this key == score descending, then index ascending.
__device__ __forceinline__ uint64_t desc_key(float score, uint32_t idx) {
  return (static_cast<uint64_t>(~float_key(score)) << 32) | idx;
}

// In-place bitonic sort (ascending) of n = power-of-two 64-bit keys in shared memory, whole block.
__device__ __forceinline__ void block_bitonic_sort(uint64_t* keys, int n) {
  for (int k = 2; k <= n; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      __syncthreads();
      for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const uint64_t a = keys[i], b = keys[ixj];
          const bool up = (i & k) == 0;
          if ((a > b) == up) {
            keys[i] = b;
            keys[ixj] = a;
          }
        }
      }
    }
  }
  __syncthreads();
}

// IOU() of TensorFlow's non_max_suppression_op.cc restated in float32 with explicit round-to-nearest
// ops (no FMA contraction) so the GPU decision `iou > thr` matches the CPU oracle bit for bit.
// Box = (a0, a1, a2, a3) corner coords in any consistent (x,y)/(y,x) order.
__device__ __forceinline__ float iou_tf(const float4 a, const float4 b) {
  const float amin0 = fminf(a.x, a.z), amax0 = fmaxf(a.x, a.z);
  const float amin1 = fminf(a.y, a.w), amax1 = fmaxf(a.y, a.w);
  const float bmin0 = fminf(b.x, b.z), bmax0 = fmaxf(b.x, b.z);
  const float bmin1 = fminf(b.y, b.w), bmax1 = fmaxf(b.y, b.w);
  const float area_a = __fmul_rn(__fsub_rn(amax0, amin0), __fsub_rn(amax1, amin1));
  const float area_b = __fmul_rn(__fsub_rn(bmax0, bmin0), __fsub_rn(bmax1, bmin1));
  if (area_a <= 0.f || area_b <= 0.f) return 0.f;
  const float i0 = fmaxf(__fsub_rn(fminf(amax0, bmax0), fmaxf(amin0, bmin0)), 0.f);
  const float i1 = fmaxf(__fsub_rn(fminf(amax1, bmax1), fmaxf(amin1, bmin1)), 0.f);
  const float inter = __fmul_rn(i0, i1);
  return __fdiv_rn(inter, __fsub_rn(__fadd_rn(area_a, area_b), inter));
}

// Greedy NMS over `n` boxes already sorted by score (descending) in shared memory.
//   boxes[n] (float4), mask = scratch of n * words uint32 (words = ceil(n/32)), keep_out[<=max_keep].
// Semantics of tf.image.non_max_suppression: keep i iff IoU(i, every kept) <= thr; stop at max_keep.
// Returns the number kept (valid in all threads after the call).  Requires blockDim.x >= 32.
__device__ __forceinline__ int block_nms_sorted(const float4* boxes, int n, float thr, int max_keep, uint32_t* mask,
                                                int* keep_out, int* s_count) {
  const int words = (n + 31) >> 5;
  for (int t = threadIdx.x; t < n * words; t += blockDim.x) {
    const int i = t / words, w = t - i * words;
    const float4 bi = boxes[i];
    uint32_t bits = 0;
    const int j0 = w * 32;
    for (int jj = 0; jj < 32; ++jj) {
      const int j = j0 + jj;
      if (j > i && j < n && iou_tf(bi, boxes[j]) > thr) bits |= (1u << jj);
    }
    mask[t] = bits;
  }
  __syncthreads();
  if (threadIdx.x < 32) {
    const int lane = threadIdx.x;
    // lane l owns removed-words l, l+32, ... (n <= 2048 => at most 2 words per lane)
    uint32_t rem0 = 0, rem1 = 0;
    int kept = 0;
    for (int i = 0; i < n && kept < max_keep; ++i) {
      const int w = i >> 5;
      const uint32_t word = __shfl_sync(0xffffffffu, (w < 32) ? rem0 : rem1, w & 31);
      if (!((word >> (i & 31)) & 1u)) {
        if (lane == 0) keep_out[kept] = i;
        ++kept;
        if (lane < words) rem0 |= mask[i * words + lane];
        if (lane + 32 < words) rem1 |= mask[i * words + lane + 32];
      }
    }
    if (lane == 0) *s_count = kept;
  }
  __syncthreads();
  return *s_count;
}

// decode_bbox_target (nn.py:1518-1538) of the box logits t[0..3] (divided by the regression weights here) against the
// ROI x1 y1 x2 y2: unclipped.  Explicit rounding intrinsics, so the box is the same in every kernel that inlines it.
__device__ __forceinline__ float4 decode_box(const float* t, const float reg_w[4], float decode_clip, float4 roi) {
  const float wa = __fsub_rn(roi.z, roi.x), ha = __fsub_rn(roi.w, roi.y);
  const float xa = __fmul_rn(__fadd_rn(roi.z, roi.x), 0.5f), ya = __fmul_rn(__fadd_rn(roi.w, roi.y), 0.5f);
  const float tx = __fdiv_rn(t[0], reg_w[0]), ty = __fdiv_rn(t[1], reg_w[1]);
  const float tw = __fdiv_rn(t[2], reg_w[2]), th = __fdiv_rn(t[3], reg_w[3]);
  const float wb = __fmul_rn(expf(fminf(tw, decode_clip)), wa);
  const float hb = __fmul_rn(expf(fminf(th, decode_clip)), ha);
  const float xb = __fadd_rn(__fmul_rn(tx, wa), xa), yb = __fadd_rn(__fmul_rn(ty, ha), ya);
  return make_float4(__fsub_rn(xb, __fmul_rn(wb, 0.5f)), __fsub_rn(yb, __fmul_rn(hb, 0.5f)),
                     __fadd_rn(xb, __fmul_rn(wb, 0.5f)), __fadd_rn(yb, __fmul_rn(hb, 0.5f)));
}

// clip_boxes (nn.py:1339-1346): max(., 0), then min(., [w, h, w, h])
__device__ __forceinline__ float4 clip_box(float4 b, float img_w, float img_h) {
  return make_float4(fminf(fmaxf(b.x, 0.f), img_w), fminf(fmaxf(b.y, 0.f), img_h), fminf(fmaxf(b.z, 0.f), img_w),
                     fminf(fmaxf(b.w, 0.f), img_h));
}

}  // namespace b2
