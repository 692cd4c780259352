// The fp16 plane format of every activation (DESIGN.md §3) on the device: x = hi + lo'/2048 with hi = rn(x) and
// lo' = rn((x - hi) * 2048).  In fp16 precision there is no lo' plane, and every lo pointer below is nullptr.
// The split-MMA combine of the conv kernels (acc0 + acc1/2048) belongs to the GEMM, not to this format.
#pragma once
#include <cuda_fp16.h>
#include <stddef.h>
#include <stdint.h>

namespace b2 {

constexpr float kLoScale = 2048.0f;
constexpr float kLoInv = 1.0f / 2048.0f;

__device__ __forceinline__ void split(float v, __half& hi, __half& lo) {
  hi = __float2half_rn(v);
  lo = __float2half_rn((v - __half2float(hi)) * kLoScale);
}

__device__ __forceinline__ void split2(float v0, float v1, __half2& hi, __half2& lo) {
  hi = __floats2half2_rn(v0, v1);
  const float2 f = __half22float2(hi);
  lo = __floats2half2_rn((v0 - f.x) * kLoScale, (v1 - f.y) * kLoScale);
}

// Adds lo'/2048 to a value that already holds hi (alone, or as a term of a sum such as a residual add), in one fmaf.
__device__ __forceinline__ float join(float hi, __half lo) { return fmaf(__half2float(lo), kLoInv, hi); }

__device__ __forceinline__ float2 join2(float2 hi, __half2 lo) {
  const float2 l = __half22float2(lo);
  return make_float2(fmaf(l.x, kLoInv, hi.x), fmaf(l.y, kLoInv, hi.y));
}

// Eight channels at element offset off (16-byte aligned) as fp32, one 16-byte load per plane.  READ_ONLY loads take the
// read-only data path (__ldg), which is only correct for planes the kernel does not also write.
template <bool READ_ONLY>
__device__ __forceinline__ void load8_planes(const __half* hi, const __half* lo, size_t off, float (&v)[8]) {
  const uint4* hp = reinterpret_cast<const uint4*>(hi + off);
  const uint4 h = READ_ONLY ? __ldg(hp) : *hp;
  const __half2* hh = reinterpret_cast<const __half2*>(&h);
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    const float2 f = __half22float2(hh[t]);
    v[2 * t] = f.x;
    v[2 * t + 1] = f.y;
  }
  if (lo != nullptr) {
    const uint4* lp = reinterpret_cast<const uint4*>(lo + off);
    const uint4 l = READ_ONLY ? __ldg(lp) : *lp;
    const __half2* ll = reinterpret_cast<const __half2*>(&l);
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const float2 f = join2(make_float2(v[2 * t], v[2 * t + 1]), ll[t]);
      v[2 * t] = f.x;
      v[2 * t + 1] = f.y;
    }
  }
}

__device__ __forceinline__ void load8(const __half* hi, const __half* lo, size_t off, float (&v)[8]) {
  load8_planes<true>(hi, lo, off, v);
}

// For kernels that write the planes they read: GroupNorm apply runs in place.
__device__ __forceinline__ void load8_coherent(const __half* hi, const __half* lo, size_t off, float (&v)[8]) {
  load8_planes<false>(hi, lo, off, v);
}

// load8 with both planes' loads issued before any conversion, for ReID's kernels.  With load8, ptxas gives
// avgpool2_kernel 8 more registers (one resident block per SM fewer), and the fp16 depthwise 3x3 ran 7 % slower (H100
// 80GB HBM3, 400 W); in the EfficientNet kernels this form makes se_partial_kernel spill.
__device__ __forceinline__ void load8_early(const __half* hi, const __half* lo, size_t off, float (&v)[8]) {
  const uint4 h = __ldg(reinterpret_cast<const uint4*>(hi + off));
  uint4 l = make_uint4(0u, 0u, 0u, 0u);
  if (lo != nullptr) l = __ldg(reinterpret_cast<const uint4*>(lo + off));
  const __half2* hh = reinterpret_cast<const __half2*>(&h);
  const __half2* ll = reinterpret_cast<const __half2*>(&l);
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    float2 f = __half22float2(hh[t]);
    if (lo != nullptr) f = join2(f, ll[t]);
    v[2 * t] = f.x;
    v[2 * t + 1] = f.y;
  }
}

__device__ __forceinline__ void store8(__half* hi, __half* lo, size_t off, const float (&v)[8]) {
  uint4 h, l;
  __half2* hh = reinterpret_cast<__half2*>(&h);
  __half2* ll = reinterpret_cast<__half2*>(&l);
#pragma unroll
  for (int t = 0; t < 4; ++t) split2(v[2 * t], v[2 * t + 1], hh[t], ll[t]);
  *reinterpret_cast<uint4*>(hi + off) = h;
  if (lo != nullptr) *reinterpret_cast<uint4*>(lo + off) = l;
}

__device__ __forceinline__ void store1(__half* hi, __half* lo, size_t off, float v) {
  __half h, l;
  split(v, h, l);
  hi[off] = h;
  if (lo != nullptr) lo[off] = l;
}

// Grid of a grid-stride launch: one thread per work item, at most `cap` blocks.
inline unsigned grid_for(size_t total, int threads, unsigned cap) {
  size_t b = (total + threads - 1) / threads;
  if (b > cap) b = cap;
  if (b == 0) b = 1;
  return static_cast<unsigned>(b);
}

}  // namespace b2
