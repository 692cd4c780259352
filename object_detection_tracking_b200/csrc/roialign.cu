// Multi-level ROIAlign: FPN level selection + 14x14 bilinear crop + 2x2 average, one kernel.
// One warp per (roi, output bin); lane = 8 consecutive channels (16-byte loads, C = 256).
//
// Reference ops replaced: fpn_map_rois_to_levels (models.py:439-461), multilevel_roi_align
// (models.py:465-485), roi_align (nn.py:1326-1335), crop_and_resize + transform_fpcoor_for_tf
// (nn.py:1229-1280) i.e. tf.image.crop_and_resize(bilinear, extrapolation 0) + tf.nn.avg_pool 2x2.
// The float32 op sequence (normalise to [0,1] box coords, de-normalise inside CropAndResize) is kept
// op for op, with explicit round-to-nearest intrinsics so no FMA contraction changes the sample grid.
#include "common.h"
#include "kernels.h"
#include "planes.cuh"

namespace b2 {
namespace {

constexpr int kOut = 7;      // box head / fpn_box_feat resolution (level_roi_feat_kernel, default of roialign_kernel)

struct Axis {
  int lo[2], hi[2];
  float lerp[2];
  bool ok[2];
};

// sample coordinates of the two crop rows/cols (2*bin, 2*bin+1) along one axis of size `dim`; kCrop = 2 * output bins
template <int kCrop = 2 * kOut>
__device__ __forceinline__ Axis make_axis(float c0, float c1, int dim, int bin) {
  const float dm1 = static_cast<float>(dim - 1);
  const float spacing = __fdiv_rn(__fsub_rn(c1, c0), static_cast<float>(kCrop));
  const float n0 = __fdiv_rn(__fsub_rn(__fadd_rn(c0, __fdiv_rn(spacing, 2.f)), 0.5f), dm1);
  const float nlen = __fdiv_rn(__fmul_rn(spacing, static_cast<float>(kCrop - 1)), dm1);
  const float n1 = __fadd_rn(n0, nlen);
  // CropAndResize: scale = (n1 - n0) * (dim-1) / (crop-1); in = n0 * (dim-1) + i * scale
  const float scale = __fdiv_rn(__fmul_rn(__fsub_rn(n1, n0), dm1), static_cast<float>(kCrop - 1));
  const float base = __fmul_rn(n0, dm1);
  Axis a;
#pragma unroll
  for (int t = 0; t < 2; ++t) {
    // A 1-pixel axis samples its only pixel: the (dim - 1) normalisation makes every coordinate NaN there, which TF casts
    // to an index (undefined).  A NaN coordinate on a longer axis (an infinite box side) is outside: extrapolation value.
    const float in = dim == 1 ? 0.f : __fadd_rn(base, __fmul_rn(static_cast<float>(2 * bin + t), scale));
    a.ok[t] = in >= 0.f && in <= dm1;
    const float inc = fminf(fmaxf(in, 0.f), dm1);
    const float fl = floorf(inc);
    a.lo[t] = static_cast<int>(fl);
    a.hi[t] = static_cast<int>(ceilf(inc));
    a.lerp[t] = __fsub_rn(inc, fl);
  }
  return a;
}

template <int kOut>
__global__ void __launch_bounds__(256) roialign_kernel(const __grid_constant__ RoiAlignParams p) {
  const int lane = threadIdx.x & 31;
  const size_t wid = (blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x) >> 5;
  const size_t total = static_cast<size_t>(p.B) * p.rois_per_image * kOut * kOut;
  if (wid >= total) return;
  const int bin = static_cast<int>(wid % (kOut * kOut));
  const size_t roi = wid / (kOut * kOut);
  const int b = static_cast<int>(roi / p.rois_per_image);
  const int j = static_cast<int>(roi % p.rois_per_image);
  const int oy = bin / kOut, ox = bin % kOut;
  const int c0 = lane * 8;
  float acc[8];
#pragma unroll
  for (int t = 0; t < 8; ++t) acc[t] = 0.f;
  const bool live = j < p.count[b];
  if (live) {
    const float4 bx = __ldg(reinterpret_cast<const float4*>(p.boxes) + roi);
    // level = floor(4 + log(sqrt(area) / 224 + 1e-6) / log 2), clamped to [2, 5]
    const float area = __fmul_rn(__fsub_rn(bx.w, bx.y), __fsub_rn(bx.z, bx.x));
    const float sq = sqrtf(area);
    const float lg = __fmul_rn(logf(__fadd_rn(__fmul_rn(sq, 1.0f / 224), 1e-6f)), 1.4426950408889634f);
    int lvl = static_cast<int>(floorf(__fadd_rn(4.f, lg)));
    lvl = min(max(lvl, 2), 5) - 2;
    const float is = p.inv_stride[lvl];
    const int H = p.H[lvl], W = p.W[lvl];
    const Axis ay = make_axis<2 * kOut>(__fmul_rn(bx.y, is), __fmul_rn(bx.w, is), H, oy);
    const Axis ax = make_axis<2 * kOut>(__fmul_rn(bx.x, is), __fmul_rn(bx.z, is), W, ox);
    const __half* fh = p.feat_hi[lvl];
    const __half* fl = p.feat_lo[lvl];
    const size_t img_off = static_cast<size_t>(p.one_image ? 0 : b) * p.pitch_H[lvl] * p.pitch_W[lvl];
    // avg-pool order: (dy,dx) = (0,0) + (0,1) + (1,0) + (1,1), then / 4
#pragma unroll
    for (int dy = 0; dy < 2; ++dy) {
#pragma unroll
      for (int dx = 0; dx < 2; ++dx) {
        if (!(ay.ok[dy] && ax.ok[dx])) continue;   // extrapolation value 0
        float tl[8], tr[8], bl[8], br[8];
        const size_t r0 = (img_off + static_cast<size_t>(ay.lo[dy]) * p.pitch_W[lvl]);
        const size_t r1 = (img_off + static_cast<size_t>(ay.hi[dy]) * p.pitch_W[lvl]);
        load8(fh, fl, (r0 + ax.lo[dx]) * p.C + c0, tl);
        load8(fh, fl, (r0 + ax.hi[dx]) * p.C + c0, tr);
        load8(fh, fl, (r1 + ax.lo[dx]) * p.C + c0, bl);
        load8(fh, fl, (r1 + ax.hi[dx]) * p.C + c0, br);
        const float xl = ax.lerp[dx], yl = ay.lerp[dy];
#pragma unroll
        for (int t = 0; t < 8; ++t) {
          const float top = __fadd_rn(tl[t], __fmul_rn(__fsub_rn(tr[t], tl[t]), xl));
          const float bot = __fadd_rn(bl[t], __fmul_rn(__fsub_rn(br[t], bl[t]), xl));
          acc[t] = __fadd_rn(acc[t], __fadd_rn(top, __fmul_rn(__fsub_rn(bot, top), yl)));
        }
      }
    }
#pragma unroll
    for (int t = 0; t < 8; ++t) acc[t] = __fdiv_rn(acc[t], 4.f);
  }
  if (p.out_nchw) {
    float* o = p.out_nchw + (roi * p.C + c0) * (kOut * kOut) + bin;
#pragma unroll
    for (int t = 0; t < 8; ++t) o[static_cast<size_t>(t) * kOut * kOut] = acc[t];
  }
  if (p.out_hi) store8(p.out_hi, p.out_lo, (roi * (kOut * kOut) + bin) * p.C + c0, acc);
}

// EfficientDet box feature: ROIAlign 7x7 on the detection's own pyramid level, then the mean of the 49 bins.
// One block per detection (blockIdx.x) of image blockIdx.y, one thread per channel octet.
__global__ void level_roi_feat_kernel(const __grid_constant__ LevelRoiFeatParams p) {
  const int roi = blockIdx.x, img = blockIdx.y;
  const size_t slot = static_cast<size_t>(img) * p.max_out + roi;
  const int cvec = p.C / 8;
  const bool live = roi < p.count[img];
  float4 bx = make_float4(0.f, 0.f, 0.f, 0.f);
  int lvl = 0;
  if (live) {
    bx = __ldg(p.boxes + slot);
    lvl = p.levels[slot] - p.min_level;
  }
  for (int cv = threadIdx.x; cv < cvec; cv += blockDim.x) {
    float sum[8];
#pragma unroll
    for (int t = 0; t < 8; ++t) sum[t] = 0.f;
    if (live) {
      const float is = p.inv_stride[lvl];
      const int H = p.H[lvl], W = p.W[lvl];
      const size_t fimg = static_cast<size_t>(img) * H * W * p.C;
      const __half* fh = p.feat_hi[lvl] + fimg;
      const __half* fl = p.feat_lo[lvl] ? p.feat_lo[lvl] + fimg : nullptr;
      for (int bin = 0; bin < kOut * kOut; ++bin) {
        const int oy = bin / kOut, ox = bin % kOut;
        const Axis ay = make_axis(__fmul_rn(bx.y, is), __fmul_rn(bx.w, is), H, oy);
        const Axis ax = make_axis(__fmul_rn(bx.x, is), __fmul_rn(bx.z, is), W, ox);
        float acc[8];
#pragma unroll
        for (int t = 0; t < 8; ++t) acc[t] = 0.f;
#pragma unroll
        for (int dy = 0; dy < 2; ++dy) {
#pragma unroll
          for (int dx = 0; dx < 2; ++dx) {
            if (!(ay.ok[dy] && ax.ok[dx])) continue;
            float tl[8], tr[8], bl[8], br[8];
            const size_t r0 = static_cast<size_t>(ay.lo[dy]) * W, r1 = static_cast<size_t>(ay.hi[dy]) * W;
            load8(fh, fl, (r0 + ax.lo[dx]) * p.C + cv * 8, tl);
            load8(fh, fl, (r0 + ax.hi[dx]) * p.C + cv * 8, tr);
            load8(fh, fl, (r1 + ax.lo[dx]) * p.C + cv * 8, bl);
            load8(fh, fl, (r1 + ax.hi[dx]) * p.C + cv * 8, br);
            const float xl = ax.lerp[dx], yl = ay.lerp[dy];
#pragma unroll
            for (int t = 0; t < 8; ++t) {
              const float top = __fadd_rn(tl[t], __fmul_rn(__fsub_rn(tr[t], tl[t]), xl));
              const float bot = __fadd_rn(bl[t], __fmul_rn(__fsub_rn(br[t], bl[t]), xl));
              acc[t] = __fadd_rn(acc[t], __fadd_rn(top, __fmul_rn(__fsub_rn(bot, top), yl)));
            }
          }
        }
#pragma unroll
        for (int t = 0; t < 8; ++t) sum[t] = __fadd_rn(sum[t], __fdiv_rn(acc[t], 4.f));
      }
    }
#pragma unroll
    for (int t = 0; t < 8; ++t) {
      const int ch = cv * 8 + t;
      if (ch < p.Creal) p.out[slot * p.Creal + ch] = __fdiv_rn(sum[t], 49.f);
    }
  }
}

}  // namespace

int level_roi_feat_launch(const LevelRoiFeatParams& p, cudaStream_t s) {
  B2_CHECK(p.C % 8 == 0 && p.max_out >= 1 && p.B >= 1 && p.B <= 65535, "level_roi_feat: bad parameters");
  level_roi_feat_kernel<<<dim3(p.max_out, p.B), 64, 0, s>>>(p);
  B2_CUDA(cudaGetLastError());
  return 0;
}

int roialign_launch(const RoiAlignParams& p, cudaStream_t s) {
  B2_CHECK(p.C == 256, "roialign: C must be 256 (one 16-byte vector per lane)");
  B2_CHECK(p.out_res == 0 || p.out_res == 7 || p.out_res == 14, "roialign: out_res must be 7 or 14");
  const int res = p.out_res == 14 ? 14 : 7;
  B2_CHECK(res == 7 || p.out_nchw == nullptr, "roialign: the 14x14 variant writes planes only");
  const size_t warps = static_cast<size_t>(p.B) * p.rois_per_image * res * res;
  const unsigned blocks = static_cast<unsigned>((warps * 32 + 255) / 256);
  if (res == 14) roialign_kernel<14><<<blocks, 256, 0, s>>>(p);
  else roialign_kernel<7><<<blocks, 256, 0, s>>>(p);
  B2_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace b2
