// Frame ingest kernels: fused preprocess + stem operand pack (7x7/2 conv -> tensor-core shape), 3x3/2 max-pool, and the
// fp32 <-> (hi, lo) fp16 plane conversions.
//
// Reference ops replaced: build_preprocess (models.py:337-357), resnet_fpn_backbone stem
// (nn.py:871-900: pad [3, 2+pad32], conv0 7x7 s2 VALID + BN + ReLU, pad [1,0], MaxPooling 3x3 s2 VALID).
#include "common.h"
#include "planes.cuh"
#include "resize_math.h"

namespace b2 {
namespace {

__global__ void f32_to_planes_kernel(const float* __restrict__ src, __half* __restrict__ hi, __half* __restrict__ lo,
                                     size_t n) {
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x) * blockDim.x)
    store1(hi, lo, i, src[i]);
}

__global__ void planes_to_f32_kernel(const __half* __restrict__ hi, const __half* __restrict__ lo,
                                     float* __restrict__ dst, size_t n) {
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    float v = __half2float(hi[i]);
    if (lo) v = join(v, lo[i]);
    dst[i] = v;
  }
}

// Stem operand pack.  The 7x7 stride-2 conv on 3 channels is not a tensor-core shape, so the frame is
// re-laid out once per pass so that it becomes a 4x1 stride-1 conv on 64 channels (K = 256) that the
// wgmma implicit-GEMM kernel takes unchanged:
//   P  = normalised frame, zero padded [3 top/left, 3 bottom/right]        (torchvision conv1 7x7/2 pad 3)
//   U[b][y][q][s*12 + ry*6 + sx*3 + c] = P[b][2y + ry][2(q + s) + sx][c]   s in 0..3, ry,sx in 0..1, c in 0..2
//   conv0[p][q][o] = sum_{r<4} sum_{ch<64} U[p + r][q][ch] * W'[o][r][ch],  W'[o][r][ch] = W[2r+ry][2s+sx][c][o]
// (taps with 2r+ry == 7 or 2s+sx == 7 and channels 48..63 carry zero weights).  This is the ReID stem: RGB uint8 crops,
// torchvision ToTensor + Normalize op by op (x / 255, - mean, / std, RGB order), exact fp32, then the (hi, lo) split.
__global__ void __launch_bounds__(256) stem_pack_kernel(const uint8_t* __restrict__ img, int B, int H, int W,
                                                        __half* __restrict__ out_hi, __half* __restrict__ out_lo,
                                                        int Hu, int Wu) {
  const float mean[3] = {0.485f, 0.456f, 0.406f};      // torchvision Normalize of the extractor (RGB order)
  const float stdv[3] = {0.229f, 0.224f, 0.225f};
  const size_t total = static_cast<size_t>(B) * Hu * Wu * 8;
  for (size_t idx = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int cg = static_cast<int>(idx & 7);
    const size_t pix = idx >> 3;
    const int b = static_cast<int>(pix / (static_cast<size_t>(Hu) * Wu));
    const int rem = static_cast<int>(pix % (static_cast<size_t>(Hu) * Wu));
    const int y = rem / Wu, q = rem % Wu;
    __align__(16) __half hb[8];
    __align__(16) __half lb[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int ch = cg * 8 + j;
      float v = 0.f;
      if (ch < 48) {
        const int s = ch / 12, r12 = ch % 12;
        const int ry = r12 / 6, sx = (r12 % 6) / 3, c = r12 % 3;
        const int iy = 2 * y + ry - 3, ix = 2 * (q + s) + sx - 3;
        if (iy >= 0 && iy < H && ix >= 0 && ix < W) {
          float x = static_cast<float>(img[((static_cast<size_t>(b) * H + iy) * W + ix) * 3 + c]);
          x = __fdiv_rn(x, 255.0f);                    // ToTensor divides
          x = __fsub_rn(x, mean[c]);
          v = __fdiv_rn(x, stdv[c]);
        }
      }
      split(v, hb[j], lb[j]);
    }
    *reinterpret_cast<uint4*>(out_hi + pix * 64 + cg * 8) = *reinterpret_cast<uint4*>(hb);
    if (out_lo) *reinterpret_cast<uint4*>(out_lo + pix * 64 + cg * 8) = *reinterpret_cast<uint4*>(lb);
  }
}

// Compact form of the same operand (detector): V[b][y][x][ry*6 + sx*3 + c] = P[b][2y + ry][2x + sx][c], 12 real channels
// padded to 16, x in [0, Wu + 3).  P is the frame normalised as models.py:345-355 does it, op by op: x * (1/255), - mean,
// / std (BGR order), exact fp32, zero padded [3 top/left, 2 + pad-to-32 bottom/right] (nn.py:871-877).  The 64-channel pixel U[b][y][q][:] of the packed form is then the 64 CONSECUTIVE halves
// V[b][y][q .. q+3][0..15]: the conv's TMA map reads it with an element stride of 16 between pixels (overlapping
// windows), so the 4x width unroll is never written to memory -- 1/4 of the bytes and of the normalisation work
// (round 1: 454 MB written per batch-8 pass, 81 % issue-bound, 0.45 ms).
template <typename TIn>
__global__ void __launch_bounds__(256) stem_pack16_kernel(const TIn* __restrict__ img, int B, int H, int W,
                                                          __half* __restrict__ out_hi, __half* __restrict__ out_lo,
                                                          int Hu, int Wv) {
  const float mean[3] = {0.406f, 0.456f, 0.485f};      // BGR order (models.py:350-352)
  const float stdv[3] = {0.225f, 0.224f, 0.229f};
  const size_t total = static_cast<size_t>(B) * Hu * Wv;
  for (size_t pix = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; pix < total;
       pix += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int b = static_cast<int>(pix / (static_cast<size_t>(Hu) * Wv));
    const int rem = static_cast<int>(pix % (static_cast<size_t>(Hu) * Wv));
    const int y = rem / Wv, x = rem % Wv;
    __align__(16) __half hb[16];
    __align__(16) __half lb[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      float v = 0.f;
      if (j < 12) {
        const int ry = j / 6, sx = (j % 6) / 3, c = j % 3;
        const int iy = 2 * y + ry - 3, ix = 2 * x + sx - 3;
        if (iy >= 0 && iy < H && ix >= 0 && ix < W) {
          float t = static_cast<float>(img[((static_cast<size_t>(b) * H + iy) * W + ix) * 3 + c]);
          t = __fmul_rn(t, 1.0f / 255);
          t = __fsub_rn(t, mean[c]);
          v = __fdiv_rn(t, stdv[c]);
        }
      }
      split(v, hb[j], lb[j]);
    }
    uint4* oh = reinterpret_cast<uint4*>(out_hi + pix * 16);
    oh[0] = reinterpret_cast<uint4*>(hb)[0];
    oh[1] = reinterpret_cast<uint4*>(hb)[1];
    if (out_lo) {
      uint4* ol = reinterpret_cast<uint4*>(out_lo + pix * 16);
      ol[0] = reinterpret_cast<uint4*>(lb)[0];
      ol[1] = reinterpret_cast<uint4*>(lb)[1];
    }
  }
}

// 3x3 stride-2 max pool with one zero row/column of padding on top/left (inputs are post-ReLU, >= 0).
// Each thread handles 8 channels of one output pixel; the (hi, lo) pair of the max element is kept.
__global__ void maxpool_kernel(const __half* __restrict__ in_hi, const __half* __restrict__ in_lo, int B, int H, int W,
                               int C, __half* __restrict__ out_hi, __half* __restrict__ out_lo, int Ho, int Wo) {
  const int cvec = C / 8;
  const size_t total = static_cast<size_t>(B) * Ho * Wo * cvec;
  for (size_t idx = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int cv = static_cast<int>(idx % cvec);
    const size_t pix = idx / cvec;
    const int b = static_cast<int>(pix / (static_cast<size_t>(Ho) * Wo));
    const int rem = static_cast<int>(pix % (static_cast<size_t>(Ho) * Wo));
    const int p = rem / Wo, q = rem % Wo;
    float best[8];
    __half bh[8], bl[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      best[j] = 0.f;
      bh[j] = __float2half_rn(0.f);
      bl[j] = __float2half_rn(0.f);
    }
    for (int r = 0; r < 3; ++r) {
      const int ih = p * 2 - 1 + r;
      if (ih < 0 || ih >= H) continue;
      for (int s = 0; s < 3; ++s) {
        const int iw = q * 2 - 1 + s;
        if (iw < 0 || iw >= W) continue;
        const size_t off = ((static_cast<size_t>(b) * H + ih) * W + iw) * C + cv * 8;
        const uint4 vh = *reinterpret_cast<const uint4*>(in_hi + off);
        uint4 vl = make_uint4(0, 0, 0, 0);
        if (in_lo) vl = *reinterpret_cast<const uint4*>(in_lo + off);
        const __half* h = reinterpret_cast<const __half*>(&vh);
        const __half* l = reinterpret_cast<const __half*>(&vl);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float v = join(__half2float(h[j]), l[j]);
          if (v > best[j]) {
            best[j] = v;
            bh[j] = h[j];
            bl[j] = l[j];
          }
        }
      }
    }
    const size_t o = pix * C + cv * 8;
    *reinterpret_cast<uint4*>(out_hi + o) = *reinterpret_cast<uint4*>(bh);
    if (out_lo) *reinterpret_cast<uint4*>(out_lo + o) = *reinterpret_cast<uint4*>(bl);
  }
}

// Frame-resize ingest (nn.py:1540-1545 resizeImage = cv2.resize INTER_LINEAR on the float32 frame): uint8 HWC source
// frames -> float32 HWC frames of the network input size, one thread per destination pixel (3 channels), coalesced
// 12-byte stores; the 4 source taps of neighbouring threads share cache lines.  Arithmetic: resize_math.h.
__global__ void resize_u8_to_f32_kernel(const uint8_t* __restrict__ src, int B, int sh, int sw, float* __restrict__ dst,
                                        int dh, int dw) {
  const size_t total = static_cast<size_t>(B) * dh * dw;
  for (size_t idx = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int x = static_cast<int>(idx % dw);
    const int y = static_cast<int>((idx / dw) % dh);
    const int b = static_cast<int>(idx / (static_cast<size_t>(dw) * dh));
    const ResizeTap tx = resize_tap_x(x, sw, dw), ty = resize_tap_y(y, sh, dh);
    const uint8_t* base = src + static_cast<size_t>(b) * sh * sw * 3;
    const uint8_t* r0 = base + static_cast<size_t>(ty.i0) * sw * 3;
    const uint8_t* r1 = base + static_cast<size_t>(ty.i1) * sw * 3;
    float* o = dst + idx * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c)
      o[c] = resize_sample(static_cast<float>(r0[tx.i0 * 3 + c]), static_cast<float>(r0[tx.i1 * 3 + c]),
                           static_cast<float>(r1[tx.i0 * 3 + c]), static_cast<float>(r1[tx.i1 * 3 + c]), tx, ty);
  }
}

}  // namespace

int f32_to_planes(const float* src, __half* hi, __half* lo, size_t n, cudaStream_t s) {
  f32_to_planes_kernel<<<grid_for(n, 256, 132 * 32), 256, 0, s>>>(src, hi, lo, n);
  B2_CUDA(cudaGetLastError());
  return 0;
}
int planes_to_f32(const __half* hi, const __half* lo, float* dst, size_t n, cudaStream_t s) {
  planes_to_f32_kernel<<<grid_for(n, 256, 132 * 32), 256, 0, s>>>(hi, lo, dst, n);
  B2_CUDA(cudaGetLastError());
  return 0;
}

int stem_pack_launch(const uint8_t* img, int B, int H, int W, __half* out_hi, __half* out_lo, int Hu, int Wu,
                     cudaStream_t s) {
  const size_t total = static_cast<size_t>(B) * Hu * Wu * 8;
  stem_pack_kernel<<<grid_for(total, 256, 132 * 32), 256, 0, s>>>(img, B, H, W, out_hi, out_lo, Hu, Wu);
  B2_CUDA(cudaGetLastError());
  return 0;
}

int stem_pack16_launch(const void* img, int is_u8, int B, int H, int W, __half* out_hi, __half* out_lo, int Hu, int Wv,
                       cudaStream_t s) {
  const size_t total = static_cast<size_t>(B) * Hu * Wv;
  const unsigned grid = grid_for(total, 256, 132 * 32);
  if (is_u8)
    stem_pack16_kernel<uint8_t><<<grid, 256, 0, s>>>(static_cast<const uint8_t*>(img), B, H, W, out_hi, out_lo, Hu, Wv);
  else
    stem_pack16_kernel<float><<<grid, 256, 0, s>>>(static_cast<const float*>(img), B, H, W, out_hi, out_lo, Hu, Wv);
  B2_CUDA(cudaGetLastError());
  return 0;
}

int resize_u8_launch(const uint8_t* src, int B, int sh, int sw, float* dst, int dh, int dw, cudaStream_t s) {
  const size_t total = static_cast<size_t>(B) * dh * dw;
  resize_u8_to_f32_kernel<<<grid_for(total, 256, 132 * 32), 256, 0, s>>>(src, B, sh, sw, dst, dh, dw);
  B2_CUDA(cudaGetLastError());
  return 0;
}

int maxpool_launch(const __half* in_hi, const __half* in_lo, int B, int H, int W, int C, __half* out_hi,
                   __half* out_lo, int Ho, int Wo, cudaStream_t s) {
  const size_t total = static_cast<size_t>(B) * Ho * Wo * (C / 8);
  maxpool_kernel<<<grid_for(total, 256, 132 * 32), 256, 0, s>>>(in_hi, in_lo, B, H, W, C, out_hi, out_lo, Ho, Wo);
  B2_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace b2
