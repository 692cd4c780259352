// Non-GEMM kernels of the EfficientNet backbone (EfficientDet config) and of the wrapper's input pre-processing.
// The 1x1 expand / project convolutions and the (im2col-packed) stem run on the wgmma conv kernel.
//
// Reference ops replaced: EfficientDet.build_preprocess (efficientdet_wrapper.py:40-61) + InputProcessor
// (efficientdet/dataloader.py:56-123: convert_image_dtype, mean/std, tf.image.resize_images BILINEAR,
// pad_to_bounding_box); MBConvBlock's DepthwiseConv2D SAME + BN + swish (efficientnet_model.py:255-268,363-364) and
// squeeze-excite (_call_se :300-326); Model's stem Conv2D 3x3/2 SAME (:519-531).
#include "common.h"
#include "kernels.h"
#include "planes.cuh"
#include "tf_resize_math.h"

namespace b2 {
namespace {

// uint8 BGR frame -> RGB, * 1/255, (x - mean) / std, TF1's legacy bilinear resize (tf_resize_math.h) to (sh, sw),
// zero-padded bottom/right to [H, W, 3] fp32.  The reference normalises first and resizes the float image; lerp of
// normalised corner values is done in the same order here.  Image blockIdx.y reads its frame and sizes from
// table[blockIdx.y] and writes out[blockIdx.y].
__global__ void effnet_preprocess_kernel(const uint8_t* __restrict__ frames, const EffnetFrame* __restrict__ table,
                                         float* __restrict__ out, int H, int W) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= H * W) return;
  const EffnetFrame f = table[blockIdx.y];
  const uint8_t* img = frames + f.src;
  const int h = f.h, w = f.w, sh = f.sh, sw = f.sw;
  const float ys = f.ys, xs = f.xs;
  out += static_cast<size_t>(blockIdx.y) * H * W * 3;
  const int y = idx / W, x = idx - y * W;
  float r[3] = {0.f, 0.f, 0.f};
  if (y < sh && x < sw) {
    const TfResizeTap ty = tf_resize_tap(y, ys, h), tx = tf_resize_tap(x, xs, w);
    const float mean[3] = {0.485f, 0.456f, 0.406f}, stdv[3] = {0.229f, 0.224f, 0.225f};
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const int sc = 2 - c;   // BGR -> RGB
      auto px = [&](int yy, int xx) {
        const float v = __fmul_rn(static_cast<float>(img[(static_cast<size_t>(yy) * w + xx) * 3 + sc]), 1.0f / 255.0f);
        return __fdiv_rn(__fsub_rn(v, mean[c]), stdv[c]);
      };
      r[c] = tf_resize_lerp(px(ty.lo, tx.lo), px(ty.lo, tx.hi), px(ty.hi, tx.lo), px(ty.hi, tx.hi), tx.lerp, ty.lerp);
    }
  }
  float* o = out + static_cast<size_t>(idx) * 3;
  o[0] = r[0]; o[1] = r[1]; o[2] = r[2];
}

// stem operand: 3x3/2 SAME patches of the fp32 images [B][H][W][3] as one 64-channel pixel (k = (r*3 + s)*3 + c, 27 live)
__global__ void stem_im2col_kernel(const float* __restrict__ img, int B, int H, int W, int Ho, int Wo, int pad_t, int pad_l,
                                   __half* __restrict__ out_hi, __half* __restrict__ out_lo) {
  const size_t idx = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;   // (image, pixel, octet)
  if (idx >= static_cast<size_t>(B) * Ho * Wo * 8) return;
  const int oct = static_cast<int>(idx & 7);
  const size_t pix = idx >> 3;                       // image-major: the output pixel of the [B][Ho][Wo] operand
  const size_t b = pix / (static_cast<size_t>(Ho) * Wo), rem = pix - b * Ho * Wo;
  img += b * H * W * 3;
  const int y = static_cast<int>(rem / Wo), x = static_cast<int>(rem - static_cast<size_t>(y) * Wo);
  float v[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int k = oct * 8 + j;
    float t = 0.f;
    if (k < 27) {
      const int c = k % 3, rs = k / 3, r = rs / 3, s = rs - r * 3;
      const int iy = 2 * y - pad_t + r, ix = 2 * x - pad_l + s;
      if (iy >= 0 && iy < H && ix >= 0 && ix < W) t = __ldg(img + (static_cast<size_t>(iy) * W + ix) * 3 + c);
    }
    v[j] = t;
  }
  store8(out_hi, out_lo, pix * 64 + oct * 8, v);
}

// depthwise KxK, stride 1/2, TF SAME padding, optional bias (folded BatchNorm shift) and swish.
// One thread = 8 channels x a strip of TX output pixels along x: every input column of a row is loaded once and feeds
// up to K outputs, the K*K weight vectors are loaded once per strip; loads are branch-free (clamped address, zeroed
// value) so that a whole row of 16-byte loads is in flight at a time.
template <int K, int S, int TX, bool ACT>
__global__ void __launch_bounds__(128) dw_strip_kernel(const __grid_constant__ DwConvParams p) {
  constexpr int NC = (TX - 1) * S + K;
  const int cvec = p.C / 8;
  const int strips = (p.Wo + TX - 1) / TX;
  const size_t total = static_cast<size_t>(p.B) * p.Ho * strips * cvec;
  for (size_t idx = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int cv = static_cast<int>(idx % cvec);
    const size_t rest = idx / cvec;
    const int sx = static_cast<int>(rest % strips), by = static_cast<int>(rest / strips);   // by = image * Ho + y
    const int b = by / p.Ho, y = by - b * p.Ho;
    const size_t in_img = static_cast<size_t>(b) * p.H;    // first input row of image b
    const int x0 = sx * TX;
    float acc[TX][8];
    {
      float b[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      if (p.bias != nullptr) {
        const float4* bp = reinterpret_cast<const float4*>(p.bias + cv * 8);
        const float4 b0 = __ldg(bp), b1 = __ldg(bp + 1);
        b[0] = b0.x; b[1] = b0.y; b[2] = b0.z; b[3] = b0.w; b[4] = b1.x; b[5] = b1.y; b[6] = b1.z; b[7] = b1.w;
      }
#pragma unroll
      for (int t = 0; t < TX; ++t)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[t][j] = b[j];
    }
    const int iy0 = y * S - p.pad_t, ix0 = x0 * S - p.pad_l;
#pragma unroll
    for (int r = 0; r < K; ++r) {
      const int iy = iy0 + r;
      const bool oky = iy >= 0 && iy < p.H;
      const int cy = min(max(iy, 0), p.H - 1);
      float col[NC][8];
#pragma unroll
      for (int i = 0; i < NC; ++i) {
        const int ix = ix0 + i;
        const bool ok = oky && ix >= 0 && ix < p.W;
        const int cx = min(max(ix, 0), p.W - 1);
        load8(p.in_hi, p.in_lo, ((in_img + cy) * p.W + cx) * p.C + cv * 8, col[i]);
        if (!ok) {
#pragma unroll
          for (int j = 0; j < 8; ++j) col[i][j] = 0.f;
        }
      }
#pragma unroll
      for (int s = 0; s < K; ++s) {
        const float4* wp = reinterpret_cast<const float4*>(p.w + static_cast<size_t>(r * K + s) * p.C + cv * 8);
        const float4 w0 = __ldg(wp), w1 = __ldg(wp + 1);
        const float w[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
        for (int t = 0; t < TX; ++t)
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[t][j] = fmaf(col[t * S + s][j], w[j], acc[t][j]);
      }
    }
#pragma unroll
    for (int t = 0; t < TX; ++t) {
      if (x0 + t >= p.Wo) break;
      if (ACT) {
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[t][j] = __fmul_rn(acc[t][j], 1.f / (1.f + expf(-acc[t][j])));
      }
      store8(p.out_hi, p.out_lo, (static_cast<size_t>(by) * p.Wo + x0 + t) * p.C + cv * 8, acc[t]);
    }
  }
}

// Squeeze-excite, shared by EfficientNet's MBConv blocks and the SE-ResNet bottleneck.  Every kernel takes the image from
// blockIdx.z / blockIdx.y and touches only that image's scratch: input [B][HW][C], partial [B][nchunks][C],
// r_part [B][kSeFc1Blocks][kSeMaxNr], gate [B][C].  The chunking depends on HW alone, so an image's gate does not depend
// on the batch it is in.
//
// squeeze: per-channel partial sums over a pixel chunk.  grid (C/64, nchunks, B)
__global__ void __launch_bounds__(256) se_partial_kernel(const __half* __restrict__ in_hi, const __half* __restrict__ in_lo,
                                                         int HW, int C, int chunk, float* __restrict__ partial) {
  const int cg = blockIdx.x, ch = blockIdx.y;
  const size_t img = static_cast<size_t>(blockIdx.z) * HW * C;
  in_hi += img;
  if (in_lo != nullptr) in_lo += img;
  partial += static_cast<size_t>(blockIdx.z) * gridDim.y * C;
  const int cv = threadIdx.x & 7, pl = threadIdx.x >> 3;
  const int p0 = ch * chunk, p1 = min(p0 + chunk, HW);
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  // four independent pixel loads in flight per thread (the loop is latency-bound otherwise)
  for (int p = p0 + pl; p < p1; p += 128) {
    float v[4][8];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int pp = p + 32 * u;
      if (pp < p1) {
        load8(in_hi, in_lo, static_cast<size_t>(pp) * C + cg * 64 + cv * 8, v[u]);
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) v[u][j] = 0.f;
      }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] += (v[0][j] + v[1][j]) + (v[2][j] + v[3][j]);
  }
  __shared__ float red[32][65];
#pragma unroll
  for (int j = 0; j < 8; ++j) red[pl][cv * 8 + j] = acc[j];
  __syncthreads();
  if (threadIdx.x < 64) {
    float s = 0.f;
    for (int i = 0; i < 32; ++i) s += red[i][threadIdx.x];
    partial[static_cast<size_t>(ch) * C + cg * 64 + threadIdx.x] = s;
  }
}

// excite, stage 1: each block owns a channel slice: mean of its channels, then its share of the 1x1 reduce
//   r_part[b][j] = sum_{c in slice b} mean[c] * w1[c][j]        (w1 = HWIO of [1,1,C,nr] or dense [C, nr]: row c is
//   contiguous in j).  grid (kSeFc1Blocks, B)
constexpr int kSeFc1Blocks = 32;
constexpr int kSeMaxNr = 192;

__global__ void __launch_bounds__(256) se_fc1_kernel(const float* __restrict__ partial, int nchunks, int Cpad, int C, int nr,
                                                     float inv_hw, const float* __restrict__ w1, float* __restrict__ r_part) {
  __shared__ float red[8][kSeMaxNr];
  partial += static_cast<size_t>(blockIdx.y) * nchunks * Cpad;
  r_part += static_cast<size_t>(blockIdx.y) * gridDim.x * kSeMaxNr;
  const int cs = (C + gridDim.x - 1) / gridDim.x;
  const int c0 = blockIdx.x * cs, c1 = min(c0 + cs, C);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  float acc[kSeMaxNr / 32];
#pragma unroll
  for (int q = 0; q < kSeMaxNr / 32; ++q) acc[q] = 0.f;
  for (int c = c0 + wid; c < c1; c += 8) {
    // mean of channel c: lanes split the chunk partials
    float g = 0.f;
#pragma unroll 4
    for (int k = lane; k < nchunks; k += 32) g += partial[static_cast<size_t>(k) * Cpad + c];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) g += __shfl_xor_sync(0xffffffffu, g, o);
    g *= inv_hw;
    const float* wr = w1 + static_cast<size_t>(c) * nr;
#pragma unroll
    for (int q = 0; q < kSeMaxNr / 32; ++q) {
      const int j = q * 32 + lane;
      if (j < nr) acc[q] = fmaf(g, __ldg(wr + j), acc[q]);
    }
  }
#pragma unroll
  for (int q = 0; q < kSeMaxNr / 32; ++q) red[wid][q * 32 + lane] = acc[q];
  __syncthreads();
  for (int j = threadIdx.x; j < nr; j += blockDim.x) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += red[w][j];
    r_part[static_cast<size_t>(blockIdx.x) * kSeMaxNr + j] = s;
  }
}

// excite, stage 2 + optional weight fold: each block owns 64 channels of one image: r = act(sum_b r_part + b1)
// (recomputed per block, tiny; ACT = swish for MBConv, ReLU for the SE-ResNet bottleneck),
// gate_c = sigmoid(b2[c] + sum_j r_j w2[j][c]) into gate_out [B][K]; then, when w is given (MBConv),
// w'[o][c] = w[o][c] * gate_c for every output row o of the projection conv, written as (hi, lo) operand planes: one
// folded copy per image, [B][rows][K].  grid (K/64, B)
enum class SeAct { kSwish, kRelu };

template <SeAct ACT>
__global__ void __launch_bounds__(256) se_fc2_scale_kernel(const float* __restrict__ r_part, int nparts, int C, int nr,
                                                           const float* __restrict__ b1, const float* __restrict__ w2,
                                                           const float* __restrict__ b2, float* __restrict__ gate_out,
                                                           const float* __restrict__ w, int rows, int K,
                                                           __half* __restrict__ hi, __half* __restrict__ lo) {
  __shared__ float r[kSeMaxNr];
  __shared__ float part[4][64];
  __shared__ float gate[64];
  r_part += static_cast<size_t>(blockIdx.y) * nparts * kSeMaxNr;
  gate_out += static_cast<size_t>(blockIdx.y) * K;
  for (int j = threadIdx.x; j < nr; j += blockDim.x) {
    float a = b1[j];
#pragma unroll 8
    for (int b = 0; b < nparts; ++b) a += __ldg(r_part + static_cast<size_t>(b) * kSeMaxNr + j);
    r[j] = ACT == SeAct::kSwish ? a * (1.f / (1.f + expf(-a))) : fmaxf(a, 0.f);
  }
  __syncthreads();
  const int c0 = blockIdx.x * 64;
  {
    const int c = c0 + (threadIdx.x & 63), grp = threadIdx.x >> 6;
    float a = 0.f;
    if (c < C) {
#pragma unroll 8
      for (int j = grp; j < nr; j += 4) a = fmaf(r[j], __ldg(w2 + static_cast<size_t>(j) * C + c), a);
    }
    part[grp][threadIdx.x & 63] = a;
  }
  __syncthreads();
  if (threadIdx.x < 64) {
    const int c = c0 + threadIdx.x;
    float a = 0.f;
    if (c < C) {
      a = b2[c] + ((part[0][threadIdx.x] + part[1][threadIdx.x]) + (part[2][threadIdx.x] + part[3][threadIdx.x]));
      a = 1.f / (1.f + expf(-a));
    }
    gate[threadIdx.x] = a;
    gate_out[c] = a;
  }
  if (w == nullptr) return;   // gate only (uniform across the block)
  __syncthreads();
  const size_t img = static_cast<size_t>(blockIdx.y) * rows * K;
  const int cc = threadIdx.x & 63;
  const float g = gate[cc];
  for (int o = threadIdx.x >> 6; o < rows; o += 4) {
    const size_t idx = static_cast<size_t>(o) * K + c0 + cc;
    store1(hi, lo, img + idx, __fmul_rn(w[idx], g));
  }
}

}  // namespace

EffnetFrame effnet_frame(unsigned long long src, int h, int w, int sh, int sw) {
  EffnetFrame f;
  f.src = src; f.h = h; f.w = w; f.sh = sh; f.sw = sw;
  f.ys = tf_resize_scale(h, sh);
  f.xs = tf_resize_scale(w, sw);
  return f;
}

int effnet_preprocess_launch(const uint8_t* frames, const EffnetFrame* table, int B, float* out, int H, int W, cudaStream_t s) {
  B2_CHECK(B >= 1 && B <= 65535, "effnet preprocess: batch out of range");
  effnet_preprocess_kernel<<<dim3((H * W + 255) / 256, B), 256, 0, s>>>(frames, table, out, H, W);
  B2_CUDA(cudaGetLastError());
  return 0;
}

int stem_im2col_launch(const float* img, int B, int H, int W, int Ho, int Wo, int pad_t, int pad_l, __half* out_hi,
                       __half* out_lo, cudaStream_t s) {
  const size_t total = static_cast<size_t>(B) * Ho * Wo * 8;
  stem_im2col_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, s>>>(img, B, H, W, Ho, Wo, pad_t, pad_l, out_hi,
                                                                                 out_lo);
  B2_CUDA(cudaGetLastError());
  return 0;
}

template <int K, int S>
int dw_strip_launch(const DwConvParams& p, bool act, cudaStream_t s) {
  constexpr int TX = S == 2 ? 2 : 4;
  const size_t total = static_cast<size_t>(p.B) * p.Ho * ((p.Wo + TX - 1) / TX) * (p.C / 8);
  const unsigned grid = grid_for(total, 128, 132 * 64);
  if (act) dw_strip_kernel<K, S, TX, true><<<grid, 128, 0, s>>>(p);
  else dw_strip_kernel<K, S, TX, false><<<grid, 128, 0, s>>>(p);
  B2_CUDA(cudaGetLastError());
  return 0;
}

// act: 0 none, 2 swish.  p.bias may be null (plain depthwise half of a separable conv).
int dwconv_launch(const DwConvParams& p, int act, cudaStream_t s) {
  B2_CHECK(p.B >= 1 && p.C % 8 == 0 && (p.K == 3 || p.K == 5) && (p.stride == 1 || p.stride == 2),
           "dwconv: unsupported geometry");
  const bool a = act != 0;
  if (p.K == 3 && p.stride == 1) return dw_strip_launch<3, 1>(p, a, s);
  if (p.K == 3 && p.stride == 2) return dw_strip_launch<3, 2>(p, a, s);
  if (p.K == 5 && p.stride == 1) return dw_strip_launch<5, 1>(p, a, s);
  return dw_strip_launch<5, 2>(p, a, s);
}

int dwconv_bn_swish_launch(const DwConvParams& p, cudaStream_t s) { return dwconv_launch(p, 2, s); }

int se_chunks(int HW) {
  int n = (HW + 511) / 512;
  return n < 1 ? 1 : (n > 1024 ? 1024 : n);
}

int se_fc1_parts() { return kSeFc1Blocks; }
int se_max_nr() { return kSeMaxNr; }

int se_squeeze_launch(const __half* in_hi, const __half* in_lo, int B, int HW, int Cpad, float* partial, cudaStream_t s) {
  B2_CHECK(Cpad % 64 == 0 && B >= 1 && HW >= 1, "se squeeze: bad geometry");
  const int nch = se_chunks(HW), chunk = (HW + nch - 1) / nch;
  se_partial_kernel<<<dim3(Cpad / 64, nch, B), 256, 0, s>>>(in_hi, in_lo, HW, Cpad, chunk, partial);
  B2_CUDA(cudaGetLastError());
  return 0;
}

int se_excite_launch(const float* partial, int B, int HW, int Cpad, int C, int nr, float* r_part, const float* w1,
                     const float* b1, const float* w2, const float* b2, int relu, float* gate, const float* w, int rows,
                     __half* w_hi, __half* w_lo, cudaStream_t s) {
  B2_CHECK(Cpad % 64 == 0 && nr >= 1 && nr <= kSeMaxNr, "se excite: channel count out of range");
  se_fc1_kernel<<<dim3(kSeFc1Blocks, B), 256, 0, s>>>(partial, se_chunks(HW), Cpad, C, nr, 1.0f / static_cast<float>(HW),
                                                       w1, r_part);
  const dim3 grid(Cpad / 64, B);
  if (relu)
    se_fc2_scale_kernel<SeAct::kRelu><<<grid, 256, 0, s>>>(r_part, kSeFc1Blocks, C, nr, b1, w2, b2, gate, w, rows, Cpad,
                                                           w_hi, w_lo);
  else
    se_fc2_scale_kernel<SeAct::kSwish><<<grid, 256, 0, s>>>(r_part, kSeFc1Blocks, C, nr, b1, w2, b2, gate, w, rows, Cpad,
                                                            w_hi, w_lo);
  B2_CUDA(cudaGetLastError());
  return 0;
}

// squeeze-excite of one MBConv block over B images, each gate folded into its image's copy of the projection weights
// (w [rows][K=Cpad] fp32 master copy -> [B][rows][K] planes)
int se_gate_launch(const __half* in_hi, const __half* in_lo, int B, int HW, int Cpad, int C, int nr, float* partial,
                   float* r_part, const float* w1, const float* b1, const float* w2, const float* b2, float* gate,
                   const float* w, int rows, __half* w_hi, __half* w_lo, cudaStream_t s) {
  if (se_squeeze_launch(in_hi, in_lo, B, HW, Cpad, partial, s)) return -1;
  return se_excite_launch(partial, B, HW, Cpad, C, nr, r_part, w1, b1, w2, b2, 0, gate, w, rows, w_hi, w_lo, s);
}

}  // namespace b2
