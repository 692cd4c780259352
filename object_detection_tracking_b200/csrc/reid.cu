// Non-GEMM kernels of the OSNet ReID embedding (HBM-bound byte/element work; the 1x1 convolutions and
// the fc run on the wgmma implicit-GEMM kernel).
//
// Reference ops replaced (torchreid/models/osnet.py): LightConv3x3's depthwise 3x3 + BN + ReLU (:128-156),
// ChannelGate (:162-220: global avg-pool -> fc1 -> ReLU -> fc2 -> sigmoid -> scale), the 4-stream gated sum
// of OSBlock.forward (:262-268), AvgPool2d(2) of the transitions (:375-381), AdaptiveAvgPool2d(1) (:428), and the
// InstanceNorm2d of the IBN / AIN variants (:52,260; osnet_ain.py:42,281).
#include "common.h"
#include "kernels.h"
#include "planes.cuh"

namespace b2 {
namespace {

// depthwise 3x3, stride 1, pad 1, + folded BN + ReLU.  w: [9][C] fp32 (BN scale folded), bias [C].
__global__ void dwconv3x3_kernel(const __half* __restrict__ in_hi, const __half* __restrict__ in_lo, int B, int H, int W,
                                 int C, const float* __restrict__ w, const float* __restrict__ bias,
                                 __half* __restrict__ out_hi, __half* __restrict__ out_lo) {
  const int cvec = C / 8;
  const size_t total = static_cast<size_t>(B) * H * W * cvec;
  for (size_t idx = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int cv = static_cast<int>(idx % cvec);
    const size_t pix = idx / cvec;
    const int b = static_cast<int>(pix / (static_cast<size_t>(H) * W));
    const int rem = static_cast<int>(pix % (static_cast<size_t>(H) * W));
    const int y = rem / W, x = rem % W;
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const int iy = y + r - 1;
      if (iy < 0 || iy >= H) continue;
#pragma unroll
      for (int s = 0; s < 3; ++s) {
        const int ix = x + s - 1;
        if (ix < 0 || ix >= W) continue;
        float v[8];
        load8_early(in_hi, in_lo, ((static_cast<size_t>(b) * H + iy) * W + ix) * C + cv * 8, v);
        const float4* wp = reinterpret_cast<const float4*>(w + static_cast<size_t>(r * 3 + s) * C + cv * 8);
        const float4 w0 = __ldg(wp), w1 = __ldg(wp + 1);
        acc[0] = fmaf(v[0], w0.x, acc[0]); acc[1] = fmaf(v[1], w0.y, acc[1]);
        acc[2] = fmaf(v[2], w0.z, acc[2]); acc[3] = fmaf(v[3], w0.w, acc[3]);
        acc[4] = fmaf(v[4], w1.x, acc[4]); acc[5] = fmaf(v[5], w1.y, acc[5]);
        acc[6] = fmaf(v[6], w1.z, acc[6]); acc[7] = fmaf(v[7], w1.w, acc[7]);
      }
    }
    const float4* bp = reinterpret_cast<const float4*>(bias + cv * 8);
    const float4 b0 = __ldg(bp), b1 = __ldg(bp + 1);
    const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = fmaxf(acc[j] + bb[j], 0.f);
    store8(out_hi, out_lo, pix * C + cv * 8, acc);
  }
}

// global average pool: one block per (image, 64-channel group); out fp32 [B][C]
__global__ void __launch_bounds__(256) gap_kernel(const __half* __restrict__ in_hi, const __half* __restrict__ in_lo,
                                                  int HW, int C, float* __restrict__ out, int out_ld) {
  const int b = blockIdx.y, cg = blockIdx.x;          // 64 channels per block: 8 vectors x 32 pixel lanes
  const int cv = threadIdx.x & 7, pl = threadIdx.x >> 3;
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  for (int p = pl; p < HW; p += 32) {
    float v[8];
    load8_early(in_hi, in_lo, (static_cast<size_t>(b) * HW + p) * C + cg * 64 + cv * 8, v);
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] += v[j];
  }
  __shared__ float red[32][65];
#pragma unroll
  for (int j = 0; j < 8; ++j) red[pl][cv * 8 + j] = acc[j];
  __syncthreads();
  if (threadIdx.x < 64) {
    float s = 0.f;
    for (int i = 0; i < 32; ++i) s += red[i][threadIdx.x];
    out[static_cast<size_t>(b) * out_ld + cg * 64 + threadIdx.x] = s / static_cast<float>(HW);
  }
}

// ChannelGate MLP on pooled vectors: one block per pooled row.  g [rows][C] -> gates [rows][C]
// fc1: [Cr][C] + b1, ReLU, fc2: [C][Cr] + b2, sigmoid.  Only the first Creal channels are live.
__global__ void __launch_bounds__(128) gate_mlp_kernel(const float* __restrict__ g, int C, int Creal, int Cr,
                                                       const float* __restrict__ w1, const float* __restrict__ b1,
                                                       const float* __restrict__ w2, const float* __restrict__ b2,
                                                       float* __restrict__ gates) {
  __shared__ float sx[512];
  __shared__ float sh[64];
  const int row = blockIdx.x;
  for (int i = threadIdx.x; i < Creal; i += blockDim.x) sx[i] = g[static_cast<size_t>(row) * C + i];
  __syncthreads();
  if (threadIdx.x < Cr) {
    float a = b1[threadIdx.x];
    for (int i = 0; i < Creal; ++i) a = fmaf(w1[threadIdx.x * Creal + i], sx[i], a);
    sh[threadIdx.x] = fmaxf(a, 0.f);
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float out = 0.f;
    if (c < Creal) {
      float a = b2[c];
      for (int i = 0; i < Cr; ++i) a = fmaf(w2[c * Cr + i], sh[i], a);
      out = 1.f / (1.f + expf(-a));
    }
    gates[static_cast<size_t>(row) * C + c] = out;
  }
}

// x2 = gate(a)*a + gate(b)*b + gate(c)*c + gate(d)*d ; gates [B][4][C] fp32
__global__ void gated_sum4_kernel(const __half* __restrict__ a_hi, const __half* __restrict__ a_lo,
                                  const __half* __restrict__ b_hi, const __half* __restrict__ b_lo,
                                  const __half* __restrict__ c_hi, const __half* __restrict__ c_lo,
                                  const __half* __restrict__ d_hi, const __half* __restrict__ d_lo,
                                  const float* __restrict__ gates, int B, int HW, int C, __half* __restrict__ out_hi,
                                  __half* __restrict__ out_lo) {
  const int cvec = C / 8;
  const size_t total = static_cast<size_t>(B) * HW * cvec;
  const __half* his[4] = {a_hi, b_hi, c_hi, d_hi};
  const __half* los[4] = {a_lo, b_lo, c_lo, d_lo};
  for (size_t idx = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int cv = static_cast<int>(idx % cvec);
    const size_t pix = idx / cvec;
    const int b = static_cast<int>(pix / HW);
    const size_t off = pix * C + cv * 8;
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
#pragma unroll
    for (int s = 0; s < 4; ++s) {
      float v[8];
      load8_early(his[s], los[s], off, v);
      const float* gp = gates + (static_cast<size_t>(b) * 4 + s) * C + cv * 8;
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] = __fadd_rn(acc[j], __fmul_rn(v[j], __ldg(gp + j)));
    }
    store8(out_hi, out_lo, off, acc);
  }
}

// 2x2 average pool, stride 2
__global__ void avgpool2_kernel(const __half* __restrict__ in_hi, const __half* __restrict__ in_lo, int B, int H, int W,
                                int C, __half* __restrict__ out_hi, __half* __restrict__ out_lo) {
  const int Ho = H / 2, Wo = W / 2, cvec = C / 8;
  const size_t total = static_cast<size_t>(B) * Ho * Wo * cvec;
  for (size_t idx = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int cv = static_cast<int>(idx % cvec);
    const size_t pix = idx / cvec;
    const int b = static_cast<int>(pix / (static_cast<size_t>(Ho) * Wo));
    const int rem = static_cast<int>(pix % (static_cast<size_t>(Ho) * Wo));
    const int y = rem / Wo, x = rem % Wo;
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
#pragma unroll
    for (int dy = 0; dy < 2; ++dy)
#pragma unroll
      for (int dx = 0; dx < 2; ++dx) {
        float v[8];
        load8_early(in_hi, in_lo, ((static_cast<size_t>(b) * H + 2 * y + dy) * W + 2 * x + dx) * C + cv * 8, v);
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] += v[j];
      }
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] *= 0.25f;
    store8(out_hi, out_lo, pix * C + cv * 8, acc);
  }
}

// InstanceNorm2d(affine=True, track_running_stats=False) of osnet_ibn / osnet_ain (osnet.py:52,260; osnet_ain.py:42,281):
// y = (x - mean_hw) / sqrt(var_hw + 1e-5) * gamma + beta per (image, channel), biased variance, then optionally + res and
// ReLU.  One block per (image, 64-channel slab): 8 channel vectors x 64 pixel lanes.  Three passes over the slab (at most
// 8192 pixels x 64 channels, 2 MB of planes, so passes 2 and 3 read L2): the shifted mean (each channel's first pixel
// taken off, so a large mean loses no bits of a small spread), the squared deviations from that mean, then the apply.
// Every sum runs in one fixed order that depends on HW alone -- the same bits for an image at any slot of any batch.
// Only channels [0, c_norm) are normalised (IBN-a's split, resnet_ibn_a.py:63-79; c_norm a multiple of 8, C for a plain
// InstanceNorm): the others skip the statistics and pass through unchanged, then take the residual and ReLU like the rest.
constexpr int kInLanes = 64;

__global__ void __launch_bounds__(512) instnorm_kernel(const __half* __restrict__ x_hi, const __half* __restrict__ x_lo,
                                                       const __half* __restrict__ r_hi, const __half* __restrict__ r_lo,
                                                       int HW, int C, int c_norm, const float* __restrict__ gamma,
                                                       const float* __restrict__ beta, int relu, __half* __restrict__ y_hi,
                                                       __half* __restrict__ y_lo) {
  const int b = blockIdx.y, c0 = blockIdx.x * 64;
  const int cv = threadIdx.x & 7, pl = threadIdx.x >> 3;
  const bool norm = c0 + cv * 8 < c_norm;   // this thread's 8 channels are normalised
  const int hw_norm = norm ? HW : 0;        // pixels the statistics passes read
  const size_t base = static_cast<size_t>(b) * HW * C + c0 + cv * 8;
  __shared__ float red[kInLanes][65];
  __shared__ float s_mean[64], s_scale[64];
  float k[8], acc[8];
  load8_early(x_hi, x_lo, base, k);   // the shift: pixel 0 of each channel
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  for (int p = pl; p < hw_norm; p += kInLanes) {
    float v[8];
    load8_early(x_hi, x_lo, base + static_cast<size_t>(p) * C, v);
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] += v[j] - k[j];
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    red[pl][cv * 8 + j] = acc[j];
    if (pl == 0) s_mean[cv * 8 + j] = k[j];
  }
  __syncthreads();
  if (threadIdx.x < 64) {
    float s = 0.f;
    for (int i = 0; i < kInLanes; ++i) s += red[i][threadIdx.x];
    s_mean[threadIdx.x] += s / static_cast<float>(HW);
  }
  __syncthreads();
  float m[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    m[j] = s_mean[cv * 8 + j];
    acc[j] = 0.f;
  }
  for (int p = pl; p < hw_norm; p += kInLanes) {
    float v[8];
    load8_early(x_hi, x_lo, base + static_cast<size_t>(p) * C, v);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float d = v[j] - m[j];
      acc[j] = fmaf(d, d, acc[j]);
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) red[pl][cv * 8 + j] = acc[j];
  __syncthreads();
  if (threadIdx.x < 64) {
    float s = 0.f;
    for (int i = 0; i < kInLanes; ++i) s += red[i][threadIdx.x];
    const float var = s / static_cast<float>(HW);
    s_scale[threadIdx.x] = c0 + static_cast<int>(threadIdx.x) < c_norm ? gamma[c0 + threadIdx.x] / sqrtf(var + 1e-5f) : 0.f;
  }
  __syncthreads();
  float sc[8], bt[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    sc[j] = s_scale[cv * 8 + j];
    bt[j] = norm ? __ldg(beta + c0 + cv * 8 + j) : 0.f;
  }
  for (int p = pl; p < HW; p += kInLanes) {
    const size_t off = base + static_cast<size_t>(p) * C;
    float v[8];
    load8_early(x_hi, x_lo, off, v);
    if (norm) {
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = fmaf(v[j] - m[j], sc[j], bt[j]);
    }
    if (r_hi) {
      float r[8];
      load8_early(r_hi, r_lo, off, r);
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] += r[j];
    }
    if (relu) {
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = fmaxf(v[j], 0.f);
    }
    store8(y_hi, y_lo, off, v);
  }
}

}  // namespace

int instnorm_launch(const __half* x_hi, const __half* x_lo, const __half* r_hi, const __half* r_lo, int B, int HW, int C,
                    const float* gamma, const float* beta, int relu, __half* y_hi, __half* y_lo, cudaStream_t s) {
  B2_CHECK(B >= 1 && HW >= 1 && C >= 64 && C % 64 == 0, "instnorm: needs B, HW >= 1 and C a multiple of 64");
  B2_CHECK(x_hi != y_hi && (r_hi == nullptr || r_hi != y_hi), "instnorm: the output may not alias the input or residual");
  instnorm_kernel<<<dim3(C / 64, B), 512, 0, s>>>(x_hi, x_lo, r_hi, r_lo, HW, C, C, gamma, beta, relu, y_hi, y_lo);
  B2_CUDA(cudaGetLastError());
  return 0;
}

int instnorm_split_launch(const __half* x_hi, const __half* x_lo, int B, int HW, int C, int c_norm, const float* gamma,
                          const float* beta, __half* y_hi, __half* y_lo, cudaStream_t s) {
  B2_CHECK(B >= 1 && HW >= 1 && C >= 64 && C % 64 == 0 && c_norm >= 8 && c_norm <= C && c_norm % 8 == 0,
           "instnorm_split: needs B, HW >= 1, C a multiple of 64 and c_norm a multiple of 8 in [8, C]");
  B2_CHECK(x_hi != y_hi, "instnorm_split: the output may not alias the input");
  instnorm_kernel<<<dim3(C / 64, B), 512, 0, s>>>(x_hi, x_lo, nullptr, nullptr, HW, C, c_norm, gamma, beta, 1, y_hi, y_lo);
  B2_CUDA(cudaGetLastError());
  return 0;
}

int dwconv3x3_launch(const __half* in_hi, const __half* in_lo, int B, int H, int W, int C, const float* w,
                     const float* bias, __half* out_hi, __half* out_lo, cudaStream_t s) {
  const size_t total = static_cast<size_t>(B) * H * W * (C / 8);
  dwconv3x3_kernel<<<grid_for(total, 256, 132 * 32), 256, 0, s>>>(in_hi, in_lo, B, H, W, C, w, bias, out_hi, out_lo);
  B2_CUDA(cudaGetLastError());
  return 0;
}

int gap_launch(const __half* in_hi, const __half* in_lo, int B, int HW, int C, float* out, int out_ld, cudaStream_t s) {
  B2_CHECK(C % 64 == 0, "gap: C must be a multiple of 64");
  gap_kernel<<<dim3(C / 64, B), 256, 0, s>>>(in_hi, in_lo, HW, C, out, out_ld);
  B2_CUDA(cudaGetLastError());
  return 0;
}

int gate_mlp_launch(const float* g, int rows, int C, int Creal, int Cr, const float* w1, const float* b1,
                    const float* w2, const float* b2, float* gates, cudaStream_t s) {
  B2_CHECK(Creal <= 512 && Cr <= 64, "gate_mlp: channel counts out of range");
  gate_mlp_kernel<<<rows, 128, 0, s>>>(g, C, Creal, Cr, w1, b1, w2, b2, gates);
  B2_CUDA(cudaGetLastError());
  return 0;
}

int gated_sum4_launch(const __half* const hi[4], const __half* const lo[4], const float* gates, int B, int HW, int C,
                      __half* out_hi, __half* out_lo, cudaStream_t s) {
  const size_t total = static_cast<size_t>(B) * HW * (C / 8);
  gated_sum4_kernel<<<grid_for(total, 256, 132 * 32), 256, 0, s>>>(hi[0], lo[0], hi[1], lo[1], hi[2], lo[2], hi[3], lo[3],
                                                                     gates, B, HW, C, out_hi, out_lo);
  B2_CUDA(cudaGetLastError());
  return 0;
}

int avgpool2_launch(const __half* in_hi, const __half* in_lo, int B, int H, int W, int C, __half* out_hi,
                    __half* out_lo, cudaStream_t s) {
  const size_t total = static_cast<size_t>(B) * (H / 2) * (W / 2) * (C / 8);
  avgpool2_kernel<<<grid_for(total, 256, 132 * 32), 256, 0, s>>>(in_hi, in_lo, B, H, W, C, out_hi, out_lo);
  B2_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace b2
