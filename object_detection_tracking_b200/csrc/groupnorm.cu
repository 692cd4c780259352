// GroupNorm at run time (group_norm, nn.py:81-108): 32 groups, statistics per sample over (C/32, H, W) as tf.nn.moments
// takes them (the mean first, then the mean of squared deviations from it), then tf.nn.batch_normalization with eps 1e-5:
//   inv = rsqrt(var + eps) * gamma,   y = x * inv + (beta - mean * inv).
//
// Three kernels, all on NHWC (hi, lo) fp16 planes (hi only in fp16 precision), all reading through the conv plan's view
// description (view extents H x W placed at (off_h, off_w) in a pitch_H x pitch_W buffer with pixel stride ld):
//   gn_stats_kernel  grid (chunks, B).  A block reduces one pixel chunk of one image to per-group (count, mean, M2).
//                    Every 16-byte load is eight channels of a pixel; a thread keeps Chan-merged moments of its channels,
//                    the block merges the threads in a fixed shuffle tree.  The last block of an image to finish (atomic
//                    ticket) merges the image's chunks in chunk order and writes (mean, var) per group.
//   gn_apply_kernel  grid (chunks, B).  Finalises (mean, var, gamma, beta) into a per-channel scale / shift table in shared
//                    memory, then y = x * inv + shift (+ residual, optionally nearest-2x upsampled) (ReLU) over the view
//                    only, in place or not, with the conv kernel's fp16 range monitor.
//   gn_roi_kernel    grid (rois).  The box head's per-ROI GroupNorm: one 7x7xC sample fits on chip, so statistics and
//                    apply run in one block.
//   se_apply_kernel  grid (chunks, B).  The SE-ResNet bottleneck's gate (use_se) through the same apply: the table is
//                    inv = gate[b][c] (from effnet.cu's squeeze-excite kernels), shift = 0.
// The chunking of an image depends only on its geometry (gn_chunks), and chunks and threads are merged in a fixed order, so
// the result for an image does not depend on the batch it is in: half-batch launches are bit-identical to full ones.
#include <algorithm>

#include "common.h"
#include "kernels.h"
#include "planes.cuh"

namespace b2 {
namespace {

constexpr int kGnThreads = 256;
constexpr int kGnGroups = 32;
constexpr float kGnEps = 1e-5f;   // tf.nn.batch_normalization(..., 1e-5) in group_norm (nn.py:105-106)

struct Moments {
  float n, mean, m2;
};

// Chan et al.: merge the moments of two disjoint sets (b into a).  Never E[x^2] - E[x]^2.
__device__ __forceinline__ void chan_merge(Moments& a, const Moments& b) {
  if (b.n == 0.f) return;
  if (a.n == 0.f) {
    a = b;
    return;
  }
  const float n = a.n + b.n;
  const float d = b.mean - a.mean;
  const float f = b.n / n;
  a.mean = fmaf(d, f, a.mean);
  a.m2 = a.m2 + b.m2 + d * d * a.n * f;
  a.n = n;
}

__device__ __forceinline__ Moments shfl_down(const Moments& m, int off) {
  return {__shfl_down_sync(0xffffffffu, m.n, off), __shfl_down_sync(0xffffffffu, m.mean, off),
          __shfl_down_sync(0xffffffffu, m.m2, off)};
}

// lane 0 ends up with the merge of all 32 lanes, always in the same order
__device__ __forceinline__ Moments warp_merge(Moments m, int lane) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    const Moments o = shfl_down(m, off);
    if (lane < off) chan_merge(m, o);
  }
  return m;
}

__device__ __forceinline__ size_t view_offset(const GnParams& p, int b, long long q, int vec) {
  const int y = static_cast<int>(q / p.W), x = static_cast<int>(q % p.W);
  return ((static_cast<size_t>(b) * p.pitch_H + y + p.off_h) * p.pitch_W + x + p.off_w) * p.ld + vec * 8;
}

// Per-group moments of pixels [q0, q1) of image b.  Thread (lane pl, vector vec) reads channels vec*8 .. vec*8+7 of every
// lanes-th pixel; NSUB = groups per 8-channel vector (1 when a group spans >= 8 channels, 2 for 4, 4 for 2).
// Result: s_grp[g] for the 32 groups (valid after the trailing __syncthreads).
template <int NSUB>
__device__ void block_moments(const GnParams& p, int b, long long q0, long long q1, Moments* s_part, Moments* s_grp) {
  constexpr int S = 8 / NSUB;
  const int tid = threadIdx.x, cvec = p.C / 8, lanes = kGnThreads / cvec;
  const int pl = tid / cvec, vec = tid % cvec;
  Moments acc[NSUB];
#pragma unroll
  for (int s = 0; s < NSUB; ++s) acc[s] = {0.f, 0.f, 0.f};
  for (long long q = q0 + pl; q < q1; q += 4LL * lanes) {
    float v[4][8];
#pragma unroll
    for (int u = 0; u < 4; ++u)
      if (q + u * lanes < q1) load8_coherent(p.x_hi, p.x_lo, view_offset(p, b, q + u * lanes, vec), v[u]);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      if (q + u * lanes >= q1) continue;
#pragma unroll
      for (int s = 0; s < NSUB; ++s) {
        float m = 0.f;
#pragma unroll
        for (int i = 0; i < S; ++i) m += v[u][s * S + i];
        m *= 1.f / S;
        float m2 = 0.f;
#pragma unroll
        for (int i = 0; i < S; ++i) {
          const float d = v[u][s * S + i] - m;
          m2 = fmaf(d, d, m2);
        }
        chan_merge(acc[s], Moments{static_cast<float>(S), m, m2});
      }
    }
  }
#pragma unroll
  for (int s = 0; s < NSUB; ++s) s_part[tid * NSUB + s] = acc[s];
  __syncthreads();
  // group g: the entries of every pixel lane (and, for groups wider than 8 channels, of every vector of the group)
  const int warp = tid / 32, lane = tid % 32;
  const int gs = p.C / kGnGroups, vpg = gs >= 8 ? gs / 8 : 1;
  const int entries = lanes * vpg;   // <= 32 for C in {64, ..., 2048}
  for (int g = warp; g < kGnGroups; g += kGnThreads / 32) {
    Moments m = {0.f, 0.f, 0.f};
    if (lane < entries) {
      if (gs >= 8) {
        const int t = (lane / vpg) * cvec + g * vpg + lane % vpg;
        m = s_part[t * NSUB];
      } else {
        const int t = lane * cvec + g / NSUB;
        m = s_part[t * NSUB + g % NSUB];
      }
    }
    m = warp_merge(m, lane);
    if (lane == 0) s_grp[g] = m;
  }
  __syncthreads();
}

// y = x * inv + shift (+ residual) (ReLU) over view pixels [q0, q1) of image b; s_inv / s_shift hold C entries
__device__ void apply_range(const GnParams& p, int b, long long q0, long long q1, const float* s_inv,
                            const float* s_shift) {
  const int tid = threadIdx.x, cvec = p.C / 8, lanes = kGnThreads / cvec;
  const int pl = tid / cvec, vec = tid % cvec;
  if (pl >= lanes) return;
  float amax = 0.f;
  for (long long q = q0 + pl; q < q1; q += lanes) {
    const size_t off = view_offset(p, b, q, vec);
    float v[8];
    load8_coherent(p.x_hi, p.x_lo, off, v);
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = v[i] * s_inv[vec * 8 + i] + s_shift[vec * 8 + i];
    if (p.r_hi != nullptr) {
      const int y = static_cast<int>(q / p.W) >> p.res_shift, x = static_cast<int>(q % p.W) >> p.res_shift;
      const size_t roff = ((static_cast<size_t>(b) * p.res_H + y) * p.res_W + x) * p.res_ld + vec * 8;
      float r[8];
      load8_coherent(p.r_hi, p.r_lo, roff, r);
#pragma unroll
      for (int i = 0; i < 8; ++i) v[i] += r[i];
    }
    if (p.relu) {
#pragma unroll
      for (int i = 0; i < 8; ++i) v[i] = fmaxf(v[i], 0.f);
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) amax = fmaxf(amax, fabsf(v[i]));
    store8(p.y_hi, p.y_lo, off, v);
  }
  // same monitor as conv_tc_kernel: inf included, a NaN can only follow an inf an earlier launch has flagged
  if (p.range_flag != nullptr && amax > 65504.f) atomicOr(p.range_flag, 1u);
}

// inv = rsqrt(var + eps) * gamma, shift = beta - mean * inv (tf.nn.batch_normalization)
__device__ __forceinline__ void finalize_channel(const GnParams& p, int c, float mean, float var, float* s_inv,
                                                 float* s_shift) {
  const float inv = (1.f / sqrtf(var + kGnEps)) * p.gamma[c];
  s_inv[c] = inv;
  s_shift[c] = p.beta[c] - mean * inv;
}

template <int NSUB>
__global__ void __launch_bounds__(kGnThreads) gn_stats_kernel(GnParams p) {
  __shared__ Moments s_part[kGnThreads * NSUB];
  __shared__ Moments s_grp[kGnGroups];
  __shared__ int s_last;
  const int b = blockIdx.y, chunk = blockIdx.x, tid = threadIdx.x;
  const long long HW = static_cast<long long>(p.H) * p.W;
  block_moments<NSUB>(p, b, HW * chunk / p.chunks, HW * (chunk + 1) / p.chunks, s_part, s_grp);
  float* part = p.partial + (static_cast<size_t>(b) * p.chunks + chunk) * kGnGroups * 3;
  if (tid < kGnGroups) {
    part[tid * 3 + 0] = s_grp[tid].n;
    part[tid * 3 + 1] = s_grp[tid].mean;
    part[tid * 3 + 2] = s_grp[tid].m2;
  }
  __threadfence();
  __syncthreads();
  if (tid == 0) s_last = atomicAdd(p.counter + b, 1u) == static_cast<unsigned>(p.chunks - 1);
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  // the image's last block: merge its chunks in chunk order (lane l folds chunks l, l + 32, ..., then the shuffle tree)
  const int warp = tid / 32, lane = tid % 32;
  for (int g = warp; g < kGnGroups; g += kGnThreads / 32) {
    Moments m = {0.f, 0.f, 0.f};
    for (int k = lane; k < p.chunks; k += 32) {
      const float* q = p.partial + (static_cast<size_t>(b) * p.chunks + k) * kGnGroups * 3 + g * 3;
      chan_merge(m, Moments{__ldcg(q), __ldcg(q + 1), __ldcg(q + 2)});
    }
    m = warp_merge(m, lane);
    if (lane == 0) {
      p.stats[(static_cast<size_t>(b) * kGnGroups + g) * 2 + 0] = m.mean;
      p.stats[(static_cast<size_t>(b) * kGnGroups + g) * 2 + 1] = m.n > 0.f ? m.m2 / m.n : 0.f;
    }
  }
  if (tid == 0) p.counter[b] = 0u;   // re-armed for the next launch (graph replays included)
}

__global__ void __launch_bounds__(kGnThreads) gn_apply_kernel(GnParams p) {
  extern __shared__ float s_tab[];
  float* s_inv = s_tab;
  float* s_shift = s_tab + p.C;
  const int b = blockIdx.y, chunk = blockIdx.x;
  const int gs = p.C / kGnGroups;
  for (int c = threadIdx.x; c < p.C; c += kGnThreads) {
    const float* st = p.stats + (static_cast<size_t>(b) * kGnGroups + c / gs) * 2;
    finalize_channel(p, c, st[0], st[1], s_inv, s_shift);
  }
  __syncthreads();
  const long long HW = static_cast<long long>(p.H) * p.W;
  apply_range(p, b, HW * chunk / p.chunks, HW * (chunk + 1) / p.chunks, s_inv, s_shift);
}

// squeeze-excite gate of the SE-ResNet bottleneck (nn.py:506-519): the apply with inv = gate[b], shift = 0
__global__ void __launch_bounds__(kGnThreads) se_apply_kernel(GnParams p) {
  extern __shared__ float s_tab[];
  float* s_inv = s_tab;
  float* s_shift = s_tab + p.C;
  const int b = blockIdx.y, chunk = blockIdx.x;
  for (int c = threadIdx.x; c < p.C; c += kGnThreads) {
    s_inv[c] = p.gate[static_cast<size_t>(b) * p.C + c];
    s_shift[c] = 0.f;
  }
  __syncthreads();
  const long long HW = static_cast<long long>(p.H) * p.W;
  apply_range(p, b, HW * chunk / p.chunks, HW * (chunk + 1) / p.chunks, s_inv, s_shift);
}

template <int NSUB>
__global__ void __launch_bounds__(kGnThreads) gn_roi_kernel(GnParams p) {
  __shared__ Moments s_part[kGnThreads * NSUB];
  __shared__ Moments s_grp[kGnGroups];
  extern __shared__ float s_tab[];
  float* s_inv = s_tab;
  float* s_shift = s_tab + p.C;
  const int b = blockIdx.x;
  const long long HW = static_cast<long long>(p.H) * p.W;
  block_moments<NSUB>(p, b, 0, HW, s_part, s_grp);
  const int gs = p.C / kGnGroups;
  for (int c = threadIdx.x; c < p.C; c += kGnThreads) {
    const Moments& m = s_grp[c / gs];
    finalize_channel(p, c, m.mean, m.n > 0.f ? m.m2 / m.n : 0.f, s_inv, s_shift);
  }
  __syncthreads();
  apply_range(p, b, 0, HW, s_inv, s_shift);
}

int nsub_of(const GnParams& p) {
  const int gs = p.C / kGnGroups;
  return gs >= 8 ? 1 : 8 / gs;
}

int check(const GnParams& p, const char* what) {
  const int cvec = p.C / 8;
  B2_CHECK(p.C % kGnGroups == 0 && p.C >= 64 && p.C % 8 == 0 && kGnThreads % cvec == 0,
           std::string(what) + ": GroupNorm needs C in {64, 128, 256, 512, 1024, 2048} (32 groups, 16-byte loads)");
  B2_CHECK(p.ld % 8 == 0 && p.ld >= p.C && (p.r_hi == nullptr || p.res_ld % 8 == 0),
           std::string(what) + ": GroupNorm needs 16-byte aligned pixel strides");
  B2_CHECK(p.B >= 1 && p.H >= 1 && p.W >= 1 && (p.gate || (p.gamma && p.beta)), std::string(what) + ": bad GroupNorm view");
  return 0;
}

}  // namespace

int gn_chunks(int H, int W, int C) {
  const long long px = static_cast<long long>(H) * W;
  long long n = (px * C * 2 + 16383) / 16384;   // ~16 KB of the hi plane per block
  n = std::min<long long>(std::max<long long>(n, 1), 256);
  return static_cast<int>(std::min(n, px));
}

int gn_stats_launch(const GnParams& p, cudaStream_t s) {
  if (check(p, "gn_stats")) return -1;
  B2_CHECK(p.partial && p.stats && p.counter && p.chunks >= 1, "gn_stats: missing scratch");
  const dim3 grid(p.chunks, p.B);
  switch (nsub_of(p)) {
    case 1: gn_stats_kernel<1><<<grid, kGnThreads, 0, s>>>(p); break;
    case 2: gn_stats_kernel<2><<<grid, kGnThreads, 0, s>>>(p); break;
    default: gn_stats_kernel<4><<<grid, kGnThreads, 0, s>>>(p); break;
  }
  B2_CUDA(cudaGetLastError());
  return 0;
}

int gn_apply_launch(const GnParams& p, cudaStream_t s) {
  if (check(p, "gn_apply")) return -1;
  B2_CHECK(p.stats && p.chunks >= 1, "gn_apply: missing statistics");
  gn_apply_kernel<<<dim3(p.chunks, p.B), kGnThreads, 2 * p.C * sizeof(float), s>>>(p);
  B2_CUDA(cudaGetLastError());
  return 0;
}

int se_apply_launch(const GnParams& p, cudaStream_t s) {
  if (check(p, "se_apply")) return -1;
  B2_CHECK(p.gate && p.chunks >= 1, "se_apply: missing gate");
  se_apply_kernel<<<dim3(p.chunks, p.B), kGnThreads, 2 * p.C * sizeof(float), s>>>(p);
  B2_CUDA(cudaGetLastError());
  return 0;
}

int gn_roi_launch(const GnParams& p, cudaStream_t s) {
  if (check(p, "gn_roi")) return -1;
  const size_t smem = 2 * p.C * sizeof(float);
  switch (nsub_of(p)) {
    case 1: gn_roi_kernel<1><<<p.B, kGnThreads, smem, s>>>(p); break;
    case 2: gn_roi_kernel<2><<<p.B, kGnThreads, smem, s>>>(p); break;
    default: gn_roi_kernel<4><<<p.B, kGnThreads, smem, s>>>(p); break;
  }
  B2_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace b2
