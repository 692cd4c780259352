// DeepSORT appearance cost: L2-normalise gallery / detection rows into tensor-core operands, and the
// segmented row-min that turns the [S, N] similarity GEMM into the [T, N] cost matrix.
// The GEMM itself runs on the wgmma conv kernel (1x1 conv, split precision).
//
// Reference ops replaced: nn_matching._cosine_distance (deep_sort/nn_matching.py:31-54),
// _nn_cosine_distance (:78-96), NearestNeighborDistanceMetric.distance (:156-177).
#include "common.h"
#include "kernels.h"
#include "planes.cuh"

namespace b2 {
namespace {

// NaN-propagating min / max (PTX min.NaN / max.NaN, sm_80+): NaN if either operand is NaN, as np.minimum / np.maximum.
// fminf / fmaxf return the other operand, so a NaN distance would vanish from a minimum.
__device__ __forceinline__ float min_nan(float a, float b) {
  float r;
  asm("min.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}
__device__ __forceinline__ float max_nan(float a, float b) {
  float r;
  asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}

// one warp per row: x / max(||x||, eps) -> (hi, lo) planes, row stride ld (zero padded to ld).  eps 0: a zero row is 0/0 =
// NaN (nn_matching); eps 1e-12: F.normalize.  A NaN norm stays NaN.
__global__ void cosine_normalize_kernel(const float* __restrict__ src, int rows, int D, float eps, __half* __restrict__ hi,
                                        __half* __restrict__ lo, int ld) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* x = src + static_cast<size_t>(row) * D;
  float ss = 0.f;
  for (int c = lane; c < D; c += 32) ss = fmaf(x[c], x[c], ss);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  float nrm = sqrtf(ss);
  if (nrm < eps) nrm = eps;
  for (int c = lane; c < ld; c += 32)
    store1(hi, lo, static_cast<size_t>(row) * ld + c, c < D ? __fdiv_rn(x[c], nrm) : 0.f);
}

// cost[t][n] = min over gallery rows s in [off[t], off[t+1]) of (1 - dots[s][n]); NaN if any of them is NaN, 3.4e38 for an
// empty segment
__global__ void cosine_segmin_kernel(const float* __restrict__ dots, int ld, const int* __restrict__ off, int T, int N,
                                     float* __restrict__ cost) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= T * N) return;
  const int t = idx / N, n = idx - t * N;
  float best = 3.4e38f;
  for (int s = off[t]; s < off[t + 1]; ++s) best = min_nan(best, __fsub_rn(1.f, dots[static_cast<size_t>(s) * ld + n]));
  cost[idx] = best;
}

// plain (un-normalised) rows -> (hi, lo) planes + squared norms.  ORs *range_flag (may be null) with 1 when a finite
// component rounds to an fp16 inf (|x| >= 65520): its planes would turn a finite distance into NaN or inf.
__global__ void rows_to_planes_kernel(const float* __restrict__ src, int rows, int D, __half* __restrict__ hi,
                                      __half* __restrict__ lo, int ld, float* __restrict__ sqnorm,
                                      unsigned int* __restrict__ range_flag) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* x = src + static_cast<size_t>(row) * D;
  float ss = 0.f;
  bool out_of_range = false;
  for (int c = lane; c < ld; c += 32) {
    const float v = c < D ? x[c] : 0.f;
    ss = fmaf(v, v, ss);
    out_of_range |= fabsf(v) >= 65520.f && fabsf(v) <= 3.402823466e38f;
    store1(hi, lo, static_cast<size_t>(row) * ld + c, v);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  out_of_range = __any_sync(0xffffffffu, out_of_range);
  if (lane == 0) {
    sqnorm[row] = ss;
    if (out_of_range && range_flag != nullptr) atomicOr(range_flag, 1u);
  }
}

// out[i][j] = metric 0: 1 - dots[i][j]   metric 1: na2[i] + nb2[j] - 2 dots[i][j]
__global__ void distance_finish_kernel(const float* __restrict__ dots, int ld, int na, int nb, int metric,
                                       const float* __restrict__ na2, const float* __restrict__ nb2,
                                       float* __restrict__ out) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= na * nb) return;
  const int i = idx / nb, j = idx - i * nb;
  const float d = dots[static_cast<size_t>(i) * ld + j];
  out[idx] = metric == 0 ? __fsub_rn(1.f, d) : __fsub_rn(__fadd_rn(na2[i], nb2[j]), __fmul_rn(2.f, d));
}

// Multi-camera ReID pair cost (multi_video_reid.py:308-324 compute_feature_dist): one warp per (track i of camera 1,
// track j of camera 2); out[i][j] = min over the tracks' crops of max(0, |a|^2 + |b|^2 - 2 a.b) where gate[i][j] != 0,
// else `fill`; NaN if any distance of the block is NaN (np.clip and np.min keep NaN), `fill` for an empty track.  Lanes
// stride over the columns of track j (coalesced reads of the dot-product rows).
__global__ void pair_segmin_kernel(const float* __restrict__ dots, int ld, const float* __restrict__ na2,
                                   const float* __restrict__ nb2, const int* __restrict__ seg_a, int N,
                                   const int* __restrict__ seg_b, int M, const unsigned char* __restrict__ gate, float fill,
                                   float* __restrict__ out) {
  const int pair = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (pair >= N * M) return;
  const int i = pair / M, j = pair - i * M;
  if (gate && !gate[pair]) {
    if (lane == 0) out[pair] = fill;
    return;
  }
  const int r0 = seg_a[i], r1 = seg_a[i + 1], c0 = seg_b[j], c1 = seg_b[j + 1];
  float best = 3.4e38f;
  for (int r = r0; r < r1; ++r) {
    const float a2 = na2[r];
    const float* row = dots + static_cast<size_t>(r) * ld;
    for (int c = c0 + lane; c < c1; c += 32) {
      const float d = __fsub_rn(__fadd_rn(a2, nb2[c]), __fmul_rn(2.f, row[c]));
      best = min_nan(best, max_nan(d, 0.f));
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) best = min_nan(best, __shfl_xor_sync(0xffffffffu, best, o));
  if (lane == 0) out[pair] = (r1 > r0 && c1 > c0) ? best : fill;
}

// Tracklet re-linking distance (single_video_reid.py:291-299, torchreid's unclamped squared euclidean): one warp per entry
// p of the explicit pair list; out[p] = min over query rows r of segment pairs[p][0] and gallery columns c of segment
// pairs[p][1] of (|a|^2 + |b|^2) - 2 a.b.  No clamp at 0, no gate, no fill (the caller refuses empty segments); NaN if any
// distance of the block is NaN, as torch.min.  Only the pair's own block of the products is read.
__global__ void tracklet_pair_min_kernel(const float* __restrict__ dots, int ld, const float* __restrict__ na2,
                                         const float* __restrict__ nb2, const int* __restrict__ seg_q,
                                         const int* __restrict__ seg_g, const int* __restrict__ pairs, int P,
                                         float* __restrict__ out) {
  const int p = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (p >= P) return;
  const int qi = pairs[2 * p], gi = pairs[2 * p + 1];
  const int r0 = seg_q[qi], r1 = seg_q[qi + 1], c0 = seg_g[gi], c1 = seg_g[gi + 1];
  float best = INFINITY;
  for (int r = r0; r < r1; ++r) {
    const float a2 = na2[r];
    const float* row = dots + static_cast<size_t>(r) * ld;
    for (int c = c0 + lane; c < c1; c += 32)
      best = min_nan(best, __fsub_rn(__fadd_rn(a2, nb2[c]), __fmul_rn(2.f, row[c])));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) best = min_nan(best, __shfl_xor_sync(0xffffffffu, best, o));
  if (lane == 0) out[p] = best;
}

// torch.mean(x, 0) of each segment, restated as the float32 sum in row order divided by the row count: one thread per
// (segment, column), mean[s][d] of rows [seg[s], seg[s+1]).  Segments are not empty (the caller refuses them).
__global__ void segment_mean_kernel(const float* __restrict__ src, const int* __restrict__ seg, int D,
                                    float* __restrict__ mean) {
  const int d = blockIdx.y * blockDim.x + threadIdx.x;
  const int s = blockIdx.x;
  if (d >= D) return;
  const int r0 = seg[s], r1 = seg[s + 1];
  float sum = 0.f;
  for (int r = r0; r < r1; ++r) sum = __fadd_rn(sum, src[static_cast<size_t>(r) * D + d]);
  mean[static_cast<size_t>(s) * D + d] = __fdiv_rn(sum, static_cast<float>(r1 - r0));
}

}  // namespace

int rows_to_planes(const float* src, int rows, int D, __half* hi, __half* lo, int ld, float* sqnorm,
                   unsigned int* range_flag, cudaStream_t s) {
  if (rows <= 0) return 0;
  rows_to_planes_kernel<<<(rows * 32 + 255) / 256, 256, 0, s>>>(src, rows, D, hi, lo, ld, sqnorm, range_flag);
  B2_CUDA(cudaGetLastError());
  return 0;
}

int distance_finish(const float* dots, int ld, int na, int nb, int metric, const float* na2, const float* nb2, float* out,
                    cudaStream_t s) {
  if (na * nb <= 0) return 0;
  distance_finish_kernel<<<(na * nb + 255) / 256, 256, 0, s>>>(dots, ld, na, nb, metric, na2, nb2, out);
  B2_CUDA(cudaGetLastError());
  return 0;
}

int pair_segmin(const float* dots, int ld, const float* na2, const float* nb2, const int* seg_a, int N, const int* seg_b,
                int M, const unsigned char* gate, float fill, float* out, cudaStream_t s) {
  if (N * M <= 0) return 0;
  const long long threads = static_cast<long long>(N) * M * 32;
  pair_segmin_kernel<<<static_cast<unsigned>((threads + 255) / 256), 256, 0, s>>>(dots, ld, na2, nb2, seg_a, N, seg_b, M,
                                                                                  gate, fill, out);
  B2_CUDA(cudaGetLastError());
  return 0;
}

int tracklet_pair_min(const float* dots, int ld, const float* na2, const float* nb2, const int* seg_q, const int* seg_g,
                      const int* pairs, int P, float* out, cudaStream_t s) {
  if (P <= 0) return 0;
  const long long threads = static_cast<long long>(P) * 32;
  tracklet_pair_min_kernel<<<static_cast<unsigned>((threads + 255) / 256), 256, 0, s>>>(dots, ld, na2, nb2, seg_q, seg_g,
                                                                                        pairs, P, out);
  B2_CUDA(cudaGetLastError());
  return 0;
}

int segment_mean(const float* src, const int* seg, int S, int D, float* mean, cudaStream_t s) {
  if (S <= 0 || D <= 0) return 0;
  segment_mean_kernel<<<dim3(S, (D + 255) / 256), 256, 0, s>>>(src, seg, D, mean);
  B2_CUDA(cudaGetLastError());
  return 0;
}

int cosine_normalize_rows(const float* src, int rows, int D, float eps, __half* hi, __half* lo, int ld, cudaStream_t s) {
  if (rows <= 0) return 0;
  const int threads = 256;
  const int blocks = (rows * 32 + threads - 1) / threads;
  cosine_normalize_kernel<<<blocks, threads, 0, s>>>(src, rows, D, eps, hi, lo, ld);
  B2_CUDA(cudaGetLastError());
  return 0;
}

int cosine_segmin(const float* dots, int ld, const int* seg_offsets, int T, int N, float* cost, cudaStream_t s) {
  if (T * N <= 0) return 0;
  cosine_segmin_kernel<<<(T * N + 255) / 256, 256, 0, s>>>(dots, ld, seg_offsets, T, N, cost);
  B2_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace b2
