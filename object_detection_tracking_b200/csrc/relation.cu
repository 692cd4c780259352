// relation.cu -- the relation module of the box head (add_relation_nn: relation_network nn.py:115-190 with
// geometric_encoding nn.py:273-298, group 16, geo_feat_dim 64), the parts that are not GEMMs on conv_tc_kernel.
//
// Per image b with n = count[b] proposals and h its [K][D] head rows:
//   relation_vt_kernel      V^T[c][j] = h[j][c] for j < n, 0 for n <= j < Kp: the B operand of the P.V layer
//   relation_attend_kernel  for every query row i < n and head g: the pairwise geometry -> geo_emb (4 -> 64, tanh) ->
//                           geo_conv (64 -> 16, ReLU) -> log(max(wg, 1e-6)), plus q_g(i).k_g(j) / sqrt(D / 16), then the
//                           softmax over j < n, written as P row i * 16 + g in the plane format; rows i >= n are zero
// query / key (one N = 2D layer), P.V (one layer of 16K rows per image) and output_linear (+ h) run on conv_tc_kernel.
//
// Everything is fp32 with the accurate tanhf / logf / expf, and every reduction has a fixed order that depends on n and
// the head geometry only: an image's P is the same whichever batch it runs in.
#include <math.h>

#include <vector>

#include "kernels.h"
#include "planes.cuh"

namespace b2 {
namespace {

constexpr int kThreads = 256;
constexpr int kTile = 32;   // V^T transpose tile
constexpr size_t kSmemBudget = 200 * 1024;

// geo weights as relation_upload_geo packs them: geo_emb W [4][64], b [64], geo_conv W [64][16], b [16]
constexpr int kEmbW = 0, kEmbB = kEmbW + 4 * kRelGeoDim, kConvW = kEmbB + kRelGeoDim, kConvB = kConvW + kRelGeoDim * kRelGroups;

size_t attend_smem(int rows, int Kp, int D) {
  return (static_cast<size_t>(rows) * kRelGroups * Kp + static_cast<size_t>(rows) * (D + 4) + kRelGeoWeights) * sizeof(float);
}

__global__ void __launch_bounds__(kTile * 8) relation_vt_kernel(const __half* __restrict__ h_hi, const __half* __restrict__ h_lo,
                                                               int D, int K, int Kp, const int* __restrict__ count, int b0,
                                                               __half* const* vt_hi, __half* const* vt_lo) {
  __shared__ __half t_hi[kTile][kTile + 2], t_lo[kTile][kTile + 2];
  const int b = b0 + blockIdx.z;
  const int n = min(max(count[b], 0), K);
  const int j0 = blockIdx.x * kTile, c0 = blockIdx.y * kTile;
  const __half zero = __float2half_rn(0.f);
  for (int r = threadIdx.y; r < kTile; r += blockDim.y) {   // rows j of h, columns c
    const int j = j0 + r, c = c0 + threadIdx.x;
    const size_t off = (static_cast<size_t>(b) * K + j) * D + c;
    const bool ok = j < n;
    t_hi[r][threadIdx.x] = ok ? h_hi[off] : zero;
    if (h_lo) t_lo[r][threadIdx.x] = ok ? h_lo[off] : zero;
  }
  __syncthreads();
  __half* oh = vt_hi[b];
  __half* ol = vt_lo ? vt_lo[b] : nullptr;
  for (int r = threadIdx.y; r < kTile; r += blockDim.y) {   // rows c of V^T, columns j
    const size_t off = static_cast<size_t>(c0 + r) * Kp + j0 + threadIdx.x;
    oh[off] = t_hi[threadIdx.x][r];
    if (ol) ol[off] = t_lo[threadIdx.x][r];
  }
}

__global__ void __launch_bounds__(kThreads) relation_attend_kernel(RelationParams p, int b0) {
  extern __shared__ float4 smem4[];
  float* s = reinterpret_cast<float*>(smem4);                       // [rows][16][Kp] logits, then exp
  const int rows = p.rows, D = p.D, Kp = p.Kp, K = p.K, qld = D + 4;
  float* q = s + static_cast<size_t>(rows) * kRelGroups * Kp;      // [rows][D + 4] query rows (padded: no bank conflicts)
  float* geo = q + static_cast<size_t>(rows) * qld;                // kRelGeoWeights
  const int b = b0 + blockIdx.y;
  const int n = min(max(p.count[b], 0), K);
  const int i0 = blockIdx.x * rows;
  const int ra = max(0, min(rows, n - i0));                        // valid query rows of this block
  const int dg = D / kRelGroups;
  const float scale = 1.0f / sqrtf(static_cast<float>(dg));
  for (int t = threadIdx.x; t < kRelGeoWeights; t += kThreads) geo[t] = p.geo[t];
  for (int t = threadIdx.x; t < ra * (D / 4); t += kThreads) {
    const int r = t / (D / 4), c = (t % (D / 4)) * 4;
    *reinterpret_cast<float4*>(q + r * qld + c) =
        __ldg(reinterpret_cast<const float4*>(p.qk + (static_cast<size_t>(b) * K + i0 + r) * p.ldqk + c));
  }
  __syncthreads();

  // pairs (r, j), r fastest: the threads of a warp share few key rows
  const float4* boxes = reinterpret_cast<const float4*>(p.boxes) + static_cast<size_t>(b) * K;
  for (int t = threadIdx.x; t < ra * n; t += kThreads) {
    const int r = t % ra, j = t / ra;
    const float4 bi = __ldg(boxes + i0 + r), bj = __ldg(boxes + j);
    // geometric_encoding (nn.py:273-298): centre offsets over the width of box i, both of them (dy too)
    const float wi = bi.z - bi.x, hi = bi.w - bi.y, wj = bj.z - bj.x, hj = bj.w - bj.y;
    const float cxi = 0.5f * (bi.x + bi.z), cyi = 0.5f * (bi.y + bi.w);
    const float cxj = 0.5f * (bj.x + bj.z), cyj = 0.5f * (bj.y + bj.w);
    const float d0 = logf(fmaxf(fabsf((cxi - cxj) / wi), 1e-3f));
    const float d1 = logf(fmaxf(fabsf((cyi - cyj) / wi), 1e-3f));
    const float d2 = logf(wi / wj);
    const float d3 = logf(hi / hj);
    float wg[kRelGroups];
#pragma unroll
    for (int g = 0; g < kRelGroups; ++g) wg[g] = geo[kConvB + g];
    for (int o = 0; o < kRelGeoDim; ++o) {
      float e = geo[kEmbB + o];
      e = fmaf(d0, geo[kEmbW + o], e);
      e = fmaf(d1, geo[kEmbW + kRelGeoDim + o], e);
      e = fmaf(d2, geo[kEmbW + 2 * kRelGeoDim + o], e);
      e = fmaf(d3, geo[kEmbW + 3 * kRelGeoDim + o], e);
      e = tanhf(e);
#pragma unroll
      for (int g = 0; g < kRelGroups; ++g) wg[g] = fmaf(e, geo[kConvW + o * kRelGroups + g], wg[g]);
    }
    const float* qr = q + r * qld;
    const float* kj = p.qk + (static_cast<size_t>(b) * K + j) * p.ldqk + D;
    float* sr = s + static_cast<size_t>(r) * kRelGroups * Kp + j;
#pragma unroll
    for (int g = 0; g < kRelGroups; ++g) {
      float dot = 0.f;
      for (int c = g * dg; c < (g + 1) * dg; c += 4) {
        const float4 a = *reinterpret_cast<const float4*>(qr + c);
        const float4 k4 = __ldg(reinterpret_cast<const float4*>(kj + c));
        dot = fmaf(a.x, k4.x, dot);
        dot = fmaf(a.y, k4.y, dot);
        dot = fmaf(a.z, k4.z, dot);
        dot = fmaf(a.w, k4.w, dot);
      }
      // ReLU then the 1e-6 clamp: max(relu(x), 1e-6) = max(x, 1e-6)
      sr[static_cast<size_t>(g) * Kp] = logf(fmaxf(wg[g], 1e-6f)) + dot * scale;
    }
  }
  __syncthreads();

  // softmax over j < n of every (r, g) row, one warp per row; rows i >= n (and the columns j >= n) are written as 0
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const int nr = min(rows, K - i0);
  for (int row = warp; row < nr * kRelGroups; row += kThreads / 32) {
    const int r = row / kRelGroups;
    const size_t prow = (static_cast<size_t>(b) * K + i0 + r) * kRelGroups + row % kRelGroups;
    __half* ph = p.p_hi + prow * Kp;
    __half* pl = p.p_lo ? p.p_lo + prow * Kp : nullptr;
    float* sr = s + static_cast<size_t>(row) * Kp;
    if (r >= ra) {
      for (int j = lane; j < Kp; j += 32) store1(ph, pl, j, 0.f);
      continue;
    }
    float m = -INFINITY;
    for (int j = lane; j < n; j += 32) m = fmaxf(m, sr[j]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    float sum = 0.f;
    for (int j = lane; j < n; j += 32) {
      const float e = expf(sr[j] - m);
      sr[j] = e;
      sum += e;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    __syncwarp();
    for (int j = lane; j < Kp; j += 32) store1(ph, pl, j, j < n ? sr[j] / sum : 0.f);
  }
}

}  // namespace

int relation_rows_per_block(int Kp, int D) {
  for (int rows = 8; rows > 1; rows >>= 1)
    if (attend_smem(rows, Kp, D) <= kSmemBudget) return rows;
  return 1;
}

int relation_attend_launch(const RelationParams& p, int b0, int n, cudaStream_t s) {
  if (n <= 0) return 0;
  B2_CHECK(p.D % 64 == 0 && p.Kp % 64 == 0 && p.Kp >= p.K && p.rows >= 1, "relation: bad geometry");
  const dim3 vt_grid(p.Kp / kTile, p.D / kTile, n);
  relation_vt_kernel<<<vt_grid, dim3(kTile, 8), 0, s>>>(p.h_hi, p.h_lo, p.D, p.K, p.Kp, p.count, b0, p.vt_hi, p.vt_lo);
  B2_CUDA(cudaGetLastError());
  const size_t smem = attend_smem(p.rows, p.Kp, p.D);
  B2_CHECK(smem <= kSmemBudget, "relation: query rows do not fit shared memory");
  B2_CUDA(cudaFuncSetAttribute(relation_attend_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                               static_cast<int>(kSmemBudget)));
  const dim3 grid((p.K + p.rows - 1) / p.rows, n);
  relation_attend_kernel<<<grid, kThreads, smem, s>>>(p, b0);
  B2_CUDA(cudaGetLastError());
  return 0;
}

void relation_pack_qk(const float* wq, const float* wk, int D, std::vector<float>& packed) {
  packed.assign(static_cast<size_t>(2 * D) * D, 0.f);
  for (int k = 0; k < D; ++k)
    for (int o = 0; o < D; ++o) {
      packed[static_cast<size_t>(o) * D + k] = wq[static_cast<size_t>(k) * D + o];
      packed[static_cast<size_t>(D + o) * D + k] = wk[static_cast<size_t>(k) * D + o];
    }
}

int relation_upload_geo(const float* emb_w, const float* emb_b, const float* conv_w, const float* conv_b, float* dst,
                        cudaStream_t s) {
  std::vector<float> g(kRelGeoWeights);
  const struct { const float* src; int off, n; } parts[] = {{emb_w, kEmbW, 4 * kRelGeoDim}, {emb_b, kEmbB, kRelGeoDim},
                                                            {conv_w, kConvW, kRelGeoDim * kRelGroups},
                                                            {conv_b, kConvB, kRelGroups}};
  for (const auto& e : parts)
    for (int i = 0; i < e.n; ++i) {
      B2_CHECK(std::isfinite(e.src[i]), "relation module: geo_emb / geo_conv weights not finite");
      g[e.off + i] = e.src[i];
    }
  B2_CUDA(cudaMemcpyAsync(dst, g.data(), g.size() * sizeof(float), cudaMemcpyHostToDevice, s));
  B2_CUDA(cudaStreamSynchronize(s));
  return 0;
}

}  // namespace b2
