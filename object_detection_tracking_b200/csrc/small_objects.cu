// small_objects.cu -- the small-object branch of the single-image graph (use_small_object_head, models.py:590-692,
// 845-897), the parts that are not GEMMs on conv_tc_kernel or the head's selection kernels.
//
//   so_select_kernel   per proposal: the selected classes' probabilities and unclipped decoded boxes (decode_box, the
//                      arithmetic of head_decode_kernel), for the per-class NMS that head.cu's class_nms_kernel runs
//   so_gather_kernel   the NMS selections -> the branch's box rows in selection order; K = the common count of the small
//                      classes, or 0 with status 1 when they differ (the reference's tf.map_fn cannot stack them)
//   so_vt_kernel /     person_object_relation (nn.py:194-270): V^T of the person rows, and the pair geometry
//   so_attend_kernel   (geometric_encoding_pair nn.py:301-332: offsets over the person box's width) -> geo_emb / geo_conv
//                      -> log(max(wg, 1e-6)) + q_g . k_g / sqrt(D / 16) -> softmax over the person rows -> P
//   so_finish_kernel   the [K][C + 1] logits rebuilt from the per-class [.., 2] logits and the rows' clipped boxes
//                      (models.py:671-681, 870-877), for head.cu's selection with num_class = C + 1
// Everything is fp32 with the accurate logf / expf / tanhf and IEEE division, with fixed reduction orders.
#include <math.h>

#include "devutil.cuh"
#include "kernels.h"
#include "planes.cuh"

namespace b2 {
namespace {

constexpr int kThreads = 256;
constexpr int kTile = 32;
constexpr size_t kSmemBudget = 200 * 1024;
// geo weights as relation_upload_geo packs them: geo_emb W [4][64], b [64], geo_conv W [64][16], b [16]
constexpr int kEmbW = 0, kEmbB = kEmbW + 4 * kRelGeoDim, kConvW = kEmbB + kRelGeoDim, kConvB = kConvW + kRelGeoDim * kRelGroups;

__global__ void so_select_kernel(const __grid_constant__ SoParams p) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= min(p.roi_count[0], p.rois)) return;
  const int ns = p.C + (p.Tp > 0 ? 1 : 0);
  const float4 roi = reinterpret_cast<const float4*>(p.roi_boxes)[r];
  const float* lg = p.logits + static_cast<size_t>(r) * p.ld + p.num_class;
  float4* ob = reinterpret_cast<float4*>(p.sel_boxes) + static_cast<size_t>(r) * (p.C + 1);
  float* op = p.sel_probs + static_cast<size_t>(r) * (p.C + 2);
  for (int s = 0; s < ns; ++s) {
    const int id = p.ids[s];
    op[s + 1] = p.probs[static_cast<size_t>(r) * p.num_class + id];
    ob[s] = decode_box(lg + id * 4, p.reg_w, p.decode_clip, roi);
  }
}

__global__ void so_gather_kernel(const __grid_constant__ SoParams p) {
  __shared__ int s_k;
  const int C = p.C, R = p.R;
  if (threadIdx.x == 0) {
    const int n0 = p.sel_count[0];
    bool eq = true;
    for (int c = 1; c < C; ++c) eq = eq && p.sel_count[c] == n0;
    s_k = eq ? n0 : 0;
    *p.k = s_k;
    *p.status = eq ? 0 : 1;
  }
  __syncthreads();
  const int K = s_k, np = p.Tp > 0 ? p.sel_count[C] : 0;
  const float4* sb = reinterpret_cast<const float4*>(p.sel_boxes);
  float4* rb = reinterpret_cast<float4*>(p.rows_boxes);
  for (int t = threadIdx.x; t < C * R + p.Tp; t += blockDim.x) {
    float4 b = make_float4(0.f, 0.f, 0.f, 0.f);
    if (t < C * R) {
      const int c = t / R, i = t - c * R;
      if (i < K) b = sb[static_cast<size_t>(p.keep[t]) * (C + 1) + c];
    } else if (t - C * R < np) {
      b = sb[static_cast<size_t>(p.person_keep[t - C * R]) * (C + 1) + C];
    }
    rb[t] = b;
  }
  for (int c = threadIdx.x; c <= C; c += blockDim.x) p.row_count[c] = c < C ? K : np;
}

__global__ void so_finish_kernel(const __grid_constant__ SoParams p) {
  const int C = p.C, R = p.R;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= R * C) return;
  const int k = t / C, c = t - k * C;
  const bool live = k < *p.k;
  float* fl = p.fin_logits + static_cast<size_t>(k) * (C + 1);
  float4 b = make_float4(0.f, 0.f, 0.f, 0.f);
  float v = 0.f;
  if (live) {
    v = p.cls_logits[(static_cast<size_t>(c) * R + k) * p.ldl + 2 * c + 1];
    b = clip_box(reinterpret_cast<const float4*>(p.rows_boxes)[static_cast<size_t>(c) * R + k], p.img_w, p.img_h);
  }
  fl[c + 1] = v;
  reinterpret_cast<float4*>(p.fin_boxes)[static_cast<size_t>(k) * C + c] = b;
  if (c == 0) {   // column 0: the mean over the classes of the background logits (never selected, models.py:677-678)
    float s = 0.f;
    if (live)
      for (int i = 0; i < C; ++i) s = __fadd_rn(s, p.cls_logits[(static_cast<size_t>(i) * R + k) * p.ldl + 2 * i]);
    fl[0] = __fdiv_rn(s, static_cast<float>(C));
  }
}

__global__ void __launch_bounds__(kTile * 8) so_vt_kernel(const __grid_constant__ SoAttendParams p) {
  __shared__ __half t_hi[kTile][kTile + 2], t_lo[kTile][kTile + 2];
  const int n = min(max(*p.nref, 0), p.Tp);
  const int j0 = blockIdx.x * kTile, c0 = blockIdx.y * kTile;
  const __half zero = __float2half_rn(0.f);
  for (int r = threadIdx.y; r < kTile; r += blockDim.y) {   // rows j of the value, columns c
    const int j = j0 + r, c = c0 + threadIdx.x;
    const size_t off = static_cast<size_t>(j) * p.D + c;
    const bool ok = j < n;
    t_hi[r][threadIdx.x] = ok ? p.v_hi[off] : zero;
    if (p.v_lo) t_lo[r][threadIdx.x] = ok ? p.v_lo[off] : zero;
  }
  __syncthreads();
  for (int r = threadIdx.y; r < kTile; r += blockDim.y) {   // rows c of V^T, columns j
    const size_t off = static_cast<size_t>(c0 + r) * p.Tpp + j0 + threadIdx.x;
    p.vt_hi[off] = t_hi[threadIdx.x][r];
    if (p.vt_lo) p.vt_lo[off] = t_lo[threadIdx.x][r];
  }
}

// grid (query row groups, C): block (x, c) handles query rows x * rows .. of class block c
__global__ void __launch_bounds__(kThreads) so_attend_kernel(const __grid_constant__ SoAttendParams p) {
  extern __shared__ float4 smem4[];
  float* s = reinterpret_cast<float*>(smem4);                       // [rows][16][Tpp] logits, then exp
  const int rows = p.rows, D = p.D, Tpp = p.Tpp, qld = D + 4;
  float* q = s + static_cast<size_t>(rows) * kRelGroups * Tpp;     // [rows][D + 4] query rows
  float* geo = q + static_cast<size_t>(rows) * qld;                // kRelGeoWeights
  const int c = blockIdx.y;
  const int kq = min(max(*p.kq, 0), p.Rq), n = min(max(*p.nref, 0), p.Tp);
  const int i0 = blockIdx.x * rows;
  const int ra = n > 0 ? max(0, min(rows, kq - i0)) : 0;           // query rows of this block with a softmax
  const size_t q0 = static_cast<size_t>(c) * p.Rq + i0;            // first query row of the block
  const size_t k0 = static_cast<size_t>(p.C) * p.Rq;               // first key row
  const int dg = D / kRelGroups;
  const float scale = 1.0f / sqrtf(static_cast<float>(dg));
  for (int t = threadIdx.x; t < kRelGeoWeights; t += kThreads) geo[t] = p.geo[t];
  for (int t = threadIdx.x; t < ra * (D / 4); t += kThreads) {
    const int r = t / (D / 4), cc = (t % (D / 4)) * 4;
    *reinterpret_cast<float4*>(q + r * qld + cc) =
        __ldg(reinterpret_cast<const float4*>(p.qk + (q0 + r) * p.ldqk + cc));
  }
  __syncthreads();

  const float4* boxes = reinterpret_cast<const float4*>(p.boxes);
  for (int t = threadIdx.x; t < ra * n; t += kThreads) {
    const int r = t % ra, j = t / ra;
    const float4 bi = __ldg(boxes + q0 + r), bj = __ldg(boxes + k0 + j);
    // geometric_encoding_pair (nn.py:301-332): both centre offsets over the width of the key (person) box j
    const float wi = bi.z - bi.x, hi = bi.w - bi.y, wj = bj.z - bj.x, hj = bj.w - bj.y;
    const float cxi = 0.5f * (bi.x + bi.z), cyi = 0.5f * (bi.y + bi.w);
    const float cxj = 0.5f * (bj.x + bj.z), cyj = 0.5f * (bj.y + bj.w);
    const float d0 = logf(fmaxf(fabsf((cxi - cxj) / wj), 1e-3f));
    const float d1 = logf(fmaxf(fabsf((cyi - cyj) / wj), 1e-3f));
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
    const float* kj = p.qk + (k0 + j) * p.ldqk + D;
    float* sr = s + static_cast<size_t>(r) * kRelGroups * Tpp + j;
#pragma unroll
    for (int g = 0; g < kRelGroups; ++g) {
      float dot = 0.f;
      for (int cc = g * dg; cc < (g + 1) * dg; cc += 4) {
        const float4 a = *reinterpret_cast<const float4*>(qr + cc);
        const float4 k4 = __ldg(reinterpret_cast<const float4*>(kj + cc));
        dot = fmaf(a.x, k4.x, dot);
        dot = fmaf(a.y, k4.y, dot);
        dot = fmaf(a.z, k4.z, dot);
        dot = fmaf(a.w, k4.w, dot);
      }
      // ReLU then the 1e-6 clamp: max(relu(x), 1e-6) = max(x, 1e-6)
      sr[static_cast<size_t>(g) * Tpp] = logf(fmaxf(wg[g], 1e-6f)) + dot * scale;
    }
  }
  __syncthreads();

  // softmax over j < n of every (r, g) row, one warp per row; the other rows and columns are written as 0
  const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
  const int nr = min(rows, p.Rq - i0);
  for (int row = warp; row < nr * kRelGroups; row += kThreads / 32) {
    const int r = row / kRelGroups;
    const size_t prow = (q0 + r) * kRelGroups + row % kRelGroups;
    __half* ph = p.p_hi + prow * Tpp;
    __half* pl = p.p_lo ? p.p_lo + prow * Tpp : nullptr;
    float* sr = s + static_cast<size_t>(row) * Tpp;
    if (r >= ra) {
      for (int j = lane; j < Tpp; j += 32) store1(ph, pl, j, 0.f);
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
    for (int j = lane; j < Tpp; j += 32) store1(ph, pl, j, j < n ? sr[j] / sum : 0.f);
  }
}

size_t attend_smem(int rows, int Tpp, int D) {
  return (static_cast<size_t>(rows) * kRelGroups * Tpp + static_cast<size_t>(rows) * (D + 4) + kRelGeoWeights) * sizeof(float);
}

}  // namespace

int so_select_launch(const SoParams& p, cudaStream_t s) {
  B2_CHECK(p.C >= 1 && p.C <= 80 && p.rois >= 1, "small objects: bad geometry");
  so_select_kernel<<<(p.rois + 127) / 128, 128, 0, s>>>(p);
  B2_CUDA(cudaGetLastError());
  return 0;
}

int so_gather_launch(const SoParams& p, cudaStream_t s) {
  so_gather_kernel<<<1, 1024, 0, s>>>(p);
  B2_CUDA(cudaGetLastError());
  return 0;
}

int so_finish_launch(const SoParams& p, cudaStream_t s) {
  const int n = p.R * p.C;
  so_finish_kernel<<<(n + 255) / 256, 256, 0, s>>>(p);
  B2_CUDA(cudaGetLastError());
  return 0;
}

int so_attend_launch(const SoAttendParams& p, cudaStream_t s) {
  B2_CHECK(p.D % 64 == 0 && p.Tpp % 64 == 0 && p.Tpp >= p.Tp && p.Tp >= 1 && p.Rq >= 1 && p.C >= 1 && p.rows >= 1,
           "person_object_relation: bad geometry");
  so_vt_kernel<<<dim3(p.Tpp / kTile, p.D / kTile), dim3(kTile, 8), 0, s>>>(p);
  B2_CUDA(cudaGetLastError());
  const size_t smem = attend_smem(p.rows, p.Tpp, p.D);
  B2_CHECK(smem <= kSmemBudget, "person_object_relation: query rows do not fit shared memory");
  B2_CUDA(cudaFuncSetAttribute(so_attend_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kSmemBudget)));
  so_attend_kernel<<<dim3((p.Rq + p.rows - 1) / p.rows, p.C), kThreads, smem, s>>>(p);
  B2_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace b2
