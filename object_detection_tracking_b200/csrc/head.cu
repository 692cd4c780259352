// Detection post-processing on device: softmax + per-class box decode + clip, [use_bg_score's background filter,]
// per-class NMS, global top-k.  Three (four) small kernels, no host round trip.
//
// Reference ops replaced: inference decode (models.py:830-843: decode_bbox_target with
// fastrcnn_bbox_reg_weights, clip_boxes, tf.nn.softmax), fastrcnn_predictions (models.py:1258-1304)
// with nms_return_masks (models.py:1202-1223: prob > thresh, tf.image.non_max_suppression per class under
// tf.map_fn) and the final tf.nn.top_k over the surviving (class, box) pairs.
#include "common.h"
#include "devutil.cuh"
#include "kernels.h"

namespace b2 {
namespace {

// one thread per ROI: softmax over classes, decode the (num_class-1) class boxes
__global__ void head_decode_kernel(const __grid_constant__ HeadPostParams p) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  const int total = p.B * p.rois_per_image;
  if (r >= total) return;
  const int nc = p.num_class;
  const float* lg = p.logits + static_cast<size_t>(r) * p.ld;
  float mx = lg[0];
  for (int c = 1; c < nc; ++c) mx = fmaxf(mx, lg[c]);
  float sum = 0.f;
  float* pr = p.probs + static_cast<size_t>(r) * nc;
  for (int c = 0; c < nc; ++c) {
    const float e = expf(__fsub_rn(lg[c], mx));
    pr[c] = e;
    sum = __fadd_rn(sum, e);
  }
  for (int c = 0; c < nc; ++c) pr[c] = __fdiv_rn(pr[c], sum);
  const float4 roi = reinterpret_cast<const float4*>(p.rois)[r];
  float4* ob = reinterpret_cast<float4*>(p.dec_boxes) + static_cast<size_t>(r) * (nc - 1);
  for (int c = 1; c < nc; ++c)
    ob[c - 1] = clip_box(decode_box(lg + nc + (p.class_agnostic ? 0 : c * 4), p.reg_w, p.decode_clip, roi), p.img_w, p.img_h);
}

// grid (B), one thread per ROI: use_bg_score's filter (models.py:1263-1270).  tf.argmax over the row's num_class values,
// restated as a scan that moves only on a strictly greater value: ties go to the lowest column, so a background value
// equal to the best class drops the row, and a NaN never wins (an all-NaN row has argmax 0).  Kept rows get their rank
// among the image's kept rows, in ROI order (tf.where + tf.gather); dropped rows and rows beyond the count get -1.
__global__ void __launch_bounds__(1024) bg_filter_kernel(const __grid_constant__ HeadPostParams p) {
  __shared__ int warp_kept[32];
  const int b = blockIdx.x, i = threadIdx.x, lane = i & 31, w = i >> 5;
  const int nc = p.num_class, R = p.rois_per_image;
  bool keep = false;
  if (i < R && i < p.roi_count[b]) {
    const float* pr = p.probs + (static_cast<size_t>(b) * R + i) * nc;
    float best = pr[0];
    int arg = 0;
    for (int c = 1; c < nc; ++c) {
      const float v = pr[c];
      if (v > best) {
        best = v;
        arg = c;
      }
    }
    keep = arg != 0;
  }
  const uint32_t bal = __ballot_sync(0xffffffffu, keep);
  if (lane == 0) warp_kept[w] = __popc(bal);
  __syncthreads();
  int rank = __popc(bal & ((1u << lane) - 1u));
  for (int k = 0; k < w; ++k) rank += warp_kept[k];
  if (i < R) p.bg_rank[static_cast<size_t>(b) * R + i] = keep ? rank : -1;
}

// grid (classes, B): per-class NMS over the ROIs of one image, classes c0, c0 + 1, ...
__global__ void __launch_bounds__(512) class_nms_kernel(const __grid_constant__ HeadPostParams p, int KP, int c0) {
  extern __shared__ __align__(16) uint8_t sm[];
  const int c = c0 + blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
  const int nc = p.num_class, R = p.rois_per_image;
  uint64_t* keys = reinterpret_cast<uint64_t*>(sm);          // [KP]
  float4* boxes = reinterpret_cast<float4*>(keys + KP);      // [KP]
  int* ridx = reinterpret_cast<int*>(boxes + KP);            // [KP]
  int* keep = ridx + KP;                                     // [KP]
  uint32_t* mask = reinterpret_cast<uint32_t*>(keep + KP);   // [R * ceil(R/32)]
  __shared__ int s_cnt, s_n;
  const int cnt = p.roi_count[b];
  if (tid == 0) s_n = 0;
  __syncthreads();
  for (int i = tid; i < KP; i += blockDim.x) {
    uint64_t k = ~0ull;
    if (i < cnt && (!p.bg_rank || p.bg_rank[static_cast<size_t>(b) * R + i] >= 0)) {
      const float pr = p.probs[(static_cast<size_t>(b) * R + i) * nc + c + 1];
      if (pr > p.score_thresh) {
        k = desc_key(pr, static_cast<uint32_t>(i));
        atomicAdd(&s_n, 1);
      }
    }
    keys[i] = k;
  }
  block_bitonic_sort(keys, KP);
  const int n = s_n;
  for (int j = tid; j < n; j += blockDim.x) {
    const int i = static_cast<int>(keys[j] & 0xffffffffu);
    ridx[j] = i;
    boxes[j] = reinterpret_cast<const float4*>(p.dec_boxes)[(static_cast<size_t>(b) * R + i) * (nc - 1) + c];
  }
  __syncthreads();
  const int kept = block_nms_sorted(boxes, n, p.nms_thr, p.max_per_class, mask, keep, &s_cnt);
  int* out = p.cls_keep + (static_cast<size_t>(b) * (nc - 1) + c) * p.max_per_class;
  for (int j = tid; j < kept; j += blockDim.x) out[j] = ridx[keep[j]];
  if (tid == 0) p.cls_count[b * (nc - 1) + c] = kept;
}

// grid (B): top-k over all surviving (class, box) pairs; ties -> (class, box) ascending, the order of
// tf.where(masks) on the [num_class-1, K] mask (models.py:1286-1296).
__global__ void __launch_bounds__(1024) final_topk_kernel(const __grid_constant__ HeadPostParams p, int KP2) {
  extern __shared__ __align__(16) uint8_t sm[];
  uint64_t* keys = reinterpret_cast<uint64_t*>(sm);
  const int b = blockIdx.x, tid = threadIdx.x;
  const int nc1 = p.num_class - 1, R = p.rois_per_image;
  __shared__ int s_total;
  if (tid == 0) s_total = 0;
  for (int i = tid; i < KP2; i += blockDim.x) keys[i] = ~0ull;
  __syncthreads();
  for (int c = 0; c < nc1; ++c) {
    const int cnt = p.cls_count[b * nc1 + c];
    const int* kp = p.cls_keep + (static_cast<size_t>(b) * nc1 + c) * p.max_per_class;
    for (int j = tid; j < cnt; j += blockDim.x) {
      const int i = kp[j];
      const float pr = p.probs[(static_cast<size_t>(b) * R + i) * p.num_class + c + 1];
      const int slot = atomicAdd(&s_total, 1);
      keys[slot] = desc_key(pr, static_cast<uint32_t>(c * R + i));
    }
  }
  block_bitonic_sort(keys, KP2);
  const int K = min(s_total, p.max_total);
  for (int j = tid; j < p.max_total; j += blockDim.x) {
    const size_t o = static_cast<size_t>(b) * p.max_total + j;
    if (j < K) {
      const uint32_t ci = static_cast<uint32_t>(keys[j] & 0xffffffffu);
      const int c = ci / R, i = ci - c * R;
      // with the background filter the box is ROI j's, j = i's rank among the kept rows: the reference gathers the
      // unfiltered boxes at the filtered index (models.py:925-930).  The key (c, i) sorts as (c, j) would
      const int row = p.bg_rank ? p.bg_rank[static_cast<size_t>(b) * R + i] : i;
      reinterpret_cast<float4*>(p.final_boxes)[o] =
          reinterpret_cast<const float4*>(p.dec_boxes)[(static_cast<size_t>(b) * R + row) * nc1 + c];
      p.final_probs[o] = p.probs[(static_cast<size_t>(b) * R + i) * p.num_class + c + 1];
      p.final_labels[o] = c + 1;
    } else {
      reinterpret_cast<float4*>(p.final_boxes)[o] = make_float4(0, 0, 0, 0);
      p.final_probs[o] = 0.f;
      p.final_labels[o] = 0;
    }
  }
  if (tid == 0) p.final_count[b] = K;
}

int next_pow2(int v) {
  int p = 1;
  while (p < v) p <<= 1;
  return p;
}

}  // namespace

int class_nms_launch(const HeadPostParams& p, int c0, int n, cudaStream_t s) {
  const int R = p.rois_per_image;
  B2_CHECK(R <= 1024, "head: at most 1024 ROIs per image");
  B2_CHECK(c0 >= 0 && n >= 1 && c0 + n <= p.num_class - 1, "head: class range outside the classes");
  // at least 2 keys, so that the float4 boxes after the 8-byte keys start 16-byte aligned (one ROI per image would put
  // them at 8)
  const int KP = next_pow2(R) < 2 ? 2 : next_pow2(R);
  const size_t smem1 = static_cast<size_t>(KP) * (8 + 16 + 4 + 4) + static_cast<size_t>(R) * ((R + 31) / 32) * 4;
  static bool attr_set = false;
  if (!attr_set) {
    B2_CUDA(cudaFuncSetAttribute(class_nms_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attr_set = true;
  }
  B2_CHECK(smem1 <= 200 * 1024, "head: too many ROIs for shared memory");
  class_nms_kernel<<<dim3(n, p.B), 512, smem1, s>>>(p, KP, c0);
  B2_CUDA(cudaGetLastError());
  return 0;
}

int head_select_launch(const HeadPostParams& p, cudaStream_t s) {
  const int nc1 = p.num_class - 1;
  // at least 2 keys here too: the sort's first __syncthreads is what publishes the keys and s_total, and a sort of one key
  // (one class, e.g. a single partial class, with max_per_class 1) has none
  const int KP2 = next_pow2(nc1 * p.max_per_class) < 2 ? 2 : next_pow2(nc1 * p.max_per_class);
  const size_t smem2 = static_cast<size_t>(KP2) * 8;
  static bool attr_set = false;
  if (!attr_set) {
    B2_CUDA(cudaFuncSetAttribute(final_topk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attr_set = true;
  }
  B2_CHECK(smem2 <= 200 * 1024, "head: too many classes for shared memory");
  if (p.bg_rank) {
    B2_CHECK(p.rois_per_image <= 1024, "head: at most 1024 ROIs per image");
    bg_filter_kernel<<<p.B, (p.rois_per_image + 31) / 32 * 32, 0, s>>>(p);
    B2_CUDA(cudaGetLastError());
  }
  if (class_nms_launch(p, 0, nc1, s)) return -1;
  final_topk_kernel<<<p.B, 1024, smem2, s>>>(p, KP2);
  B2_CUDA(cudaGetLastError());
  return 0;
}

int head_post_launch(const HeadPostParams& p, cudaStream_t s) {
  B2_CHECK(p.rois_per_image <= 1024, "head: at most 1024 ROIs per image");
  const int total = p.B * p.rois_per_image;
  head_decode_kernel<<<(total + 127) / 128, 128, 0, s>>>(p);
  B2_CUDA(cudaGetLastError());
  return head_select_launch(p, s);
}

}  // namespace b2
