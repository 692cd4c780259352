// Non-GEMM kernels of the EfficientDet feature network (BiFPN), heads and post-processing.  The pointwise
// halves of every separable conv and the 1x1 resampling convs run on the wgmma implicit-GEMM kernel.
//
// Reference ops replaced: resample_feature_map (efficientdet_arch.py:105-200: max_pooling2d SAME / nearest
// upsampling), the node combine + swish of build_bifpn_layer (:594-682), the depthwise half of
// tf.layers.separable_conv2d (:241,651), add_metric_fn_inputs' global top-k (efficientdet_wrapper.py:367-474),
// _generate_detections_tf (anchors.py:399-487: sigmoid, decode_box_outputs_tf, class-agnostic
// non_max_suppression_with_scores).
#include "common.h"
#include "devutil.cuh"
#include "kernels.h"
#include "planes.cuh"

namespace b2 {
namespace {

// One BiFPN node input resampled on the fly to the node resolution (Ho x Wo):
//   mode 0: same size; mode 1: 3x3 stride-2 max-pool with TF SAME padding from a 2x finer map;
//   mode 2: nearest-neighbour 2x upsampling from a coarser map.
__device__ __forceinline__ void fetch_resampled(const BifpnInput& in, int b, int y, int x, int C, int cv,
                                                float (&v)[8]) {
  if (in.mode == 0) {
    load8(in.hi, in.lo, ((static_cast<size_t>(b) * in.H + y) * in.W + x) * C + cv * 8, v);
  } else if (in.mode == 2) {
    load8(in.hi, in.lo, ((static_cast<size_t>(b) * in.H + (y >> 1)) * in.W + (x >> 1)) * C + cv * 8, v);
  } else {
    // SAME padding for k=3, s=2: pad_total = max((out-1)*2 + 3 - in, 0), pad_before = pad_total / 2
    const int y0 = 2 * y - in.pad_t, x0 = 2 * x - in.pad_l;
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = -3.4e38f;
    for (int r = 0; r < 3; ++r) {
      const int iy = y0 + r;
      if (iy < 0 || iy >= in.H) continue;
      for (int s = 0; s < 3; ++s) {
        const int ix = x0 + s;
        if (ix < 0 || ix >= in.W) continue;
        float t[8];
        load8(in.hi, in.lo, ((static_cast<size_t>(b) * in.H + iy) * in.W + ix) * C + cv * 8, t);
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = fmaxf(v[j], t[j]);
      }
    }
  }
}

// node = act(sum_i w_i * resample_i(x_i)); act = swish (x * sigmoid(x)) or identity (plain resampling)
__global__ void bifpn_combine_kernel(const __grid_constant__ BifpnCombineParams p) {
  const int cvec = p.C / 8;
  const size_t total = static_cast<size_t>(p.B) * p.Ho * p.Wo * cvec;
  for (size_t idx = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int cv = static_cast<int>(idx % cvec);
    const size_t pix = idx / cvec;
    const int b = static_cast<int>(pix / (static_cast<size_t>(p.Ho) * p.Wo));
    const int rem = static_cast<int>(pix % (static_cast<size_t>(p.Ho) * p.Wo));
    const int y = rem / p.Wo, x = rem % p.Wo;
    float acc[8];
    for (int i = 0; i < p.n_in; ++i) {
      float v[8];
      fetch_resampled(p.in[i], b, y, x, p.C, cv, v);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float t = p.weighted ? __fdiv_rn(__fmul_rn(v[j], p.in[i].weight), p.denom) : v[j];
        acc[j] = i == 0 ? t : __fadd_rn(acc[j], t);
      }
    }
    if (p.swish) {
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] = __fmul_rn(acc[j], 1.f / (1.f + expf(-acc[j])));
    }
    store8(p.out_hi, p.out_lo, pix * p.C + cv * 8, acc);
  }
}

// ---- global top-k over all class logits: multi-block radix select on order-preserving keys ----------
// Every kernel below works on image blockIdx.y (blockIdx.z for the NMS mask) and touches only that image's slices.
constexpr unsigned kTopkMaxBlocks = 132 * 8;

__device__ __forceinline__ int level_of(const EffdetPostParams& p, unsigned long long i) {
  int l = 0;
  while (l + 1 < p.n_levels && i >= p.level_off[l + 1]) ++l;
  return l;
}

__device__ __forceinline__ float logit_at(const EffdetPostParams& p, int b, unsigned long long i) {
  const int l = level_of(p, i);
  const unsigned long long r = i - p.level_off[l];
  const unsigned int per_pos = static_cast<unsigned int>(p.anchors * p.num_classes);
  const unsigned long long pos = r / per_pos;
  const unsigned int k = static_cast<unsigned int>(r - pos * per_pos);
  return __ldg(p.logits[l] + b * p.logit_bstride[l] + pos * p.ld[l] + k);
}

__device__ __forceinline__ uint32_t* state_of(const EffdetPostParams& p, int b) { return p.state + 8 * b; }
__device__ __forceinline__ unsigned int* hist_of(const EffdetPostParams& p, int b) { return p.hist + 256 * b; }
__device__ __forceinline__ size_t kslice(const EffdetPostParams& p, int b) { return static_cast<size_t>(b) * p.k; }

__global__ void topk_hist_kernel(const __grid_constant__ EffdetPostParams p, int pass) {
  __shared__ unsigned int h[256];
  const int b = blockIdx.y;
  for (int i = threadIdx.x; i < 256; i += blockDim.x) h[i] = 0;
  __syncthreads();
  const int shift = 24 - 8 * pass;
  const uint32_t* state = state_of(p, b);
  const uint32_t prefix = state[0], pmask = state[1];
  for (unsigned long long i = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x; i < p.total;
       i += static_cast<unsigned long long>(gridDim.x) * blockDim.x) {
    const uint32_t key = float_key(logit_at(p, b, i));
    if ((key & pmask) == prefix) atomicAdd(&h[(key >> shift) & 255], 1u);
  }
  __syncthreads();
  unsigned int* hist = hist_of(p, b);
  for (int i = threadIdx.x; i < 256; i += blockDim.x)
    if (h[i]) atomicAdd(&hist[i], h[i]);
}

__global__ void topk_pick_kernel(const __grid_constant__ EffdetPostParams p, int pass) {
  uint32_t* state = state_of(p, blockIdx.y);
  unsigned int* hist = hist_of(p, blockIdx.y);
  if (threadIdx.x == 0) {
    const int shift = 24 - 8 * pass;
    unsigned int need = state[2], cum = 0;
    int bsel = 0;
    for (int b = 255; b >= 0; --b) {
      if (cum + hist[b] >= need) { bsel = b; break; }
      cum += hist[b];
    }
    state[2] = need - cum;
    state[0] |= static_cast<uint32_t>(bsel) << shift;
    state[1] |= 255u << shift;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 256; i += blockDim.x) hist[i] = 0;
}

// collect every key > kth (any order) and count the ties == kth per block (blocks own contiguous index ranges)
__global__ void topk_collect_kernel(const __grid_constant__ EffdetPostParams p, unsigned long long chunk) {
  __shared__ unsigned int s_ties;
  if (threadIdx.x == 0) s_ties = 0;
  __syncthreads();
  const int b = blockIdx.y;
  uint32_t* state = state_of(p, b);
  unsigned long long* cand = p.cand + kslice(p, b);
  const uint32_t kth = state[0];
  const unsigned long long lo = blockIdx.x * chunk;
  const unsigned long long hi = lo + chunk < p.total ? lo + chunk : p.total;
  unsigned int mine = 0;
  for (unsigned long long i = lo + threadIdx.x; i < hi; i += blockDim.x) {
    const float v = logit_at(p, b, i);
    const uint32_t key = float_key(v);
    if (key > kth) {
      const unsigned int slot = atomicAdd(&state[3], 1u);
      if (slot < static_cast<unsigned int>(p.k)) cand[slot] = desc_key(v, static_cast<uint32_t>(i));
    } else if (key == kth) {
      ++mine;
    }
  }
  if (mine) atomicAdd(&s_ties, mine);
  __syncthreads();
  if (threadIdx.x == 0) p.tie_cnt[static_cast<size_t>(b) * kTopkMaxBlocks + blockIdx.x] = s_ties;
}

// exclusive prefix of the per-block tie counts (one block per image; <= a few thousand entries)
__global__ void topk_tie_scan_kernel(const __grid_constant__ EffdetPostParams p, int nblocks) {
  if (threadIdx.x == 0) {
    const size_t o = static_cast<size_t>(blockIdx.y) * kTopkMaxBlocks;
    unsigned int run = 0;
    for (int b = 0; b < nblocks; ++b) {
      const unsigned int c = p.tie_cnt[o + b];
      p.tie_off[o + b] = run;
      run += c;
    }
    state_of(p, blockIdx.y)[4] = run;
  }
}

// tf.nn.top_k keeps the lowest flat indices among equal values: write the first `need` ties in index order
__global__ void __launch_bounds__(256) topk_tie_write_kernel(const __grid_constant__ EffdetPostParams p, unsigned long long chunk) {
  const int img = blockIdx.y;
  const uint32_t* state = state_of(p, img);
  const size_t o = static_cast<size_t>(img) * kTopkMaxBlocks + blockIdx.x;
  unsigned long long* ties = p.ties + kslice(p, img);
  const unsigned int need = state[2];
  unsigned int base = p.tie_off[o];
  if (p.tie_cnt[o] == 0 || base >= need) return;
  __shared__ unsigned int warp_cnt[8];
  const uint32_t kth = state[0];
  const unsigned long long lo = blockIdx.x * chunk;
  const unsigned long long hi = lo + chunk < p.total ? lo + chunk : p.total;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (unsigned long long t0 = lo; t0 < hi && base < need; t0 += blockDim.x) {
    const unsigned long long i = t0 + threadIdx.x;
    float v = 0.f;
    bool tie = false;
    if (i < hi) {
      v = logit_at(p, img, i);
      tie = float_key(v) == kth;
    }
    const unsigned int bal = __ballot_sync(0xffffffffu, tie);
    if (lane == 0) warp_cnt[wid] = __popc(bal);
    __syncthreads();
    unsigned int before = 0, tile = 0;
#pragma unroll
    for (int w = 0; w < 8; ++w) {
      const unsigned int c = warp_cnt[w];
      if (w < wid) before += c;
      tile += c;
    }
    if (tie) {
      const unsigned int rank = base + before + __popc(bal & ((1u << lane) - 1u));
      if (rank < need) ties[rank] = desc_key(v, static_cast<uint32_t>(i));
    }
    base += tile;
    __syncthreads();
  }
}

// one block per image: (selected U lowest-index ties) sorted by (logit desc, index asc) = tf.nn.top_k order; then
// sigmoid + anchor decode per candidate
__global__ void __launch_bounds__(1024, 1) det_prepare_kernel(const __grid_constant__ EffdetPostParams p, int KP) {
  extern __shared__ __align__(16) uint8_t sm[];
  uint64_t* keys = reinterpret_cast<uint64_t*>(sm);     // [KP]
  const int tid = threadIdx.x, img = blockIdx.y;
  uint32_t* state = state_of(p, img);
  const size_t ks = kslice(p, img);
  const unsigned long long* cand = p.cand + ks;
  const unsigned long long* ties = p.ties + ks;
  float4* cand_box = p.cand_box + ks;
  float* cand_score = p.cand_score + ks;
  int* cand_cls = p.cand_cls + ks;
  int* cand_lvl = p.cand_lvl + ks;
  const int n_gt = min(static_cast<int>(state[3]), p.k);
  const int take = min(min(static_cast<int>(state[2]), static_cast<int>(state[4])), p.k - n_gt);
  const int K = n_gt + take;
  for (int i = tid; i < KP; i += blockDim.x) keys[i] = i < n_gt ? cand[i] : (i < K ? ties[i - n_gt] : ~0ull);
  block_bitonic_sort(keys, KP);
  const unsigned int per_pos = static_cast<unsigned int>(p.anchors * p.num_classes);
  for (int j = tid; j < K; j += blockDim.x) {
    const unsigned long long i = keys[j] & 0xffffffffull;
    const int l = level_of(p, i);
    const unsigned long long r = i - p.level_off[l];
    const unsigned long long pos = r / per_pos;
    const int kk = static_cast<int>(r - pos * per_pos);
    const int a = kk / p.num_classes, cls = kk - a * p.num_classes;
    const int y = static_cast<int>(pos / p.w[l]), x = static_cast<int>(pos - static_cast<unsigned long long>(y) * p.w[l]);
    const float logit = __ldg(p.logits[l] + img * p.logit_bstride[l] + pos * p.ld[l] + kk);
    const float score = 1.f / (1.f + expf(-logit));
    // anchor (anchors.py:216-257), float64 grid like numpy, rounded once to float32
    const double yc_d = __dadd_rn(p.stride_y[l] / 2.0, __dmul_rn(static_cast<double>(y), p.stride_y[l]));
    const double xc_d = __dadd_rn(p.stride_x[l] / 2.0, __dmul_rn(static_cast<double>(x), p.stride_x[l]));
    const float ymin_a = __double2float_rn(__dsub_rn(yc_d, p.half_y[l][a]));
    const float xmin_a = __double2float_rn(__dsub_rn(xc_d, p.half_x[l][a]));
    const float ymax_a = __double2float_rn(__dadd_rn(yc_d, p.half_y[l][a]));
    const float xmax_a = __double2float_rn(__dadd_rn(xc_d, p.half_x[l][a]));
    // decode_box_outputs_tf (anchors.py:369-396)
    const float yca = __fdiv_rn(__fadd_rn(ymin_a, ymax_a), 2.f), xca = __fdiv_rn(__fadd_rn(xmin_a, xmax_a), 2.f);
    const float ha = __fsub_rn(ymax_a, ymin_a), wa = __fsub_rn(xmax_a, xmin_a);
    const float* t = p.boxes[l] + img * p.box_bstride[l] + pos * p.ldb[l] + a * 4;
    const float ty = __ldg(t), tx = __ldg(t + 1), th = __ldg(t + 2), tw = __ldg(t + 3);
    const float w = __fmul_rn(expf(tw), wa), h = __fmul_rn(expf(th), ha);
    const float yc = __fadd_rn(__fmul_rn(ty, ha), yca), xc = __fadd_rn(__fmul_rn(tx, wa), xca);
    cand_box[j] = make_float4(__fsub_rn(yc, __fdiv_rn(h, 2.f)), __fsub_rn(xc, __fdiv_rn(w, 2.f)),
                              __fadd_rn(yc, __fdiv_rn(h, 2.f)), __fadd_rn(xc, __fdiv_rn(w, 2.f)));
    cand_score[j] = score;
    cand_cls[j] = cls + 1;
    cand_lvl[j] = l + p.min_level;
  }
  if (tid == 0) state[5] = static_cast<uint32_t>(K);
}

// 64x64 tiles of the suppression bit matrix: mask[i][w] bit j = IoU(i, 64w + j) > thr, only j > i; image blockIdx.z
// (boxes [B][k], state [B][8], mask [B][k][words])
__global__ void nms_mask_kernel(const float4* __restrict__ boxes, const uint32_t* __restrict__ state, float thr, int k,
                                int words, unsigned long long* __restrict__ mask) {
  boxes += static_cast<size_t>(blockIdx.z) * k;
  state += 8 * blockIdx.z;
  mask += static_cast<size_t>(blockIdx.z) * k * words;
  const int n = static_cast<int>(state[5]);
  const int row0 = blockIdx.y * 64, col0 = blockIdx.x * 64;
  if (row0 >= n || col0 >= n || col0 + 63 < row0) return;
  __shared__ float4 cb[64];
  if (col0 + threadIdx.x < n) cb[threadIdx.x] = boxes[col0 + threadIdx.x];
  __syncthreads();
  const int i = row0 + threadIdx.x;
  if (i < n) {
    const float4 bi = boxes[i];
    unsigned long long bits = 0;
    for (int jj = 0; jj < 64; ++jj) {
      const int j = col0 + jj;
      if (j > i && j < n && iou_tf(bi, cb[jj]) > thr) bits |= 1ull << jj;
    }
    mask[static_cast<size_t>(i) * words + blockIdx.x] = bits;
  }
}

// one warp per image: greedy scan in score order (non_max_suppression_with_scores, hard NMS, score threshold), stops at
// max_out.  Lane l owns removed-words l, l+32, l+64, l+96 (k <= 8192).
__global__ void __launch_bounds__(32, 1) nms_scan_kernel(const __grid_constant__ EffdetPostParams p, int words,
                                                        const float* __restrict__ scale_ptr) {
  const int lane = threadIdx.x, img = blockIdx.y;
  const float scale = __ldg(scale_ptr + img);
  const size_t ks = kslice(p, img), os = static_cast<size_t>(img) * p.max_out;
  const float4* cand_box = p.cand_box + ks;
  const float* cand_score = p.cand_score + ks;
  const int* cand_cls = p.cand_cls + ks;
  const int* cand_lvl = p.cand_lvl + ks;
  const unsigned long long* mask = p.mask + ks * words;
  float4* out_boxes = p.out_boxes + os;
  float* out_scores = p.out_scores + os;
  int* out_classes = p.out_classes + os;
  int* out_levels = p.out_levels + os;
  const int n = static_cast<int>(state_of(p, img)[5]);
  unsigned long long rem[4] = {0ull, 0ull, 0ull, 0ull};
  int kept = 0;
  bool done = false;
  for (int base = 0; base < n && !done; base += 32) {
    const float sc = base + lane < n ? cand_score[base + lane] : -1.f;
    for (int t = 0; t < 32; ++t) {
      const int i = base + t;
      if (i >= n || kept >= p.max_out) { done = true; break; }
      const float s = __shfl_sync(0xffffffffu, sc, t);
      if (!(s > p.score_thresh)) { done = true; break; }        // sorted: nothing later passes either
      const int w = i >> 6, q = w >> 5;
      const unsigned long long mine = q == 0 ? rem[0] : q == 1 ? rem[1] : q == 2 ? rem[2] : rem[3];
      const unsigned long long word = __shfl_sync(0xffffffffu, mine, w & 31);
      if ((word >> (i & 63)) & 1ull) continue;
#pragma unroll
      for (int qq = 0; qq < 4; ++qq) {
        const int ww = lane + 32 * qq;
        if (ww >= w && ww < words) rem[qq] |= mask[static_cast<size_t>(i) * words + ww];
      }
      if (lane == 0) {
        const float4 b = cand_box[i];                 // (ymin, xmin, ymax, xmax) * scale -> x1 y1 x2 y2
        out_boxes[kept] = make_float4(__fmul_rn(b.y, scale), __fmul_rn(b.x, scale), __fmul_rn(b.w, scale),
                                      __fmul_rn(b.z, scale));
        out_scores[kept] = s;
        out_classes[kept] = cand_cls[i];
        out_levels[kept] = cand_lvl[i];
      }
      ++kept;
    }
  }
  for (int j = kept + lane; j < p.max_out; j += 32) {
    out_boxes[j] = make_float4(0.f, 0.f, 0.f, 0.f);
    out_scores[j] = 0.f;
    out_classes[j] = 0;
    out_levels[j] = p.min_level;
  }
  if (lane == 0) p.out_count[img] = kept;
}

__global__ void topk_seed_kernel(uint32_t* state, uint32_t need) { state[8 * blockIdx.x + 2] = need; }

int next_pow2(int v) {
  int p = 1;
  while (p < v) p <<= 1;
  return p;
}

}  // namespace

int bifpn_set_input(BifpnInput& bi, const __half* hi, const __half* lo, int H, int W, int th, int tw) {
  bi.hi = hi; bi.lo = lo; bi.H = H; bi.W = W; bi.pad_t = bi.pad_l = 0; bi.weight = 1.f;
  if (H == th && W == tw) {
    bi.mode = 0;
  } else if (H > th && W > tw) {
    B2_CHECK((H - 1) / th + 1 == 2 && (W - 1) / tw + 1 == 2, "effdet: only stride-2 downsampling between levels");
    const int ph = (th - 1) * 2 + 3 - H, pw = (tw - 1) * 2 + 3 - W;
    bi.mode = 1;
    bi.pad_t = (ph > 0 ? ph : 0) / 2;
    bi.pad_l = (pw > 0 ? pw : 0) / 2;
  } else {
    B2_CHECK(H * 2 == th && W * 2 == tw, "effdet: only exact 2x nearest upsampling between levels");
    bi.mode = 2;
  }
  return 0;
}

void bifpn_set_weights(BifpnCombineParams& p, const float* raw) {
  float tot32 = 0.f;
  for (int i = 0; i < p.n_in; ++i) {
    const float r = raw[i] > 0.f ? raw[i] : 0.f;          // tf.nn.relu
    p.in[i].weight = r;
    tot32 = i == 0 ? r : tot32 + r;                       // tf.add_n in float32
  }
  p.denom = tot32 + 0.0001f;
}

int bifpn_combine_launch(const BifpnCombineParams& p, cudaStream_t s) {
  B2_CHECK(p.C % 8 == 0 && p.n_in >= 1 && p.n_in <= 3, "bifpn_combine: bad parameters");
  const size_t total = static_cast<size_t>(p.B) * p.Ho * p.Wo * (p.C / 8);
  bifpn_combine_kernel<<<grid_for(total, 256, 132 * 32), 256, 0, s>>>(p);
  B2_CUDA(cudaGetLastError());
  return 0;
}

int dw3x3_plain_launch(const __half* in_hi, const __half* in_lo, int B, int H, int W, int C, const float* w, __half* out_hi,
                       __half* out_lo, cudaStream_t s) {
  DwConvParams p{in_hi, in_lo, B, H, W, C, 3, 1, 1, 1, H, W, w, nullptr, out_hi, out_lo};
  return dwconv_launch(p, 0, s);
}

int effdet_topk_blocks() { return static_cast<int>(kTopkMaxBlocks); }

// top-k -> candidates -> sigmoid/decode -> class-agnostic NMS -> outputs for p.B images, each kernel once with the image
// as a grid dimension; all on the stream, no host sync
int effdet_post_launch(const EffdetPostParams& p, const float* image_scale_dev, cudaStream_t s) {
  B2_CHECK(p.k >= 1 && p.k <= 8192, "effdet post: max_detection_topk must be in [1, 8192]");
  B2_CHECK(p.total < (1ull << 32), "effdet post: more than 2^32 class logits");
  B2_CHECK(p.anchors <= 9 && p.n_levels <= 5, "effdet post: at most 9 anchors per cell and 5 levels");
  B2_CHECK(p.B >= 1 && p.B <= 1024, "effdet post: batch out of range");
  const unsigned B = static_cast<unsigned>(p.B);
  B2_CUDA(cudaMemsetAsync(p.hist, 0, B * 256 * sizeof(unsigned int), s));
  B2_CUDA(cudaMemsetAsync(p.state, 0, B * 8 * sizeof(uint32_t), s));
  const uint32_t need = static_cast<uint32_t>(static_cast<unsigned long long>(p.k) < p.total ? p.k : p.total);
  topk_seed_kernel<<<B, 1, 0, s>>>(p.state, need);
  const unsigned grid = grid_for(p.total, 256, kTopkMaxBlocks);
  for (int pass = 0; pass < 4; ++pass) {
    topk_hist_kernel<<<dim3(grid, B), 256, 0, s>>>(p, pass);
    topk_pick_kernel<<<dim3(1, B), 256, 0, s>>>(p, pass);
  }
  const unsigned long long chunk = (p.total + grid - 1) / grid;
  topk_collect_kernel<<<dim3(grid, B), 256, 0, s>>>(p, chunk);
  topk_tie_scan_kernel<<<dim3(1, B), 32, 0, s>>>(p, static_cast<int>(grid));
  topk_tie_write_kernel<<<dim3(grid, B), 256, 0, s>>>(p, chunk);
  const int KP = next_pow2(p.k);
  B2_CUDA(cudaFuncSetAttribute(det_prepare_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
  det_prepare_kernel<<<dim3(1, B), 1024, static_cast<size_t>(KP) * 8, s>>>(p, KP);
  const int words = (p.k + 63) / 64;
  nms_mask_kernel<<<dim3(words, words, B), 64, 0, s>>>(p.cand_box, p.state, p.nms_thr, p.k, words, p.mask);
  nms_scan_kernel<<<dim3(1, B), 32, 0, s>>>(p, words, image_scale_dev);
  B2_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace b2
