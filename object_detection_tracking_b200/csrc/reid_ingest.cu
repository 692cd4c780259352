// ReID ingest: track boxes of uint8 BGR frames -> the ReID engines' RGB uint8 crops [n][out_h][out_w][3], each box cut
// out and resized exactly as Pillow's Image.resize(BILINEAR) does (pil_resize_math.h), the host step the drivers run before
// FeatureExtractor (single_video_reid.py:211-227: image[y:y+h, x:x+w] -> cvtColor(BGR2RGB) -> T.Resize).
//
// One CTA per (box, band of kBand output rows).  The CTA builds the fixed-point weights of every output column and of its
// band's rows in shared memory, then:
//   - horizontal first (the usual case): it streams the source rows its band reads through shared memory in chunks of
//     kChunk rows, each chunk resampled horizontally into uint8 exactly like Pillow's intermediate image, and adds every
//     chunk row into its band's int32 vertical sums held in registers.  The sums are exact integers, so the order in
//     which chunks arrive cannot change a result, and a band of any height needs only one chunk of shared memory.
//   - vertical first (a crop more than 100 times taller than wide that shrinks in height): the band's rows of the
//     in_w-wide vertical pass fit in shared memory whole (in_w <= (H - 1) / 100), then the horizontal pass reads them.
// BGR -> RGB happens on the read.  Boxes are checked on the host (reid_boxes_check) before any launch; the kernel then
// never reads outside its box.
#include <limits.h>

#include <algorithm>
#include <string>

#include "kernels.h"
#include "pil_resize_math.h"

namespace b2 {
namespace {

constexpr int kThreads = 256;
constexpr int kBand = 8;                 // output rows per CTA
constexpr int kChunk = 32;               // source rows per horizontal-pass chunk
constexpr int kEpt = 3;                  // output elements (column x channel) per thread and row: out_w * 3 <= 3 * kThreads
constexpr int kMaxOutW = kEpt * kThreads / 3;

// Shared-memory layout, the same on host and device: the column weights [out_w][kx_cap], first tap and tap count of every
// column, the band's row weights [kBand][ky_cap] with their first tap and count, then the uint8 intermediate.
struct IngestLayout {
  int kx_cap, ky_cap;
  size_t inter_off, bytes;
};

IngestLayout ingest_layout(int H, int W, int out_h, int out_w) {
  IngestLayout L;
  L.kx_cap = pil_axis(W, out_w).ksize;   // ksize grows with the input size: the frame's bounds every box's
  L.ky_cap = pil_axis(H, out_h).ksize;
  L.inter_off = sizeof(int) * (static_cast<size_t>(out_w) * (L.kx_cap + 2) + static_cast<size_t>(kBand) * (L.ky_cap + 2));
  const size_t vfirst_w = std::min(W, (H - 1) / 100);   // widest crop that takes the vertical-first order
  L.bytes = L.inter_off + std::max(static_cast<size_t>(kChunk) * out_w * 3, static_cast<size_t>(kBand) * vfirst_w * 3);
  return L;
}

__global__ void __launch_bounds__(kThreads) reid_crop_resize_kernel(const uint8_t* __restrict__ frames, int H, int W,
                                                                    const int32_t* __restrict__ boxes,
                                                                    uint8_t* __restrict__ crops, int out_h, int out_w,
                                                                    int kx_cap, int ky_cap, int inter_off) {
  extern __shared__ __align__(16) unsigned char smem[];
  int* kx = reinterpret_cast<int*>(smem);
  int* kx0 = kx + out_w * kx_cap;
  int* kxn = kx0 + out_w;
  int* ky = kxn + out_w;
  int* ky0 = ky + kBand * ky_cap;
  int* kyn = ky0 + kBand;
  uint8_t* inter = smem + inter_off;

  const int b = blockIdx.y, y0 = blockIdx.x * kBand, rows = min(kBand, out_h - y0);
  const int32_t* box = boxes + static_cast<size_t>(b) * 5;
  const int w = box[3], h = box[4];
  const size_t pitch = static_cast<size_t>(W) * 3;
  const uint8_t* crop = frames + (static_cast<size_t>(box[0]) * H + box[2]) * pitch + static_cast<size_t>(box[1]) * 3;
  const PilAxis ax = pil_axis(w, out_w), ay = pil_axis(h, out_h);
  for (int xx = threadIdx.x; xx < out_w; xx += kThreads) kxn[xx] = pil_coeffs(ax, xx, kx + xx * kx_cap, kx0 + xx);
  if (threadIdx.x < rows) kyn[threadIdx.x] = pil_coeffs(ay, y0 + threadIdx.x, ky + threadIdx.x * ky_cap, ky0 + threadIdx.x);
  __syncthreads();

  const int ow3 = out_w * 3;
  uint8_t* dst = crops + (static_cast<size_t>(b) * out_h + y0) * ow3;
  if (pil_vertical_first(w, h, out_h)) {
    const int w3 = w * 3;
    for (int idx = threadIdx.x; idx < rows * w3; idx += kThreads) {
      const int i = idx / w3, e = idx - i * w3, x = e / 3, c = e - 3 * x;
      const uint8_t* s = crop + static_cast<size_t>(ky0[i]) * pitch + x * 3 + (2 - c);
      const int* k = ky + i * ky_cap;
      int acc = pil_round();
      for (int t = 0; t < kyn[i]; ++t) acc += s[t * pitch] * k[t];
      inter[idx] = pil_clip8(acc);
    }
    __syncthreads();
    for (int idx = threadIdx.x; idx < rows * ow3; idx += kThreads) {
      const int i = idx / ow3, e = idx - i * ow3, xx = e / 3, c = e - 3 * xx;
      const uint8_t* s = inter + i * w3 + kx0[xx] * 3 + c;
      const int* k = kx + xx * kx_cap;
      int acc = pil_round();
      for (int t = 0; t < kxn[xx]; ++t) acc += s[3 * t] * k[t];
      dst[idx] = pil_clip8(acc);
    }
    return;
  }

  int acc[kBand][kEpt];
#pragma unroll
  for (int i = 0; i < kBand; ++i)
#pragma unroll
    for (int j = 0; j < kEpt; ++j) acc[i][j] = pil_round();
  const int s0 = ky0[0], s1 = ky0[rows - 1] + kyn[rows - 1];   // source rows the band reads
  for (int c0 = s0; c0 < s1; c0 += kChunk) {
    const int nr = min(kChunk, s1 - c0);
    for (int idx = threadIdx.x; idx < nr * ow3; idx += kThreads) {
      const int r = idx / ow3, e = idx - r * ow3, xx = e / 3, c = e - 3 * xx;
      const uint8_t* s = crop + static_cast<size_t>(c0 + r) * pitch + kx0[xx] * 3 + (2 - c);
      const int* k = kx + xx * kx_cap;
      int a = pil_round();
      for (int t = 0; t < kxn[xx]; ++t) a += s[3 * t] * k[t];
      inter[idx] = pil_clip8(a);
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < kBand; ++i) {
      if (i >= rows) break;
      const int lo = max(ky0[i], c0), hi = min(ky0[i] + kyn[i], c0 + nr);
      const int* k = ky + i * ky_cap - ky0[i];
      for (int y = lo; y < hi; ++y) {
        const uint8_t* s = inter + (y - c0) * ow3;
        const int kv = k[y];
#pragma unroll
        for (int j = 0; j < kEpt; ++j) {
          const int e = threadIdx.x + j * kThreads;
          if (e < ow3) acc[i][j] += s[e] * kv;
        }
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < kBand; ++i) {
    if (i >= rows) break;
#pragma unroll
    for (int j = 0; j < kEpt; ++j) {
      const int e = threadIdx.x + j * kThreads;
      if (e < ow3) dst[i * ow3 + e] = pil_clip8(acc[i][j]);
    }
  }
}

}  // namespace

int reid_boxes_check(const int32_t* boxes, int n, int nf, int H, int W, const char* who) {
  B2_CHECK(boxes, std::string(who) + ": null box table");
  for (int i = 0; i < n; ++i) {
    const int32_t* b = boxes + static_cast<size_t>(i) * 5;
    const char* why = nullptr;
    if (b[0] < 0 || b[0] >= nf) why = "frame index out of range";
    else if (b[3] < 1 || b[4] < 1) why = "width and height must be at least 1";
    else if (b[1] < 0 || b[2] < 0 || static_cast<int64_t>(b[1]) + b[3] > W || static_cast<int64_t>(b[2]) + b[4] > H)
      why = "box leaves the frame";
    B2_CHECK(!why, std::string(who) + ": box " + std::to_string(i) + " (frame " + std::to_string(b[0]) + ", x " +
                       std::to_string(b[1]) + ", y " + std::to_string(b[2]) + ", w " + std::to_string(b[3]) + ", h " +
                       std::to_string(b[4]) + ") of " + std::to_string(nf) + " frames of " + std::to_string(W) + "x" +
                       std::to_string(H) + ": " + (why ? why : ""));
  }
  return 0;
}

int reid_crop_resize_launch(const uint8_t* frames, int H, int W, const int32_t* boxes, int n, uint8_t* crops, int out_h,
                            int out_w, cudaStream_t s) {
  B2_CHECK(n >= 1 && n <= 65535 && H >= 1 && W >= 1 && out_h >= 1 && out_w >= 1 && out_w <= kMaxOutW,
           "reid_crop_resize: needs 1 <= n <= 65535, positive sizes and out_w <= " + std::to_string(kMaxOutW));
  B2_CHECK(static_cast<size_t>(W) * 3 * kChunk <= INT_MAX, "reid_crop_resize: frame too wide");
  const IngestLayout L = ingest_layout(H, W, out_h, out_w);
  int dev = 0, optin = 0;
  B2_CUDA(cudaGetDevice(&dev));
  B2_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  B2_CHECK(L.bytes <= static_cast<size_t>(optin),
           "reid_crop_resize: a " + std::to_string(W) + "x" + std::to_string(H) + " frame needs " + std::to_string(L.bytes) +
               " bytes of shared memory for its resize weights, more than the " + std::to_string(optin) + " a CTA can have");
  if (L.bytes > 48 * 1024)
    B2_CUDA(cudaFuncSetAttribute(reid_crop_resize_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 static_cast<int>(L.bytes)));
  const dim3 grid((out_h + kBand - 1) / kBand, n);
  reid_crop_resize_kernel<<<grid, kThreads, L.bytes, s>>>(frames, H, W, boxes, crops, out_h, out_w, L.kx_cap, L.ky_cap,
                                                          static_cast<int>(L.inter_off));
  B2_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace b2
