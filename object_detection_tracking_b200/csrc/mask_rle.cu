// Mask paste and COCO RLE: the drivers' per-detection post-processing of final_masks (obj_detect_tracking.py:716-739,
// obj_detect_imgs.py:501-527), fill_full_mask (nn.py:1565-1584) then pycocotools.mask.encode of the Fortran-ordered frame
// and counts.decode("ascii"), without ever building an H x W frame per detection.
//
// A detection's frame mask is 0 outside its box, so its column-major run lengths follow from the thresholded h x w patch
// and the patch's place.  Work and memory are proportional to the sum of the patches' areas:
//   mask_paste_bits_kernel  one CTA column per mask: the 28x28 source in shared memory, one warp per 32-row word of a
//                           patch column, each lane resizing one pixel (mask_rle_math.h) and __ballot_sync packing the
//                           thresholded column into bits, row r of column c at bit r % 32 of word c * ceil(h / 32) + r / 32,
//                           so bit order is the RLE's column-major order
//   mask_rle_bounds_kernel  one CTA per mask: the positions in the frame's column-major order where the value changes.
//                           Inside the patch they are the bits of v ^ (v << 1 | carry).  The pixel before a column's
//                           first row is outside the patch (0) unless the patch spans the full height, where it is the
//                           previous column's last row; the pixel after a column's last row is outside (0), except the
//                           full-height columns that abut.  Then the characters each count needs.
//   mask_rle_scan_kernel    the masks' string offsets (exclusive scan), the only values read back before the strings
//   mask_rle_chars_kernel   one CTA per mask: counts from consecutive change positions (the first run starts at 0, the
//                           last ends at H * W), rleToString's deltas, and the characters at their scanned offsets
//   mask_unpack_kernel      the full-frame variant: the patch bits into a zeroed [n][H][W] uint8 frame
// Every box's geometry is computed and checked on the host (mask_geometry) before anything is uploaded or launched.
#include <algorithm>
#include <string>
#include <vector>

#include "../../include/b200det.h"
#include "kernels.h"
#include "mask_rle_math.h"

struct b2_masks {
  int device = 0;
  cudaStream_t stream = nullptr;   // the standalone calls' stream (the engine's encode runs on the engine's)
  b2::DevBuf geom, src, words, pos, nbound, nchars, offs, chars, full;
  int64_t last_bytes = -1;         // string bytes of the last encode, held in `chars` for b2_masks_fetch
};

namespace b2 {

int DevBuf::reserve(size_t bytes, cudaStream_t s) {
  if (bytes <= cap) return 0;
  B2_CUDA(cudaStreamSynchronize(s));
  if (p) B2_CUDA(cudaFree(p));
  p = nullptr;
  cap = 0;
  B2_CUDA(cudaMalloc(&p, bytes));
  cap = bytes;
  return 0;
}

DevBuf::~DevBuf() {
  if (p) cudaFree(p);
}

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;

// Per mask: the patch (w = h = 0 when nothing lands) and its offsets into the bit and change-position workspaces.
struct MaskGeom {
  int32_t x0, y0, w, h;
  int64_t word_off, pos_off;
};

__device__ __forceinline__ int words_per_col(int h) { return (h + 31) >> 5; }

__global__ void __launch_bounds__(kThreads) mask_paste_bits_kernel(const MaskGeom* __restrict__ geom,
                                                                   const float* __restrict__ masks,
                                                                   uint32_t* __restrict__ words) {
  __shared__ float src[kMaskSide * kMaskSide];
  const MaskGeom m = geom[blockIdx.y];
  if (m.w == 0) return;
  const float* in = masks + static_cast<size_t>(blockIdx.y) * kMaskSide * kMaskSide;
  for (int i = threadIdx.x; i < kMaskSide * kMaskSide; i += kThreads) src[i] = in[i];
  __syncthreads();
  const int lane = threadIdx.x & 31, nw = words_per_col(m.h);
  const int64_t total = static_cast<int64_t>(m.w) * nw;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * kWarps + (threadIdx.x >> 5); i < total;
       i += static_cast<int64_t>(gridDim.x) * kWarps) {
    const int c = static_cast<int>(i / nw), r = static_cast<int>(i - static_cast<int64_t>(c) * nw) * 32 + lane;
    const bool on = r < m.h && mask_on(mask_resize_at(src, mask_tap(c, m.w), mask_tap(r, m.h)));
    const uint32_t word = __ballot_sync(0xffffffffu, on);
    if (lane == 0) words[m.word_off + i] = word;
  }
}

// Exclusive scan of v over the CTA; *total = the CTA's sum.  Every thread must call it.
template <typename T>
__device__ T block_exclusive_scan(T v, T* total) {
  __shared__ T warp_sum[kWarps];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  T x = v;
  for (int o = 1; o < 32; o <<= 1) {
    const T y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warp_sum[warp] = x;
  __syncthreads();
  T before = 0, all = 0;
  for (int w = 0; w < kWarps; ++w) {
    if (w < warp) before += warp_sum[w];
    all += warp_sum[w];
  }
  __syncthreads();   // warp_sum is reused by the next call
  *total = all;
  return before + x - v;
}

// Change position j of a mask with k changes: 0 before the first, H * W after the last.
__device__ __forceinline__ int64_t change_at(const uint32_t* pos, int64_t k, int64_t j, int64_t hw) {
  return j < 0 ? 0 : (j < k ? static_cast<int64_t>(pos[j]) : hw);
}

// rleToString's value for count j: the count, minus the count two before it from j = 3 on.
__device__ __forceinline__ long long rle_value(const uint32_t* pos, int64_t k, int64_t j, int64_t hw) {
  long long x = change_at(pos, k, j, hw) - change_at(pos, k, j - 1, hw);
  if (j > 2) x -= change_at(pos, k, j - 2, hw) - change_at(pos, k, j - 3, hw);
  return x;
}

__global__ void __launch_bounds__(kThreads) mask_rle_bounds_kernel(const MaskGeom* __restrict__ geom,
                                                                   const uint32_t* __restrict__ words, int H, int W,
                                                                   uint32_t* __restrict__ pos, int64_t* __restrict__ nbound,
                                                                   int64_t* __restrict__ nchars) {
  const MaskGeom m = geom[blockIdx.x];
  const int64_t hw = static_cast<int64_t>(H) * W;
  uint32_t* out = pos + m.pos_off;
  int64_t k = 0;
  if (m.w > 0) {
    const int nw = words_per_col(m.h);
    const bool full = m.h == H;   // then y0 == 0 and columns abut
    const int64_t total = static_cast<int64_t>(m.w) * nw;
    const uint32_t* wd = words + m.word_off;
    for (int64_t c0 = 0; c0 < total; c0 += kThreads) {
      const int64_t i = c0 + threadIdx.x;
      uint32_t d = 0, base = 0;
      bool tail = false;
      if (i < total) {
        const int c = static_cast<int>(i / nw), q = static_cast<int>(i - static_cast<int64_t>(c) * nw);
        const uint32_t v = wd[i];
        uint32_t carry = 0;
        if (q > 0)
          carry = wd[i - 1] >> 31;
        else if (full && c > 0)
          carry = (wd[i - 1] >> ((m.h - 1) & 31)) & 1u;
        const int rows = min(32, m.h - 32 * q);
        const uint32_t valid = rows == 32 ? 0xffffffffu : (1u << rows) - 1u;
        d = (v ^ ((v << 1) | carry)) & valid;
        base = static_cast<uint32_t>(m.x0 + c) * static_cast<uint32_t>(H) + static_cast<uint32_t>(m.y0 + 32 * q);
        if (q == nw - 1 && ((v >> (rows - 1)) & 1u) && !(full && c + 1 < m.w))
          tail = static_cast<int64_t>(base) + rows < hw;   // the run of ones stops after the column
      }
      int64_t chunk;
      int64_t at = k + block_exclusive_scan<int64_t>(__popc(d) + (tail ? 1 : 0), &chunk);
      for (uint32_t b = d; b; b &= b - 1) out[at++] = base + __ffs(b) - 1;
      if (tail) out[at] = base + (m.h - 32 * (nw - 1));
      k += chunk;
    }
  }
  __syncthreads();   // the positions are read across threads below
  long long chars = 0;
  for (int64_t j = threadIdx.x; j <= k; j += kThreads) chars += rle_char_len(rle_value(out, k, j, hw));
  long long sum;
  block_exclusive_scan<long long>(chars, &sum);
  if (threadIdx.x == 0) {
    nbound[blockIdx.x] = k;
    nchars[blockIdx.x] = sum;
  }
}

__global__ void mask_rle_scan_kernel(const int64_t* __restrict__ nchars, int n, int64_t* __restrict__ offs) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  int64_t s = 0;
  offs[0] = 0;
  for (int i = 0; i < n; ++i) offs[i + 1] = s += nchars[i];
}

__global__ void __launch_bounds__(kThreads) mask_rle_chars_kernel(const MaskGeom* __restrict__ geom,
                                                                  const uint32_t* __restrict__ pos,
                                                                  const int64_t* __restrict__ nbound,
                                                                  const int64_t* __restrict__ offs, int H, int W,
                                                                  char* __restrict__ chars) {
  const uint32_t* p = pos + geom[blockIdx.x].pos_off;
  const int64_t hw = static_cast<int64_t>(H) * W, k = nbound[blockIdx.x];
  char* out = chars + offs[blockIdx.x];
  int64_t done = 0;
  for (int64_t j0 = 0; j0 <= k; j0 += kThreads) {
    const int64_t j = j0 + threadIdx.x;
    const long long x = j <= k ? rle_value(p, k, j, hw) : 0;
    long long chunk;
    const long long at = block_exclusive_scan<long long>(j <= k ? rle_char_len(x) : 0, &chunk);
    if (j <= k) rle_emit(x, out + done + at);
    done += chunk;
  }
}

__global__ void __launch_bounds__(kThreads) mask_unpack_kernel(const MaskGeom* __restrict__ geom,
                                                               const uint32_t* __restrict__ words, int H, int W,
                                                               uint8_t* __restrict__ out) {
  const MaskGeom m = geom[blockIdx.y];
  if (m.w == 0) return;
  const int nw = words_per_col(m.h);
  const int64_t total = static_cast<int64_t>(m.w) * m.h;
  uint8_t* frame = out + static_cast<size_t>(blockIdx.y) * H * W;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * kThreads + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * kThreads) {
    const int r = static_cast<int>(i / m.w), c = static_cast<int>(i - static_cast<int64_t>(r) * m.w);
    const uint32_t word = words[m.word_off + static_cast<int64_t>(c) * nw + (r >> 5)];
    frame[static_cast<size_t>(m.y0 + r) * W + m.x0 + c] = static_cast<uint8_t>((word >> (r & 31)) & 1u);
  }
}

int refuse(const std::string& msg) {
  set_error(msg);
  return kMaskRefused;
}

// Host geometry of every box, the uploads and the paste.  On return the packed patches of the n masks are in e->words
// (enqueued on s); *max_words / the workspaces are sized from the geometry alone.
int paste(b2_masks* e, const float* boxes, const float* masks, int masks_on_device, int n, int mask_h, int mask_w, int H,
          int W, cudaStream_t s, const char* who) {
  const std::string w(who);
  if (n < 0 || n > 65535) return refuse(w + ": needs 0 <= n <= 65535 masks");
  if (n > 0 && (!boxes || !masks)) return refuse(w + ": null argument");
  if (mask_h != kMaskSide || mask_w != kMaskSide) return refuse(w + ": masks must be 28x28 (the mask head's output)");
  if (H < 1 || W < 1 || static_cast<int64_t>(H) * W >= (int64_t{1} << 31))
    return refuse(w + ": needs a frame of 1 to 2^31 - 1 pixels");
  std::vector<MaskGeom> g(n);
  int64_t words = 0, positions = 0, max_words = 0;
  for (int i = 0; i < n; ++i) {
    MaskPlace p;
    const int st = mask_geometry(boxes + 4 * i, H, W, &p);
    const std::string box = w + ": box " + std::to_string(i);
    if (st == kMaskGeomRange) return refuse(box + " has a coordinate that is not finite or not below 2^30");
    if (st == kMaskGeomNegative) return refuse(box + " has a corner int(box[:2] + 0.5) below 0");
    if (st == kMaskGeomOverhang)
      return refuse(box + ": could not broadcast its " + std::to_string(p.h) + "x" + std::to_string(p.w) +
                    " patch into the frame at (" + std::to_string(p.y0) + ", " + std::to_string(p.x0) + ")");
    g[i].x0 = p.x0;
    g[i].y0 = p.y0;
    g[i].w = p.pasted ? p.w : 0;
    g[i].h = p.pasted ? p.h : 0;
    g[i].word_off = words;
    g[i].pos_off = positions;
    const int64_t nwords = static_cast<int64_t>(g[i].w) * ((g[i].h + 31) / 32);
    words += nwords;
    positions += static_cast<int64_t>(g[i].w) * (g[i].h + 1);   // at most one change per pixel plus one per column
    max_words = std::max(max_words, nwords);
  }
  if (n == 0) return 0;
  if (e->geom.reserve(sizeof(MaskGeom) * n, s) || e->words.reserve(sizeof(uint32_t) * std::max<int64_t>(words, 1), s) ||
      e->pos.reserve(sizeof(uint32_t) * std::max<int64_t>(positions, 1), s))
    return -1;
  B2_CUDA(cudaMemcpyAsync(e->geom.p, g.data(), sizeof(MaskGeom) * n, cudaMemcpyHostToDevice, s));
  const float* d_masks = masks;
  if (!masks_on_device) {
    const size_t bytes = sizeof(float) * kMaskSide * kMaskSide * n;
    if (e->src.reserve(bytes, s)) return -1;
    B2_CUDA(cudaMemcpyAsync(e->src.p, masks, bytes, cudaMemcpyHostToDevice, s));
    d_masks = static_cast<const float*>(e->src.p);
  }
  const unsigned gx = static_cast<unsigned>(std::min<int64_t>(std::max<int64_t>((max_words + kWarps - 1) / kWarps, 1), 256));
  mask_paste_bits_kernel<<<dim3(gx, n), kThreads, 0, s>>>(static_cast<const MaskGeom*>(e->geom.p), d_masks,
                                                          static_cast<uint32_t*>(e->words.p));
  B2_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace

int mask_encode(b2_masks* e, const float* boxes, const float* masks, int masks_on_device, int n, int mask_h, int mask_w,
                int H, int W, int64_t* offsets, char* bytes, int64_t capacity, cudaStream_t s, const char* who) {
  if (!offsets) return refuse(std::string(who) + ": null argument");
  e->last_bytes = -1;
  if (int rc = paste(e, boxes, masks, masks_on_device, n, mask_h, mask_w, H, W, s, who)) return rc;
  offsets[0] = 0;
  if (n == 0) {
    e->last_bytes = 0;
    return 0;
  }
  if (e->nbound.reserve(sizeof(int64_t) * n, s) || e->nchars.reserve(sizeof(int64_t) * n, s) ||
      e->offs.reserve(sizeof(int64_t) * (n + 1), s))
    return -1;
  const MaskGeom* g = static_cast<const MaskGeom*>(e->geom.p);
  uint32_t* pos = static_cast<uint32_t*>(e->pos.p);
  int64_t* nbound = static_cast<int64_t*>(e->nbound.p);
  int64_t* offs = static_cast<int64_t*>(e->offs.p);
  mask_rle_bounds_kernel<<<n, kThreads, 0, s>>>(g, static_cast<const uint32_t*>(e->words.p), H, W, pos, nbound,
                                               static_cast<int64_t*>(e->nchars.p));
  B2_CUDA(cudaGetLastError());
  mask_rle_scan_kernel<<<1, 32, 0, s>>>(static_cast<const int64_t*>(e->nchars.p), n, offs);
  B2_CUDA(cudaGetLastError());
  B2_CUDA(cudaMemcpyAsync(offsets, offs, sizeof(int64_t) * (n + 1), cudaMemcpyDeviceToHost, s));
  B2_CUDA(cudaStreamSynchronize(s));
  const int64_t total = offsets[n];
  if (e->chars.reserve(std::max<int64_t>(total, 1), s)) return -1;
  mask_rle_chars_kernel<<<n, kThreads, 0, s>>>(g, pos, nbound, offs, H, W, static_cast<char*>(e->chars.p));
  B2_CUDA(cudaGetLastError());
  if (bytes && capacity >= total) B2_CUDA(cudaMemcpyAsync(bytes, e->chars.p, total, cudaMemcpyDeviceToHost, s));
  B2_CUDA(cudaStreamSynchronize(s));
  e->last_bytes = total;
  return 0;
}

}  // namespace b2

using namespace b2;

extern "C" {

int b2_masks_create(b2_masks** out, int device) {
  B2_CHECK(out, "b2_masks_create: null argument");
  *out = nullptr;
  B2_CUDA(cudaSetDevice(device));
  b2_masks* e = new b2_masks();
  e->device = device;
  if (cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking) != cudaSuccess) {
    delete e;
    B2_CHECK(false, "b2_masks_create: cudaStreamCreate failed");
  }
  *out = e;
  return 0;
}

void b2_masks_destroy(b2_masks* e) {
  if (!e) return;
  cudaSetDevice(e->device);
  cudaStreamSynchronize(e->stream);
  cudaStreamDestroy(e->stream);
  delete e;   // the workspaces free themselves
}

int b2_masks_paste(b2_masks* e, const float* boxes_host, const float* masks, int masks_on_device, int n, int mask_h,
                   int mask_w, int im_h, int im_w, uint8_t* out_host, int64_t capacity_bytes) {
  B2_CHECK(e, "b2_masks_paste: null argument");
  B2_CUDA(cudaSetDevice(e->device));
  if (n > 0 && (!out_host || capacity_bytes < static_cast<int64_t>(n) * im_h * im_w))
    return refuse("b2_masks_paste: the output needs n * im_h * im_w bytes");
  cudaStream_t s = e->stream;
  if (int rc = paste(e, boxes_host, masks, masks_on_device, n, mask_h, mask_w, im_h, im_w, s, "b2_masks_paste")) return rc;
  if (n == 0) return 0;
  const size_t bytes = static_cast<size_t>(n) * im_h * im_w;
  if (e->full.reserve(bytes, s)) return -1;
  B2_CUDA(cudaMemsetAsync(e->full.p, 0, bytes, s));
  mask_unpack_kernel<<<dim3(1024, n), kThreads, 0, s>>>(static_cast<const MaskGeom*>(e->geom.p),
                                                        static_cast<const uint32_t*>(e->words.p), im_h, im_w,
                                                        static_cast<uint8_t*>(e->full.p));
  B2_CUDA(cudaGetLastError());
  B2_CUDA(cudaMemcpyAsync(out_host, e->full.p, bytes, cudaMemcpyDeviceToHost, s));
  B2_CUDA(cudaStreamSynchronize(s));
  return 0;
}

int b2_masks_encode(b2_masks* e, const float* boxes_host, const float* masks, int masks_on_device, int n, int mask_h,
                    int mask_w, int im_h, int im_w, int64_t* offsets_host, char* bytes_host, int64_t capacity) {
  B2_CHECK(e, "b2_masks_encode: null argument");
  B2_CUDA(cudaSetDevice(e->device));
  return mask_encode(e, boxes_host, masks, masks_on_device, n, mask_h, mask_w, im_h, im_w, offsets_host, bytes_host,
                     capacity, e->stream, "b2_masks_encode");
}

int b2_masks_fetch(b2_masks* e, char* bytes_host, int64_t capacity) {
  B2_CHECK(e && (bytes_host || capacity == 0), "b2_masks_fetch: null argument");
  B2_CHECK(e->last_bytes >= 0, "b2_masks_fetch: no encode to fetch");
  B2_CHECK(capacity >= e->last_bytes, "b2_masks_fetch: buffer too small");
  B2_CUDA(cudaSetDevice(e->device));
  if (e->last_bytes) B2_CUDA(cudaMemcpy(bytes_host, e->chars.p, e->last_bytes, cudaMemcpyDeviceToHost));
  return 0;
}

}  // extern "C"

int b2::mask_encoder_device(const b2_masks* e) { return e->device; }
