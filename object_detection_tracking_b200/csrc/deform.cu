// deform.cu -- the bilinear sampler of a deformable conv2 (use_deformable: deformable_conv2d nn.py:1642-1712 with
// deformable_helper.py:42-137), the part of the layer that is not a GEMM.
//
// Output pixel (i, j) of image b reads the input around (2i, 2j): the reference samples every input position and the
// stride-2 conv3d keeps the even ones.  For tap k with base (by, bx) (kTapBase) and offsets (dy, dx):
//   y = (2i - 1 + by) + dy, x = (2j - 1 + bx) + dx          fp32, one rounding each
//   clamp y to [0, H - 1], x to [0, W - 1]                   border replication, no zero padding
//   y0 = floor(y), y1 = ceil(y), fy = y - y0 (x likewise)
//   t = v(y0, x0) + (v(y1, x0) - v(y0, x0)) * fy,  b = v(y0, x1) + (v(y1, x1) - v(y0, x1)) * fy
//   sample = t + (b - t) * fx
// each operation rounded on its own (no FMA), so the fp32 sample equals the reference's bit for bit before the split into
// planes.  The sample lands at [b][i][j][k][c]: the operand of a 1x1 conv with K = 9 * C whose weights are the 3x3
// kernel packed [Cout][3][3][C].  Samples are convex combinations of in-range inputs, so the store needs no range monitor.
#include "kernels.h"
#include "planes.cuh"

namespace b2 {
namespace {

constexpr int kThreads = 256;
constexpr int kPix = 4;   // output pixels per block

// Tap k's base relative to (2i - 1, 2j - 1).  initial_offset = reshape(stack(meshgrid(range(3), range(3), "ij")), (-1, 2))
// pairs up the [2][3][3] stack row-major, so the bases are not the 3x3 grid; tap k still multiplies W[k / 3][k % 3].
__constant__ int kTapBase[9][2] = {{0, 0}, {0, 1}, {1, 1}, {2, 2}, {2, 0}, {1, 2}, {0, 1}, {2, 0}, {1, 2}};

__global__ void __launch_bounds__(kThreads) deform_sample_kernel(DeformParams p, int npix) {
  __shared__ int s_pix[kPix * 9][4];   // input pixel index b * H * W + y * W + x of (y0, x0), (y1, x0), (y0, x1), (y1, x1)
  __shared__ float s_f[kPix * 9][2];   // fy, fx
  const int pix0 = blockIdx.x * kPix;
  const int np = min(kPix, npix - pix0);
  const int HoWo = p.Ho * p.Wo;
  // coordinates and weights once per (pixel, tap)
  for (int t = threadIdx.x; t < np * 9; t += blockDim.x) {
    const int pix = pix0 + t / 9, k = t % 9;
    const int b = pix / HoWo, r = pix - b * HoWo, i = r / p.Wo, j = r - i * p.Wo;
    const float* o = p.offset + static_cast<size_t>(pix) * p.ld_off + 2 * k;
    float y = __fadd_rn(static_cast<float>(2 * i - 1 + kTapBase[k][0]), o[0]);
    float x = __fadd_rn(static_cast<float>(2 * j - 1 + kTapBase[k][1]), o[1]);
    y = fminf(fmaxf(y, 0.f), static_cast<float>(p.H - 1));
    x = fminf(fmaxf(x, 0.f), static_cast<float>(p.W - 1));
    const float fy0 = floorf(y), fx0 = floorf(x);
    const int y0 = static_cast<int>(fy0), y1 = static_cast<int>(ceilf(y));
    const int x0 = static_cast<int>(fx0), x1 = static_cast<int>(ceilf(x));
    const int img = b * p.H * p.W;
    s_pix[t][0] = img + y0 * p.W + x0;
    s_pix[t][1] = img + y1 * p.W + x0;
    s_pix[t][2] = img + y0 * p.W + x1;
    s_pix[t][3] = img + y1 * p.W + x1;
    s_f[t][0] = __fsub_rn(y, fy0);
    s_f[t][1] = __fsub_rn(x, fx0);
  }
  __syncthreads();
  // eight channels per thread: consecutive threads read consecutive 16-byte pieces of the same input pixels
  const int cv = p.C / 8;
  for (int t = threadIdx.x; t < np * 9 * cv; t += blockDim.x) {
    const int q = t / cv;
    const size_t c = static_cast<size_t>(t - q * cv) * 8;
    float v00[8], v10[8], v01[8], v11[8], out[8];
    load8(p.in_hi, p.in_lo, static_cast<size_t>(s_pix[q][0]) * p.C + c, v00);
    load8(p.in_hi, p.in_lo, static_cast<size_t>(s_pix[q][1]) * p.C + c, v10);
    load8(p.in_hi, p.in_lo, static_cast<size_t>(s_pix[q][2]) * p.C + c, v01);
    load8(p.in_hi, p.in_lo, static_cast<size_t>(s_pix[q][3]) * p.C + c, v11);
    const float fy = s_f[q][0], fx = s_f[q][1];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const float top = __fadd_rn(v00[e], __fmul_rn(__fsub_rn(v10[e], v00[e]), fy));
      const float bot = __fadd_rn(v01[e], __fmul_rn(__fsub_rn(v11[e], v01[e]), fy));
      out[e] = __fadd_rn(top, __fmul_rn(__fsub_rn(bot, top), fx));
    }
    store8(p.out_hi, p.out_lo, (static_cast<size_t>(pix0) * 9 + q) * p.C + c, out);
  }
}

}  // namespace

int deform_sample_launch(const DeformParams& p, int b0, int n, cudaStream_t s) {
  B2_CHECK(p.C % 8 == 0 && p.Ho == (p.H + 1) / 2 && p.Wo == (p.W + 1) / 2 && p.ld_off >= 18,
           "deform_sample: bad geometry");
  DeformParams q = p;
  const size_t in_img = static_cast<size_t>(p.H) * p.W * p.C, out_img = static_cast<size_t>(p.Ho) * p.Wo * 9 * p.C;
  q.in_hi += b0 * in_img;
  if (q.in_lo) q.in_lo += b0 * in_img;
  q.offset += static_cast<size_t>(b0) * p.Ho * p.Wo * p.ld_off;
  q.out_hi += b0 * out_img;
  if (q.out_lo) q.out_lo += b0 * out_img;
  const int npix = n * p.Ho * p.Wo;
  deform_sample_kernel<<<(npix + kPix - 1) / kPix, kThreads, 0, s>>>(q, npix);
  B2_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace b2
