// CUDA-core implementation of the ConvDesc contract (same operands, same hi/lo arithmetic, fp32
// accumulate) -- the on-device cross-check for the tensor-core kernel and the path for shapes the
// tensor-core kernel does not take (Cin % 64 != 0).  One thread per (pixel, 4 output channels).
#include "common.h"
#include "planes.cuh"

namespace b2 {
namespace {

template <bool SPLIT>
__global__ void conv_simt_kernel(ConvDesc d, ConvWeights w, ConvIO io, int Ho, int Wo) {
  const int in_ld = d.in_ld > 0 ? d.in_ld : d.Cin;
  const int ngroups = w.Cout_pad / 4;
  const size_t total = static_cast<size_t>(d.B) * Ho * Wo * ngroups;
  for (size_t idx = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int ng = static_cast<int>(idx % ngroups);
    const size_t m = idx / ngroups;
    const int img = static_cast<int>(m / (Ho * Wo));
    const int rem = static_cast<int>(m % (Ho * Wo));
    const int p = rem / Wo, q = rem % Wo;
    float acc0[4] = {0, 0, 0, 0}, acc1[4] = {0, 0, 0, 0};
    for (int r = 0; r < d.R; ++r) {
      const int ih = p * d.stride - d.pad_t + r * d.dil;
      if (ih < 0 || ih >= d.in_H) continue;
      for (int s = 0; s < d.S; ++s) {
        const int iw = q * d.stride - d.pad_l + s * d.dil;
        if (iw < 0 || iw >= d.in_W) continue;
        const size_t ipix = (static_cast<size_t>(img) * d.in_pitch_H + ih) * d.in_pitch_W + iw;
        const __half* xh = io.in_hi + ipix * in_ld;
        const __half* xl = SPLIT ? io.in_lo + ipix * in_ld : nullptr;
        const size_t kbase = static_cast<size_t>(r * d.S + s) * d.Cin;
        for (int c = 0; c < d.Cin; ++c) {
          const float ah = __half2float(xh[c]);
          const float al = SPLIT ? __half2float(xl[c]) : 0.f;
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const size_t wi = static_cast<size_t>(ng * 4 + j) * w.K + kbase + c;
            const float bh = __half2float(w.w_hi[wi]);
            acc0[j] = fmaf(ah, bh, acc0[j]);
            if (SPLIT) {
              const float bl = __half2float(w.w_lo[wi]);
              acc1[j] = fmaf(ah, bl, acc1[j]);
              acc1[j] = fmaf(al, bh, acc1[j]);
            }
          }
        }
      }
    }
    const int pp = p + d.off_h, qq = q + d.off_w;
    const size_t opix = (static_cast<size_t>(img) * d.out_H + pp) * d.out_W + qq;
    const size_t rpix = (static_cast<size_t>(img) * d.res_H + (pp >> d.res_shift)) * d.res_W + (qq >> d.res_shift);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = ng * 4 + j;
      float v = acc0[j];
      if (SPLIT) v = fmaf(acc1[j], kLoInv, v);
      v += w.bias[n];
      if (io.res_hi) {
        v += __half2float(io.res_hi[rpix * d.ldr + n]);
        if (SPLIT && io.res_lo) v = join(v, io.res_lo[rpix * d.ldr + n]);
      }
      if (d.relu == 1) v = fmaxf(v, 0.f);
      else if (d.relu == 2) v = __fmul_rn(v, 1.f / (1.f + expf(-v)));
      if (io.out_f32) io.out_f32[opix * d.ldc + n] = v;
      else store1(io.out_hi, SPLIT ? io.out_lo : nullptr, opix * d.ldc + n, v);
    }
  }
}

}  // namespace

int conv_simt_launch(const ConvDesc& d, const ConvWeights& w, const ConvIO& io, bool split, cudaStream_t stream) {
  const int Ho = d.Ho(), Wo = d.Wo();
  B2_CHECK(Ho > 0 && Wo > 0, "conv_simt: empty output");
  B2_CHECK(w.Cout_pad % 4 == 0 && d.ldc >= w.Cout_pad, "conv_simt: bad Cout_pad/ldc");
  const size_t total = static_cast<size_t>(d.B) * Ho * Wo * (w.Cout_pad / 4);
  const unsigned blocks = grid_for(total, 256, 132 * 64);
  if (split)
    conv_simt_kernel<true><<<blocks, 256, 0, stream>>>(d, w, io, Ho, Wo);
  else
    conv_simt_kernel<false><<<blocks, 256, 0, stream>>>(d, w, io, Ho, Wo);
  B2_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace b2
