// The pool of the attention box head (use_att_frcnn_head, fastrcnn_2fc_head models.py:1064-1089, batch graph :2682-2707):
//
//   attention = conv2d(feature, 1, kernel 3, SAME, bias, activation=softmax)   [K][7][7][1]
//   attended  = sum over the 49 cells of feature * attention                  [K][256]
//
// The softmax runs over the last axis, which has length 1: for a finite logit x the weight is exp(x - x) / exp(x - x) = 1
// exactly, and for a non-finite one it is NaN (inf - inf).  With the load-time check on the attention weights (finite,
// 65536 * sum|W| + |b| < FLT_MAX, detplan.cu load_att) a logit of finite features (|x| < 65536 in the fp16 planes) is
// finite, and a non-finite feature of a cell reaches the logit of that cell through the centre tap, which reads all its
// channels.  So attended is the plain sum of the ROI's 49 cells when its 7 x 7 x C block is finite, and NaN in every
// channel otherwise.  That is what this kernel computes; it never evaluates the 3x3 conv.
#include <math.h>

#include "common.h"
#include "kernels.h"
#include "planes.cuh"

namespace b2 {
namespace {

// One block per ROI, one thread per channel octet (blockDim = C / 8).  Each thread sums its octet over bins 0 .. 48 in
// that order, in fp32.  Finite inputs are below 65536 in magnitude, so their 49-term sum is finite, and a non-finite input
// makes its channel's sum non-finite (inf, or NaN from inf - inf or a NaN): the block ORs "some sum is not finite", which
// is "some input of the ROI is not finite".
__global__ void att_pool_kernel(const __half* __restrict__ in_hi, const __half* __restrict__ in_lo, int C,
                                __half* __restrict__ out_hi, __half* __restrict__ out_lo, unsigned int* range_flag) {
  const size_t roi = blockIdx.x;
  const int c0 = threadIdx.x * 8;
  const size_t base = roi * 49 * C + c0;
  float s[8];
#pragma unroll
  for (int t = 0; t < 8; ++t) s[t] = 0.f;
#pragma unroll 7
  for (int bin = 0; bin < 49; ++bin) {
    float v[8];
    load8(in_hi, in_lo, base + static_cast<size_t>(bin) * C, v);
#pragma unroll
    for (int t = 0; t < 8; ++t) s[t] = __fadd_rn(s[t], v[t]);
  }
  bool bad = false;
#pragma unroll
  for (int t = 0; t < 8; ++t) bad = bad || !isfinite(s[t]);
  if (__syncthreads_or(bad)) {
#pragma unroll
    for (int t = 0; t < 8; ++t) s[t] = __int_as_float(0x7fc00000);   // the NaN weight of fact 2: the whole row
  } else if (range_flag != nullptr) {
    // a finite sum beyond the fp16 planes' range: the conv kernel's range monitor
    float amax = 0.f;
#pragma unroll
    for (int t = 0; t < 8; ++t) amax = fmaxf(amax, fabsf(s[t]));
    if (amax > 65504.f) atomicOr(range_flag, 1u);
  }
  store8(out_hi, out_lo, roi * C + c0, s);
}

}  // namespace

int att_pool_launch(const __half* in_hi, const __half* in_lo, int M, int C, __half* out_hi, __half* out_lo,
                    unsigned int* range_flag, cudaStream_t s) {
  B2_CHECK(M >= 1 && C >= 8 && C % 8 == 0 && C / 8 <= 1024, "att_pool: needs M >= 1 and C a multiple of 8 up to 8192");
  att_pool_kernel<<<M, C / 8, 0, s>>>(in_hi, in_lo, C, out_hi, out_lo, range_flag);
  B2_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace b2
