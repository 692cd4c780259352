// The mask head's last step (models.py:950-958): per final detection the logits of its own class, sigmoid, and the
// un-shuffle of the 2x2 transposed-conv taps.  The convs before it are conv_tc layers (detplan.cu: add_mask_head).
#include <algorithm>

#include "common.h"
#include "kernels.h"

namespace b2 {
namespace {

// logits rows are ((roi * 196 + y * 14 + x) * 4 + dy * 2 + dx); out [B*R][28][28]
__global__ void mask_select_kernel(const float* __restrict__ logits, int ld, const int* __restrict__ labels,
                                   const int* __restrict__ count, int B, int R, float* __restrict__ out) {
  const size_t total = static_cast<size_t>(B) * R * 784;
  for (size_t idx = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int px = static_cast<int>(idx % 784);
    const size_t roi = idx / 784;
    const int b = static_cast<int>(roi / R), j = static_cast<int>(roi % R);
    float v = 0.f;
    if (j < count[b]) {
      const int Y = px / 28, X = px % 28;
      const size_t row = (roi * 196 + static_cast<size_t>(Y >> 1) * 14 + (X >> 1)) * 4 + (Y & 1) * 2 + (X & 1);
      const float z = logits[row * ld + (labels[roi] - 1)];
      v = 1.f / (1.f + expf(-z));
    }
    out[idx] = v;
  }
}

}  // namespace

int mask_select_launch(const float* logits, int ld, const int* labels, const int* count, int B, int R, float* out,
                       cudaStream_t s) {
  const size_t total = static_cast<size_t>(B) * R * 784;
  mask_select_kernel<<<static_cast<unsigned>(std::min<size_t>((total + 255) / 256, 132 * 32)), 256, 0, s>>>(
      logits, ld, labels, count, B, R, out);
  B2_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace b2
