// Shared host-side declarations for libb200det: error plumbing, the conv description and its launchers.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>

namespace b2 {

void set_error(const std::string& msg);
const char* last_error();

#define B2_CUDA(expr)                                                                              \
  do {                                                                                             \
    cudaError_t _e = (expr);                                                                       \
    if (_e != cudaSuccess) {                                                                       \
      ::b2::set_error(std::string(#expr) + ": " + cudaGetErrorString(_e) + " @" + __FILE__ + ":" + \
                      std::to_string(__LINE__));                                                   \
      return -1;                                                                                   \
    }                                                                                              \
  } while (0)

#define B2_CHECK(cond, msg)                                                          \
  do {                                                                               \
    if (!(cond)) {                                                                   \
      ::b2::set_error(std::string(msg) + " @" + __FILE__ + ":" + std::to_string(__LINE__)); \
      return -1;                                                                     \
    }                                                                                \
  } while (0)

// Geometry + epilogue description of one implicit-GEMM convolution (also dense layers, as 1x1).
struct ConvDesc {
  // input view (may be a crop of a larger buffer: in_H/in_W are the view, pitch_* the buffer)
  int B = 1, in_H = 0, in_W = 0, Cin = 0;
  int in_pitch_H = 0, in_pitch_W = 0;       // buffer dims used for strides (>= view dims)
  int in_ld = 0;                            // pixel stride in elements (0 => Cin)
  int force_a_mode = -1;                    // tests: -1 auto, 0 tiled-2D A operand, 1 im2col TMA
  int force_epi = -1;                       // tests: -1 auto, 0 direct epilogue, 1 staged (refused where not eligible)
  int acc_kb = 0;                           // split precision: K-blocks per accumulation restart (0 default, <0 off)
  int R = 1, S = 1, stride = 1, dil = 1;
  int pad_t = 0, pad_b = 0, pad_l = 0, pad_r = 0;   // zero padding (pad_b/pad_r may be negative = crop)
  int Cout = 0;
  // output placement: conv output (Ho x Wo) written at (off_h, off_w) inside an out_H x out_W buffer
  int out_H = 0, out_W = 0, off_h = 0, off_w = 0, ldc = 0;
  int relu = 0;        // 0 none, 1 ReLU, 2 swish (x * sigmoid(x))
  int res_shift = 0;   // residual pixel = (p >> shift, q >> shift) in a res_H x res_W buffer
  int res_H = 0, res_W = 0, ldr = 0;
  // grouped conv (ResNeXt's conv2, nn.py:352-355): groups > 1 splits Cin and Cout into that many equal ranges, output
  // range g reading input range g only.  conv_tc takes Cin == Cout, Cin % 64 == 0 and groups of at most 64 channels that
  // tile 64: output columns [n0, n0 + 64) then read input channels [n0, n0 + 64) only, and the weights are packed per
  // 64-channel window, [Cout_pad][R*S*kGroupWindow] with the group blocks on each window's diagonal.  conv_simt reads the
  // dense block-diagonal expansion [Cout_pad][R*S*Cin] and ignores `groups`.
  int groups = 1;
  int Ho() const { return (in_H + pad_t + pad_b - ((R - 1) * dil + 1)) / stride + 1; }
  int Wo() const { return (in_W + pad_l + pad_r - ((S - 1) * dil + 1)) / stride + 1; }
};

constexpr int kGroupWindow = 64;   // input channels a grouped conv_tc layer's 64 output columns read (ConvDesc::groups)

// Packed weights of one conv: [Cout_pad][R*S*Cin] fp16 hi (+lo) ([Cout_pad][R*S*kGroupWindow] for a grouped conv_tc
// layer), fp32 bias[Cout_pad].
struct ConvWeights {
  __half* w_hi = nullptr;
  __half* w_lo = nullptr;
  float* bias = nullptr;
  int Cout_pad = 0;
  int K = 0;
};

struct ConvIO {
  const __half* in_hi = nullptr;
  const __half* in_lo = nullptr;
  __half* out_hi = nullptr;
  __half* out_lo = nullptr;
  float* out_f32 = nullptr;       // when set, fp32 output instead of fp16 planes
  const __half* res_hi = nullptr;
  const __half* res_lo = nullptr;
  // device word that the kernel ORs with 1 when an fp16-plane output leaves the representable range (|x| > 65504: the
  // hi plane would hold inf and every later layer would silently compute on it); nullptr = not monitored
  unsigned int* range_flag = nullptr;
};

// A fully prepared tensor-core conv launch (tensor maps encoded once, reused every frame).
struct ConvPlan;
ConvPlan* conv_tc_plan_create(const ConvDesc& d, const ConvWeights& w, const ConvIO& io, bool split, int num_sms);
void conv_tc_plan_destroy(ConvPlan*);
int conv_tc_launch(const ConvPlan*, cudaStream_t);
int conv_tc_init();   // resolves the driver entry point for cuTensorMapEncode*

// CUDA-core reference implementation of exactly the same contract (validation + odd shapes).
int conv_simt_launch(const ConvDesc& d, const ConvWeights& w, const ConvIO& io, bool split, cudaStream_t);

}  // namespace b2
