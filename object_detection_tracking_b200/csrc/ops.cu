// Single-kernel entry points for parity tests and host tools: one conv, one grouped conv, one GroupNorm, one squeeze-excite,
// one relation module, the attention head's pool, the deformable sampler and conv, the frame resize, and the element-wise
// and reduction kernels around the GEMMs (depthwise convs, pools, the BiFPN combine, MBConv's squeeze-excite, OSNet's
// channel gate, EfficientNet's stem im2col, the ResNet stems' operand packs), and the distance kernels around the tracker / ReID GEMMs.  Each call owns its device buffers in an Arena, so
// every return path frees them.
// The squeeze-excite, relation and deformable-conv calls build a one-block plan with the detector's builders (detplan.h).
#include <limits.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "../../include/b200det.h"
#include "detplan.h"

using namespace b2;

namespace {

// Runs the conv `d` (input, geometry, epilogue and residual size filled in; output placement and strides set here) on
// host x [B][H][W][Cin] with the packed weights pw [Cout_pad][K] and bias pb [Cout_pad]; res [B][res_H][res_W][Cout]
// may be null.  Writes out [B][Ho][Wo][Cout].
int run_conv(int device, ConvDesc d, const float* x, const std::vector<float>& pw, int K, const std::vector<float>& pb,
             const float* res, int impl, int split, float* out, const char* who) {
  const int Ho = d.Ho(), Wo = d.Wo(), Cout = d.Cout;
  const int Cp = (Cout + 15) / 16 * 16;
  d.out_H = Ho; d.out_W = Wo; d.ldc = Cp;
  d.ldr = Cp;
  const size_t nx = static_cast<size_t>(d.B) * d.in_H * d.in_W * d.Cin;
  const size_t nw = static_cast<size_t>(Cp) * K, no = static_cast<size_t>(d.B) * Ho * Wo * Cp;
  const size_t nr = static_cast<size_t>(d.B) * d.res_H * d.res_W * Cp;
  std::vector<float> pr;
  if (res) {
    pr.assign(nr, 0.f);
    for (size_t p = 0; p < static_cast<size_t>(d.B) * d.res_H * d.res_W; ++p)
      for (int o = 0; o < Cout; ++o) pr[p * Cp + o] = res[p * Cout + o];
  }
  // every operand is converted to both planes; fp16 precision leaves the lo planes unused
  Arena a;
  __half *xh = a.alloc<__half>(nx), *xl = a.alloc<__half>(nx), *oh = a.alloc<__half>(no), *ol = a.alloc<__half>(no);
  __half *rh = res ? a.alloc<__half>(nr) : nullptr, *rl = res ? a.alloc<__half>(nr) : nullptr;
  ConvWeights cw;
  cw.w_hi = a.alloc<__half>(nw);
  cw.w_lo = a.alloc<__half>(nw);
  cw.bias = a.alloc<float>(Cp);
  B2_CHECK(xh && xl && oh && ol && (!res || (rh && rl)) && cw.w_hi && cw.w_lo && cw.bias,
           std::string(who) + ": out of device memory");
  cudaStream_t st = nullptr;
  if (upload_planes(x, xh, xl, nx, st) || upload_planes(pw.data(), cw.w_hi, cw.w_lo, nw, st)) return -1;
  if (res && upload_planes(pr.data(), rh, rl, nr, st)) return -1;
  B2_CUDA(cudaMemcpy(cw.bias, pb.data(), Cp * 4, cudaMemcpyHostToDevice));
  cw.Cout_pad = Cp; cw.K = K;
  ConvIO io;
  io.in_hi = xh; io.in_lo = split ? xl : nullptr;
  io.out_hi = oh; io.out_lo = split ? ol : nullptr;
  io.res_hi = rh; io.res_lo = split ? rl : nullptr;
  if (!split) cw.w_lo = nullptr;
  if (impl == 0) {
    cudaDeviceProp prop;
    B2_CUDA(cudaGetDeviceProperties(&prop, device));
    PlanPtr plan(conv_tc_plan_create(d, cw, io, split != 0, prop.multiProcessorCount));
    B2_CHECK(plan != nullptr, std::string(who) + ": " + last_error());
    const int rc = conv_tc_launch(plan.get(), st);
    const cudaError_t e = cudaDeviceSynchronize();   // the kernel is done before its plan goes away
    if (rc) return -1;
    B2_CUDA(e);
  } else {
    if (conv_simt_launch(d, cw, io, split != 0, st)) return -1;
    B2_CUDA(cudaDeviceSynchronize());
  }
  std::vector<float> ho(no);
  if (download_planes(oh, split ? ol : nullptr, no, ho.data(), st)) return -1;
  for (size_t p = 0; p < static_cast<size_t>(d.B) * Ho * Wo; ++p)
    for (int o = 0; o < Cout; ++o) out[p * Cout + o] = ho[p * Cp + o];
  return 0;
}

// A one-block plan over B images in the caller's precision and conv implementation, its outputs not range-monitored.
void op_plan(DetPlan& p, int B, int split, int impl) {
  p.batch = B;
  p.split = split != 0;
  p.conv_impl = impl;
}

// Plans the convs of `p`, loads its weights from `ws`, runs its steps on the legacy stream and waits for them.
int run_plan(DetPlan& p, int device, const WeightSet& ws) {
  cudaDeviceProp prop;
  B2_CUDA(cudaGetDeviceProperties(&prop, device));
  if (plan_layers(p, prop.multiProcessorCount) || load_weights(p, ws, 0, nullptr)) return -1;
  const int rc = run_steps(p.steps, ~0u, nullptr);
  const cudaError_t e = cudaDeviceSynchronize();   // the kernels are done before their plans go away
  if (rc) return -1;
  B2_CUDA(e);
  return 0;
}

// A device copy of n host floats (16-byte aligned, as the kernels' float4 loads need); nullptr for a null host pointer,
// when out of memory or when the copy fails.
float* upload_f32(Arena& a, const float* host, size_t n) {
  if (!host) return nullptr;
  float* d = a.alloc<float>(n);
  if (d && cudaMemcpy(d, host, n * sizeof(float), cudaMemcpyHostToDevice) != cudaSuccess) d = nullptr;
  return d;
}

// The first n elements of the planes p joined to fp32 in out and, where given, raw into out_hi / out_lo.
int return_planes(const Planes& p, size_t n, float* out, uint16_t* out_hi, uint16_t* out_lo) {
  if (download_planes(p.hi, p.lo, n, out, nullptr)) return -1;
  if (out_hi) B2_CUDA(cudaMemcpy(out_hi, p.hi, n * sizeof(__half), cudaMemcpyDeviceToHost));
  if (out_lo && p.lo) B2_CUDA(cudaMemcpy(out_lo, p.lo, n * sizeof(__half), cudaMemcpyDeviceToHost));
  return 0;
}

}  // namespace

extern "C" {

int b2_op_conv2d(int device, const float* x, const float* w, const float* bias, const float* res, int B, int H, int W,
                 int Cin, int R, int S, int Cout, int stride, int dil, int pad_t, int pad_b, int pad_l, int pad_r,
                 int relu, int res_shift, int impl, int split, int a_mode, float* out) {
  B2_CHECK(x && w && out, "b2_op_conv2d: null argument");
  B2_CUDA(cudaSetDevice(device));
  ConvDesc d;
  d.B = B; d.in_H = H; d.in_W = W; d.Cin = Cin; d.in_pitch_H = H; d.in_pitch_W = W; d.in_ld = Cin;
  d.R = R; d.S = S; d.stride = stride; d.dil = dil;
  d.pad_t = pad_t; d.pad_b = pad_b; d.pad_l = pad_l; d.pad_r = pad_r;
  d.Cout = Cout; d.relu = relu; d.force_a_mode = a_mode;
  const int Ho = d.Ho(), Wo = d.Wo();
  B2_CHECK(Ho > 0 && Wo > 0, "b2_op_conv2d: empty output");
  const int Cp = (Cout + 15) / 16 * 16;
  d.res_H = res_shift ? (Ho + 1) / 2 : Ho; d.res_W = res_shift ? (Wo + 1) / 2 : Wo; d.res_shift = res_shift;
  const size_t K = static_cast<size_t>(R) * S * Cin;
  // pack HWIO -> [Cout_pad][R*S*Cin]
  std::vector<float> pw(static_cast<size_t>(Cp) * K, 0.f), pb(Cp, 0.f);
  for (size_t k = 0; k < K; ++k)
    for (int o = 0; o < Cout; ++o) pw[static_cast<size_t>(o) * K + k] = w[k * Cout + o];
  if (bias) for (int o = 0; o < Cout; ++o) pb[o] = bias[o];
  return run_conv(device, d, x, pw, static_cast<int>(K), pb, res, impl, split, out, "b2_op_conv2d");
}

int b2_op_conv2d_view(int device, const b2_conv_view* a, const float* x, const float* w, const float* bias,
                      const float* res, const float* out_init, float* out, uint16_t* out_hi, uint16_t* out_lo,
                      uint32_t* range_flag) {
  B2_CHECK(a && x && w && out_init && out, "b2_op_conv2d_view: null argument");
  const b2_conv_view& v = *a;
  B2_CHECK(v.B >= 1 && v.in_H >= 1 && v.in_W >= 1 && v.Cin >= 1 && v.Cout >= 1 && v.in_ld >= 1 && v.R >= 1 && v.S >= 1 &&
               v.stride >= 1 && v.dil >= 1 && v.pad_t >= 0 && v.pad_l >= 0,
           "b2_op_conv2d_view: sizes, strides and dilation must be positive, pad_t / pad_l not negative");
  B2_CHECK(v.in_H <= v.pitch_H && v.in_W <= v.pitch_W, "b2_op_conv2d_view: the view lies outside the input buffer");
  // the last pixel of the view reads Cin channels from its first element on (past its own in_ld when in_ld < Cin)
  const size_t n_in = static_cast<size_t>(v.B) * v.pitch_H * v.pitch_W * v.in_ld;
  const size_t last_px = (static_cast<size_t>(v.B - 1) * v.pitch_H + v.in_H - 1) * v.pitch_W + v.in_W - 1;
  B2_CHECK(last_px * v.in_ld + v.Cin <= n_in, "b2_op_conv2d_view: the last pixel's Cin channels run past the input buffer");
  ConvDesc d;
  d.B = v.B; d.in_H = v.in_H; d.in_W = v.in_W; d.Cin = v.Cin;
  d.in_pitch_H = v.pitch_H; d.in_pitch_W = v.pitch_W; d.in_ld = v.in_ld;
  d.force_a_mode = v.a_mode; d.force_epi = v.force_epi; d.acc_kb = v.acc_kb;
  d.R = v.R; d.S = v.S; d.stride = v.stride; d.dil = v.dil;
  d.pad_t = v.pad_t; d.pad_b = v.pad_b; d.pad_l = v.pad_l; d.pad_r = v.pad_r;
  d.Cout = v.Cout;
  d.out_H = v.out_H; d.out_W = v.out_W; d.off_h = v.off_h; d.off_w = v.off_w; d.ldc = v.ldc;
  d.relu = v.relu;
  const int Ho = d.Ho(), Wo = d.Wo(), Cp = (v.Cout + 15) / 16 * 16;
  B2_CHECK(Ho > 0 && Wo > 0, "b2_op_conv2d_view: empty output");
  B2_CHECK(v.off_h >= 0 && v.off_w >= 0 && v.off_h + Ho <= v.out_H && v.off_w + Wo <= v.out_W,
           "b2_op_conv2d_view: the placed output does not fit the output buffer");
  B2_CHECK(v.ldc >= Cp, "b2_op_conv2d_view: ldc must cover Cout_pad");
  if (res) {
    B2_CHECK(v.ldr >= Cp, "b2_op_conv2d_view: ldr must cover Cout_pad");
    B2_CHECK(v.res_shift >= 0 && v.res_shift < 16 && ((v.off_h + Ho - 1) >> v.res_shift) < v.res_H &&
                 ((v.off_w + Wo - 1) >> v.res_shift) < v.res_W,
             "b2_op_conv2d_view: the residual is smaller than the output coordinates index");
    d.res_H = v.res_H; d.res_W = v.res_W; d.ldr = v.ldr; d.res_shift = v.res_shift;
  }
  const int b0 = v.b0, nb = v.nb > 0 ? v.nb : v.B - v.b0;
  B2_CHECK(b0 >= 0 && nb >= 1 && b0 + nb <= v.B, "b2_op_conv2d_view: image range outside the batch");
  B2_CUDA(cudaSetDevice(device));
  const bool sp = v.split != 0;
  const size_t K = static_cast<size_t>(v.R) * v.S * v.Cin;
  const size_t n_out = static_cast<size_t>(v.B) * v.out_H * v.out_W * v.ldc;
  const size_t n_res = res ? static_cast<size_t>(v.B) * v.res_H * v.res_W * v.ldr : 0;
  // pack HWIO -> [Cout_pad][R*S*Cin]; columns [Cout, Cout_pad) have zero weights and bias
  std::vector<float> pw(static_cast<size_t>(Cp) * K, 0.f), pb(Cp, 0.f);
  for (size_t k = 0; k < K; ++k)
    for (int o = 0; o < v.Cout; ++o) pw[static_cast<size_t>(o) * K + k] = w[k * v.Cout + o];
  if (bias) std::copy(bias, bias + v.Cout, pb.begin());
  Arena ar;
  __half *xh = ar.alloc<__half>(n_in), *xl = sp ? ar.alloc<__half>(n_in) : nullptr;
  __half *oh = nullptr, *ol = nullptr, *rh = nullptr, *rl = nullptr;
  float* of = nullptr;
  if (v.out_f32) {
    of = ar.alloc<float>(n_out);
  } else {
    oh = ar.alloc<__half>(n_out);
    ol = sp ? ar.alloc<__half>(n_out) : nullptr;
  }
  if (res) {
    rh = ar.alloc<__half>(n_res);
    rl = sp ? ar.alloc<__half>(n_res) : nullptr;
  }
  ConvWeights cw;
  cw.w_hi = ar.alloc<__half>(pw.size());
  cw.w_lo = sp ? ar.alloc<__half>(pw.size()) : nullptr;
  cw.bias = ar.alloc<float>(Cp);
  cw.Cout_pad = Cp;
  cw.K = static_cast<int>(K);
  unsigned int* flag = ar.alloc<unsigned int>(1);
  B2_CHECK(xh && (!sp || xl) && (of || (oh && (!sp || ol))) && (!res || (rh && (!sp || rl))) && cw.w_hi &&
               (!sp || cw.w_lo) && cw.bias && flag,
           "b2_op_conv2d_view: out of device memory");
  // fp16 precision: the lo planes of the operands are not allocated and the conversion skips them
  cudaStream_t st = nullptr;
  if (upload_planes(x, xh, xl, n_in, st) || upload_planes(pw.data(), cw.w_hi, cw.w_lo, pw.size(), st)) return -1;
  if (res && upload_planes(res, rh, rl, n_res, st)) return -1;
  if (of) {
    B2_CUDA(cudaMemcpy(of, out_init, n_out * sizeof(float), cudaMemcpyHostToDevice));
  } else if (upload_planes(out_init, oh, ol, n_out, st)) {
    return -1;
  }
  B2_CUDA(cudaMemcpy(cw.bias, pb.data(), Cp * sizeof(float), cudaMemcpyHostToDevice));
  // images [b0, b0 + nb): every operand offset by whole images of its own buffer, as the engine's batch parts
  auto at = [b0](auto* p, int H, int W, int C) { return p ? p + static_cast<size_t>(b0) * H * W * C : p; };
  ConvIO io;
  io.in_hi = at(xh, v.pitch_H, v.pitch_W, v.in_ld);
  io.in_lo = at(xl, v.pitch_H, v.pitch_W, v.in_ld);
  io.out_hi = at(oh, v.out_H, v.out_W, v.ldc);
  io.out_lo = at(ol, v.out_H, v.out_W, v.ldc);
  io.out_f32 = at(of, v.out_H, v.out_W, v.ldc);
  io.res_hi = at(rh, v.res_H, v.res_W, v.ldr);
  io.res_lo = at(rl, v.res_H, v.res_W, v.ldr);
  io.range_flag = flag;
  d.B = nb;
  if (v.impl == 0) {
    cudaDeviceProp prop;
    B2_CUDA(cudaGetDeviceProperties(&prop, device));
    PlanPtr plan(conv_tc_plan_create(d, cw, io, sp, prop.multiProcessorCount));
    B2_CHECK(plan != nullptr, std::string("b2_op_conv2d_view: ") + last_error());
    const int rc = conv_tc_launch(plan.get(), st);
    const cudaError_t e = cudaDeviceSynchronize();   // the kernel is done before its plan goes away
    if (rc) return -1;
    B2_CUDA(e);
  } else {
    if (conv_simt_launch(d, cw, io, sp, st)) return -1;
    B2_CUDA(cudaDeviceSynchronize());
  }
  if (of) {
    B2_CUDA(cudaMemcpy(out, of, n_out * sizeof(float), cudaMemcpyDeviceToHost));
  } else {
    if (download_planes(oh, ol, n_out, out, st)) return -1;
    if (out_hi) B2_CUDA(cudaMemcpy(out_hi, oh, n_out * sizeof(__half), cudaMemcpyDeviceToHost));
    if (out_lo && ol) B2_CUDA(cudaMemcpy(out_lo, ol, n_out * sizeof(__half), cudaMemcpyDeviceToHost));
  }
  if (range_flag) B2_CUDA(cudaMemcpy(range_flag, flag, sizeof(unsigned int), cudaMemcpyDeviceToHost));
  return 0;
}

int b2_op_group_conv2d(int device, const float* x, const float* w, const float* bias, const float* res, int B, int H, int W,
                       int C, int R, int S, int groups, int stride, int dil, int pad_t, int pad_b, int pad_l, int pad_r,
                       int relu, int impl, int split, float* out) {
  B2_CHECK(x && w && out, "b2_op_group_conv2d: null argument");
  B2_CHECK(B >= 1 && C >= 1 && groups >= 1 && C % groups == 0, "b2_op_group_conv2d: groups must divide C");
  B2_CHECK(impl != 0 || (C % kGroupWindow == 0 && kGroupWindow % (C / groups) == 0),
           "b2_op_group_conv2d: the tensor-core windows need C % 64 == 0 and C / groups dividing 64");
  B2_CUDA(cudaSetDevice(device));
  ConvDesc d;
  d.B = B; d.in_H = H; d.in_W = W; d.Cin = C; d.in_pitch_H = H; d.in_pitch_W = W; d.in_ld = C;
  d.R = R; d.S = S; d.stride = stride; d.dil = dil;
  d.pad_t = pad_t; d.pad_b = pad_b; d.pad_l = pad_l; d.pad_r = pad_r;
  d.Cout = C; d.relu = relu; d.groups = groups;
  const int Ho = d.Ho(), Wo = d.Wo();
  B2_CHECK(Ho > 0 && Wo > 0, "b2_op_group_conv2d: empty output");
  d.res_H = Ho; d.res_W = Wo;
  const int Cp = (C + 15) / 16 * 16;
  // the tensor-core kernel reads 64-channel windows, the CUDA-core kernel the dense block-diagonal expansion
  const int K = R * S * (impl == 0 ? kGroupWindow : C);
  std::vector<float> pw(static_cast<size_t>(Cp) * K, 0.f), pb(Cp, 0.f);
  pack_grouped(w, R * S, C, C, groups, nullptr, K, pw);
  if (bias) for (int o = 0; o < C; ++o) pb[o] = bias[o];
  return run_conv(device, d, x, pw, K, pb, res, impl, split, out, "b2_op_group_conv2d");
}

int b2_op_group_norm(int device, const float* x, const float* res, const float* gamma, const float* beta, int B,
                     int pitch_H, int pitch_W, int C, int H, int W, int off_h, int off_w, int res_H, int res_W, int res_shift,
                     int relu, int per_roi, int split, int in_place, float* out) {
  B2_CHECK(x && gamma && beta && out, "b2_op_group_norm: null argument");
  B2_CHECK(B >= 1 && H >= 1 && W >= 1 && off_h >= 0 && off_w >= 0 && off_h + H <= pitch_H && off_w + W <= pitch_W,
           "b2_op_group_norm: view outside the buffer");
  B2_CHECK(!res || (res_shift >= 0 && ((H - 1) >> res_shift) < res_H && ((W - 1) >> res_shift) < res_W),
           "b2_op_group_norm: residual smaller than the view");
  B2_CUDA(cudaSetDevice(device));
  const size_t n = static_cast<size_t>(B) * pitch_H * pitch_W * C, nr = res ? static_cast<size_t>(B) * res_H * res_W * C : 0;
  Arena a;
  const Planes xp = a.planes(B, pitch_H, pitch_W, C, split != 0);
  const Planes yp = in_place ? xp : a.planes(B, pitch_H, pitch_W, C, split != 0);
  const Planes rp = res ? a.planes(B, res_H, res_W, C, split != 0) : Planes();
  GnParams p;
  memset(&p, 0, sizeof(p));
  p.chunks = gn_chunks(H, W, C);
  p.gamma = a.alloc<float>(C);
  p.beta = a.alloc<float>(C);
  p.partial = a.alloc<float>(static_cast<size_t>(B) * p.chunks * 32 * 3);
  p.stats = a.alloc<float>(static_cast<size_t>(B) * 32 * 2);
  p.counter = a.alloc<unsigned int>(B);
  B2_CHECK(xp.hi && yp.hi && (!res || rp.hi) && p.gamma && p.beta && p.partial && p.stats && p.counter,
           "b2_op_group_norm: out of device memory");
  if (upload_planes(x, xp.hi, xp.lo, n, nullptr)) return -1;
  if (res && upload_planes(res, rp.hi, rp.lo, nr, nullptr)) return -1;
  B2_CUDA(cudaMemcpy(const_cast<float*>(p.gamma), gamma, C * 4, cudaMemcpyHostToDevice));
  B2_CUDA(cudaMemcpy(const_cast<float*>(p.beta), beta, C * 4, cudaMemcpyHostToDevice));
  p.x_hi = xp.hi; p.x_lo = xp.lo; p.y_hi = yp.hi; p.y_lo = yp.lo;
  p.B = B; p.H = H; p.W = W; p.C = C;
  p.pitch_H = pitch_H; p.pitch_W = pitch_W; p.ld = C; p.off_h = off_h; p.off_w = off_w;
  if (res) {
    p.r_hi = rp.hi; p.r_lo = rp.lo; p.res_H = res_H; p.res_W = res_W; p.res_ld = C; p.res_shift = res_shift;
  }
  p.relu = relu;
  if (per_roi) {
    if (gn_roi_launch(p, nullptr)) return -1;
  } else {
    if (gn_stats_launch(p, nullptr) || gn_apply_launch(p, nullptr)) return -1;
  }
  B2_CUDA(cudaDeviceSynchronize());
  return download_planes(yp.hi, yp.lo, n, out, nullptr);
}

int b2_op_squeeze_excite(int device, const float* x, const float* res, const float* w1, const float* b1, const float* w2,
                         const float* b2, int B, int H, int W, int C, int nr, int split, float* out, float* gate_out) {
  B2_CHECK(x && w1 && b1 && w2 && b2 && out, "b2_op_squeeze_excite: null argument");
  B2_CHECK(B >= 1 && H >= 1 && W >= 1 && C >= 64 && C <= 2048 && (C & (C - 1)) == 0 && nr == C / 16,
           "b2_op_squeeze_excite: C must be a power of two from 64 to 2048 and nr = C / 16 (the SE-ResNet bottleneck's)");
  B2_CUDA(cudaSetDevice(device));
  DetPlan p;
  op_plan(p, B, split, 0);
  Planes xp, rp;
  B2_CHECK(p.alloc_planes(xp, B, H, W, C) && (!res || p.alloc_planes(rp, B, H, W, C)),
           "b2_op_squeeze_excite: out of device memory");
  if (upload_planes(x, xp.hi, xp.lo, xp.elems(), nullptr)) return -1;
  if (res && upload_planes(res, rp.hi, rp.lo, rp.elems(), nullptr)) return -1;
  if (add_se(p, 0, "block", xp, res ? &rp : nullptr)) return -1;
  WeightSet ws;
  ws.add("block/fc1/W", w1, static_cast<int64_t>(C) * nr);
  ws.add("block/fc1/b", b1, nr);
  ws.add("block/fc2/W", w2, static_cast<int64_t>(nr) * C);
  ws.add("block/fc2/b", b2, C);
  if (run_plan(p, device, ws)) return -1;
  if (gate_out) B2_CUDA(cudaMemcpy(gate_out, p.ses[0]->gate, static_cast<size_t>(B) * C * 4, cudaMemcpyDeviceToHost));
  return download_planes(xp.hi, xp.lo, xp.elems(), out, nullptr);
}

// One relation module through the box head's builder (add_relation).
int b2_op_relation(int device, const float* h, const float* boxes, const int32_t* count, const float* geo_emb_w,
                   const float* geo_emb_b, const float* geo_conv_w, const float* geo_conv_b, const float* query_w,
                   const float* key_w, const float* output_w, int B, int K, int D, int split, float* out) {
  B2_CHECK(h && boxes && count && geo_emb_w && geo_emb_b && geo_conv_w && geo_conv_b && query_w && key_w && output_w && out,
           "b2_op_relation: null argument");
  B2_CHECK(B >= 1 && K >= 1 && K <= 1024 && D >= 64 && D % 64 == 0,
           "b2_op_relation: needs B >= 1, 1 <= K <= 1024 and D a multiple of 64");
  for (int b = 0; b < B; ++b) B2_CHECK(count[b] >= 0 && count[b] <= K, "b2_op_relation: count outside [0, K]");
  B2_CUDA(cudaSetDevice(device));
  const int M = B * K;
  DetPlan p;
  op_plan(p, B, split, 0);
  Planes hp, op;
  float* dbox = p.arena.alloc<float>(static_cast<size_t>(M) * 4);
  int* dcount = p.arena.alloc<int>(B);
  B2_CHECK(p.alloc_rows(hp, M, D) && p.alloc_rows(op, M, D) && dbox && dcount, "b2_op_relation: out of device memory");
  if (upload_planes(h, hp.hi, hp.lo, static_cast<size_t>(M) * D, nullptr)) return -1;
  B2_CUDA(cudaMemcpy(dbox, boxes, static_cast<size_t>(M) * 4 * sizeof(float), cudaMemcpyHostToDevice));
  B2_CUDA(cudaMemcpy(dcount, count, B * sizeof(int), cudaMemcpyHostToDevice));
  if (add_relation(p, "rm", B, K, D, dbox, dcount, hp, op)) return -1;
  WeightSet ws;
  ws.add("rm/geo_emb/W", geo_emb_w, 4 * kRelGeoDim);
  ws.add("rm/geo_emb/b", geo_emb_b, kRelGeoDim);
  ws.add("rm/geo_conv/W", geo_conv_w, kRelGeoDim * kRelGroups);
  ws.add("rm/geo_conv/b", geo_conv_b, kRelGroups);
  ws.add("rm/query_linear/W", query_w, static_cast<int64_t>(D) * D);
  ws.add("rm/key_linear/W", key_w, static_cast<int64_t>(D) * D);
  ws.add("rm/output_linear/W", output_w, static_cast<int64_t>(kRelGroups) * D * D);
  if (run_plan(p, device, ws)) return -1;
  return download_planes(op.hi, op.lo, static_cast<size_t>(M) * D, out, nullptr);
}

// The attention head's pool alone (att_head.cu): fp32 [M][49][C] in, converted to the engine's planes; the pooled planes
// joined to fp32 out.
int b2_op_att_pool(int device, const float* x, int M, int C, int split, float* out) {
  B2_CHECK(x && out, "b2_op_att_pool: null argument");
  B2_CHECK(M >= 1 && C >= 8 && C % 8 == 0 && C <= 8192, "b2_op_att_pool: needs M >= 1 and C a multiple of 8 up to 8192");
  B2_CUDA(cudaSetDevice(device));
  Arena a;
  const Planes in = a.planes(1, 1, M, 49 * C, split != 0), o = a.planes(1, 1, M, C, split != 0);
  B2_CHECK(in.hi && o.hi, "b2_op_att_pool: out of device memory");
  if (upload_planes(x, in.hi, in.lo, static_cast<size_t>(M) * 49 * C, nullptr)) return -1;
  if (att_pool_launch(in.hi, in.lo, M, C, o.hi, o.lo, nullptr, nullptr)) return -1;
  B2_CUDA(cudaDeviceSynchronize());
  return download_planes(o.hi, o.lo, static_cast<size_t>(M) * C, out, nullptr);
}

// The deformable sampler alone: fp32 x and offsets in, the sampled operand's planes joined to fp32 out.
int b2_op_deform_sample(int device, const float* x, const float* offsets, int B, int H, int W, int C, int split, float* out) {
  B2_CHECK(x && offsets && out, "b2_op_deform_sample: null argument");
  B2_CHECK(B >= 1 && H >= 1 && W >= 1 && C >= 64 && C % 64 == 0, "b2_op_deform_sample: needs C a multiple of 64");
  B2_CUDA(cudaSetDevice(device));
  const bool sp = split != 0;
  const int Ho = (H + 1) / 2, Wo = (W + 1) / 2;
  const size_t nx = static_cast<size_t>(B) * H * W * C, noff = static_cast<size_t>(B) * Ho * Wo * 18;
  Arena a;
  const Planes xp = a.planes(B, H, W, C, sp), op = a.planes(B, Ho, Wo, 9 * C, sp);
  float* off = a.alloc<float>(noff);
  B2_CHECK(xp.hi && op.hi && off, "b2_op_deform_sample: out of device memory");
  if (upload_planes(x, xp.hi, xp.lo, nx, nullptr)) return -1;
  B2_CUDA(cudaMemcpy(off, offsets, noff * sizeof(float), cudaMemcpyHostToDevice));
  DeformParams p;
  p.in_hi = xp.hi; p.in_lo = xp.lo;
  p.offset = off; p.ld_off = 18;
  p.H = H; p.W = W; p.C = C; p.Ho = Ho; p.Wo = Wo;
  p.out_hi = op.hi; p.out_lo = op.lo;
  if (deform_sample_launch(p, 0, B, nullptr)) return -1;
  B2_CUDA(cudaDeviceSynchronize());
  return download_planes(op.hi, op.lo, op.elems(), out, nullptr);
}

// The deformable conv2 through the bottleneck's builder (add_deform).
int b2_op_deform_conv2d(int device, const float* x, const float* offset_w, const float* offset_b, const float* w, int B,
                        int H, int W, int C, int Cout, int impl, int split, float* out, float* offsets_out) {
  B2_CHECK(x && offset_w && offset_b && w && out, "b2_op_deform_conv2d: null argument");
  B2_CHECK(B >= 1 && H >= 2 && W >= 2 && C >= 64 && C % 64 == 0,
           "b2_op_deform_conv2d: needs C a multiple of 64");
  B2_CHECK(Cout == C, "b2_op_deform_conv2d: Cout must equal C (the bottleneck's deformable conv2 keeps its width)");
  B2_CUDA(cudaSetDevice(device));
  DetPlan p;
  op_plan(p, B, split, impl);
  Planes xp, op;
  B2_CHECK(p.alloc_planes(xp, B, H, W, C) && p.alloc_planes(op, B, (H + 1) / 2, (W + 1) / 2, C),
           "b2_op_deform_conv2d: out of device memory");
  if (upload_planes(x, xp.hi, xp.lo, xp.elems(), nullptr)) return -1;
  if (add_deform(p, "block", xp, op)) return -1;
  WeightSet ws;
  ws.add("block/conv2_offset/W", offset_w, static_cast<int64_t>(9) * C * 18);
  ws.add("block/conv2_offset/b", offset_b, 18);
  ws.add("block/conv2/W", w, static_cast<int64_t>(9) * C * C);
  if (run_plan(p, device, ws)) return -1;
  if (download_planes(op.hi, op.lo, op.elems(), out, nullptr)) return -1;
  if (offsets_out) {   // the offset conv's 18 columns of each [kDeformOffsetLd] row
    const Stage* s = p.stages.find("block/conv2_offset");
    if (!s) return -1;
    B2_CUDA(cudaMemcpy2D(offsets_out, 18 * sizeof(float), s->ptr, s->shape[3] * sizeof(float), 18 * sizeof(float),
                         op.elems() / C, cudaMemcpyDeviceToHost));
  }
  return 0;
}

// One depthwise conv: EfficientNet's strip kernel (impl 0) or OSNet's 3x3 (impl 1).
int b2_op_depthwise(int device, const float* x, const float* w, const float* bias, int B, int H, int W, int C, int K,
                    int stride, int pad_t, int pad_l, int Ho, int Wo, int act, int impl, int split, float* out,
                    uint16_t* out_hi, uint16_t* out_lo) {
  B2_CHECK(x && w && out, "b2_op_depthwise: null argument");
  B2_CHECK(B >= 1 && H >= 1 && W >= 1 && C >= 8 && C % 8 == 0,
           "b2_op_depthwise: needs positive sizes and C a multiple of 8");
  if (impl == 0) {
    B2_CHECK(B == 1 && (K == 3 || K == 5) && (stride == 1 || stride == 2) && pad_t >= 0 && pad_t < K && pad_l >= 0 &&
                 pad_l < K && Ho >= 1 && Wo >= 1 && (act == 0 || act == 2),
             "b2_op_depthwise: the strip kernel takes one image, K 3 or 5, stride 1 or 2, pads in [0, K), act 0 or 2");
  } else {
    B2_CHECK(impl == 1 && K == 3 && stride == 1 && pad_t == 1 && pad_l == 1 && Ho == H && Wo == W && act == 1 && bias,
             "b2_op_depthwise: OSNet's depthwise conv is 3x3, stride 1, pad 1, with a bias and ReLU");
  }
  B2_CUDA(cudaSetDevice(device));
  const bool sp = split != 0;
  Arena a;
  const Planes xp = a.planes(B, H, W, C, sp), op = a.planes(B, Ho, Wo, C, sp);
  float* dw = upload_f32(a, w, static_cast<size_t>(K) * K * C);
  float* db = upload_f32(a, bias, C);
  B2_CHECK(xp.hi && op.hi && dw && (!bias || db), "b2_op_depthwise: out of device memory");
  if (upload_planes(x, xp.hi, xp.lo, xp.elems(), nullptr)) return -1;
  if (impl == 0) {
    const DwConvParams p{xp.hi, xp.lo, 1, H, W, C, K, stride, pad_t, pad_l, Ho, Wo, dw, db, op.hi, op.lo};
    if (dwconv_launch(p, act, nullptr)) return -1;
  } else if (dwconv3x3_launch(xp.hi, xp.lo, B, H, W, C, dw, db, op.hi, op.lo, nullptr)) {
    return -1;
  }
  B2_CUDA(cudaDeviceSynchronize());
  return return_planes(op, op.elems(), out, out_hi, out_lo);
}

// One pool: the stems' 3x3/2 max-pool (kind 0), OSNet's AvgPool2d(2) (kind 1) or the global average pool (kind 2).
int b2_op_pool(int device, const float* x, int kind, int B, int H, int W, int C, int Ho, int Wo, int out_ld, int split,
               float* out, uint16_t* out_hi, uint16_t* out_lo) {
  B2_CHECK(x && out, "b2_op_pool: null argument");
  B2_CHECK(B >= 1 && H >= 1 && W >= 1 && C >= 8 && C % 8 == 0, "b2_op_pool: needs positive sizes and C a multiple of 8");
  if (kind == 0) {
    B2_CHECK(Ho >= 1 && Wo >= 1 && Ho <= (H + 1) / 2 && Wo <= (W + 1) / 2,
             "b2_op_pool: the max-pool's output must be at least 1 x 1 and at most ceil(H / 2) x ceil(W / 2)");
  } else if (kind == 1) {
    B2_CHECK(H >= 2 && W >= 2, "b2_op_pool: AvgPool2d(2) needs H, W >= 2");
    Ho = H / 2;
    Wo = W / 2;
  } else {
    B2_CHECK(kind == 2 && C % 64 == 0 && out_ld >= C, "b2_op_pool: kind 0, 1 or 2; the global pool needs C % 64 == 0 "
                                                      "and out_ld >= C");
  }
  B2_CUDA(cudaSetDevice(device));
  const bool sp = split != 0;
  Arena a;
  const Planes xp = a.planes(B, H, W, C, sp);
  const Planes op = kind == 2 ? Planes() : a.planes(B, Ho, Wo, C, sp);
  float* g = kind == 2 ? upload_f32(a, out, static_cast<size_t>(B) * out_ld) : nullptr;
  B2_CHECK(xp.hi && (kind == 2 ? g != nullptr : op.hi != nullptr), "b2_op_pool: out of device memory");
  if (upload_planes(x, xp.hi, xp.lo, xp.elems(), nullptr)) return -1;
  const int rc = kind == 0   ? maxpool_launch(xp.hi, xp.lo, B, H, W, C, op.hi, op.lo, Ho, Wo, nullptr)
                 : kind == 1 ? avgpool2_launch(xp.hi, xp.lo, B, H, W, C, op.hi, op.lo, nullptr)
                             : gap_launch(xp.hi, xp.lo, B, H * W, C, g, out_ld, nullptr);
  if (rc) return -1;
  B2_CUDA(cudaDeviceSynchronize());
  if (kind == 2) {
    B2_CUDA(cudaMemcpy(out, g, static_cast<size_t>(B) * out_ld * sizeof(float), cudaMemcpyDeviceToHost));
    return 0;
  }
  return return_planes(op, op.elems(), out, out_hi, out_lo);
}

// One BiFPN node combine, its inputs resampled and weighted as the EfficientDet engine sets them up.
int b2_op_bifpn_combine(int device, const float* x, const int32_t* hw, const float* weights, int n_in, int B, int Ho,
                        int Wo, int C, int swish, int split, float* out, uint16_t* out_hi, uint16_t* out_lo,
                        int32_t* resample) {
  B2_CHECK(x && hw && out, "b2_op_bifpn_combine: null argument");
  B2_CHECK(n_in >= 1 && n_in <= 3 && B >= 1 && Ho >= 1 && Wo >= 1 && C >= 8 && C % 8 == 0,
           "b2_op_bifpn_combine: needs 1 to 3 inputs, positive sizes and C a multiple of 8");
  BifpnCombineParams p;
  memset(&p, 0, sizeof(p));
  for (int i = 0; i < n_in; ++i) {
    B2_CHECK(hw[2 * i] >= 1 && hw[2 * i + 1] >= 1, "b2_op_bifpn_combine: empty input map");
    if (bifpn_set_input(p.in[i], nullptr, nullptr, hw[2 * i], hw[2 * i + 1], Ho, Wo)) return -1;
  }
  B2_CUDA(cudaSetDevice(device));
  const bool sp = split != 0;
  Arena a;
  Planes ip[3];
  const Planes op = a.planes(B, Ho, Wo, C, sp);
  B2_CHECK(op.hi, "b2_op_bifpn_combine: out of device memory");
  size_t at = 0;
  for (int i = 0; i < n_in; ++i) {
    ip[i] = a.planes(B, hw[2 * i], hw[2 * i + 1], C, sp);
    B2_CHECK(ip[i].hi, "b2_op_bifpn_combine: out of device memory");
    if (upload_planes(x + at, ip[i].hi, ip[i].lo, ip[i].elems(), nullptr)) return -1;
    at += ip[i].elems();
    p.in[i].hi = ip[i].hi;
    p.in[i].lo = ip[i].lo;
  }
  p.n_in = n_in; p.B = B; p.Ho = Ho; p.Wo = Wo; p.C = C;
  p.weighted = weights != nullptr; p.denom = 1.f; p.swish = swish != 0;
  if (weights) bifpn_set_weights(p, weights);
  p.out_hi = op.hi; p.out_lo = op.lo;
  if (bifpn_combine_launch(p, nullptr)) return -1;
  B2_CUDA(cudaDeviceSynchronize());
  if (resample)
    for (int i = 0; i < n_in; ++i) {
      resample[3 * i] = p.in[i].mode;
      resample[3 * i + 1] = p.in[i].pad_t;
      resample[3 * i + 2] = p.in[i].pad_l;
    }
  return return_planes(op, op.elems(), out, out_hi, out_lo);
}

// MBConv's squeeze-excite: the gate, and with the projection's master weight the folded weight (se_gate_launch); without
// it the gate of B images (se_squeeze_launch + se_excite_launch).
int b2_op_mbconv_se(int device, const float* x, const float* w1, const float* b1, const float* w2, const float* b2,
                    const float* w, int B, int HW, int Cpad, int Creal, int nr, int rows, int split, float* gate,
                    float* w_out, uint16_t* w_hi, uint16_t* w_lo) {
  B2_CHECK(x && w1 && b1 && w2 && b2 && gate && (!w || w_out), "b2_op_mbconv_se: null argument");
  B2_CHECK(B >= 1 && HW >= 1 && Cpad >= 64 && Cpad % 64 == 0 && Creal >= 1 && Creal <= Cpad && nr >= 1 &&
               nr <= se_max_nr(),
           "b2_op_mbconv_se: needs Cpad a multiple of 64, 1 <= Creal <= Cpad and 1 <= nr <= se_max_nr()");
  B2_CHECK(!w || (B == 1 && rows >= 1), "b2_op_mbconv_se: the weight fold takes one image and at least one row");
  B2_CUDA(cudaSetDevice(device));
  const bool sp = split != 0;
  Arena a;
  const Planes xp = a.planes(B, HW, 1, Cpad, sp);
  const Planes wp = w ? a.planes(1, rows, 1, Cpad, sp) : Planes();
  float* partial = a.alloc<float>(static_cast<size_t>(B) * se_chunks(HW) * Cpad);
  float* r_part = a.alloc<float>(static_cast<size_t>(B) * se_fc1_parts() * se_max_nr());
  float* g = a.alloc<float>(static_cast<size_t>(B) * Cpad);
  float* d_w1 = upload_f32(a, w1, static_cast<size_t>(Creal) * nr);
  float* d_b1 = upload_f32(a, b1, nr);
  float* d_w2 = upload_f32(a, w2, static_cast<size_t>(nr) * Creal);
  float* d_b2 = upload_f32(a, b2, Creal);
  float* d_w = upload_f32(a, w, static_cast<size_t>(rows) * Cpad);
  B2_CHECK(xp.hi && (!w || (wp.hi && d_w)) && partial && r_part && g && d_w1 && d_b1 && d_w2 && d_b2,
           "b2_op_mbconv_se: out of device memory");
  if (upload_planes(x, xp.hi, xp.lo, xp.elems(), nullptr)) return -1;
  if (w) {
    if (se_gate_launch(xp.hi, xp.lo, 1, HW, Cpad, Creal, nr, partial, r_part, d_w1, d_b1, d_w2, d_b2, g, d_w, rows, wp.hi,
                       wp.lo, nullptr))
      return -1;
  } else if (se_squeeze_launch(xp.hi, xp.lo, B, HW, Cpad, partial, nullptr) ||
             se_excite_launch(partial, B, HW, Cpad, Creal, nr, r_part, d_w1, d_b1, d_w2, d_b2, 0, g, nullptr, 0, nullptr,
                              nullptr, nullptr)) {
    return -1;
  }
  B2_CUDA(cudaDeviceSynchronize());
  B2_CUDA(cudaMemcpy(gate, g, static_cast<size_t>(B) * Cpad * sizeof(float), cudaMemcpyDeviceToHost));
  return w ? return_planes(wp, wp.elems(), w_out, w_hi, w_lo) : 0;
}

// OSNet's ChannelGate over an OSBlock's four streams and their gated sum, as reid_engine.cu runs them.
int b2_op_channel_gate(int device, const float* s, const float* w1, const float* b1, const float* w2, const float* b2,
                       const float* gates_in, int B, int HW, int C, int Creal, int Cr, int split, float* gates_out,
                       float* out, uint16_t* out_hi, uint16_t* out_lo) {
  B2_CHECK(s && out && (gates_in || (w1 && b1 && w2 && b2)), "b2_op_channel_gate: null argument");
  B2_CHECK(B >= 1 && HW >= 1 && C >= 64 && C % 64 == 0 && Creal >= 1 && Creal <= C && Creal <= 512 && Cr >= 1 && Cr <= 64,
           "b2_op_channel_gate: needs C a multiple of 64, 1 <= Creal <= min(C, 512) and 1 <= Cr <= 64");
  B2_CUDA(cudaSetDevice(device));
  const bool sp = split != 0;
  const size_t n = static_cast<size_t>(B) * HW * C, ng = static_cast<size_t>(B) * 4 * C;
  Arena a;
  Planes sp4[4];
  for (int k = 0; k < 4; ++k) sp4[k] = a.planes(B, HW, 1, C, sp);
  const Planes op = a.planes(B, HW, 1, C, sp);
  float* pooled = a.alloc<float>(ng);
  float* gates = gates_in ? upload_f32(a, gates_in, ng) : a.alloc<float>(ng);
  float* d_w1 = upload_f32(a, w1, static_cast<size_t>(Cr) * Creal);
  float* d_b1 = upload_f32(a, b1, Cr);
  float* d_w2 = upload_f32(a, w2, static_cast<size_t>(Creal) * Cr);
  float* d_b2 = upload_f32(a, b2, Creal);
  B2_CHECK(sp4[0].hi && sp4[1].hi && sp4[2].hi && sp4[3].hi && op.hi && pooled && gates &&
               (gates_in || (d_w1 && d_b1 && d_w2 && d_b2)),
           "b2_op_channel_gate: out of device memory");
  for (int k = 0; k < 4; ++k)
    if (upload_planes(s + k * n, sp4[k].hi, sp4[k].lo, n, nullptr)) return -1;
  if (!gates_in) {
    for (int k = 0; k < 4; ++k)
      if (gap_launch(sp4[k].hi, sp4[k].lo, B, HW, C, pooled + static_cast<size_t>(k) * C, 4 * C, nullptr)) return -1;
    if (gate_mlp_launch(pooled, B * 4, C, Creal, Cr, d_w1, d_b1, d_w2, d_b2, gates, nullptr)) return -1;
  }
  const __half* hi[4] = {sp4[0].hi, sp4[1].hi, sp4[2].hi, sp4[3].hi};
  const __half* lo[4] = {sp4[0].lo, sp4[1].lo, sp4[2].lo, sp4[3].lo};
  if (gated_sum4_launch(hi, lo, gates, B, HW, C, op.hi, op.lo, nullptr)) return -1;
  B2_CUDA(cudaDeviceSynchronize());
  if (gates_out) B2_CUDA(cudaMemcpy(gates_out, gates, ng * sizeof(float), cudaMemcpyDeviceToHost));
  return return_planes(op, n, out, out_hi, out_lo);
}

// EfficientNet's stem operand: 3x3/2 patches of the fp32 image as 64-channel pixels (stem_im2col_launch).
int b2_op_stem_im2col(int device, const float* img, int H, int W, int Ho, int Wo, int pad_t, int pad_l, int split,
                      float* out, uint16_t* out_hi, uint16_t* out_lo) {
  B2_CHECK(img && out, "b2_op_stem_im2col: null argument");
  B2_CHECK(H >= 1 && W >= 1 && Ho >= 1 && Wo >= 1 && pad_t >= 0 && pad_t < 3 && pad_l >= 0 && pad_l < 3,
           "b2_op_stem_im2col: needs positive sizes and pads in [0, 3)");
  B2_CUDA(cudaSetDevice(device));
  Arena a;
  const Planes op = a.planes(1, Ho, Wo, 64, split != 0);
  float* d_img = upload_f32(a, img, static_cast<size_t>(H) * W * 3);
  B2_CHECK(op.hi && d_img, "b2_op_stem_im2col: out of device memory");
  if (stem_im2col_launch(d_img, 1, H, W, Ho, Wo, pad_t, pad_l, op.hi, op.lo, nullptr)) return -1;
  B2_CUDA(cudaDeviceSynchronize());
  return return_planes(op, op.elems(), out, out_hi, out_lo);
}

// The ResNet stems' operand packs: the detector's compact 16-lane operand (stem_pack16_launch, layout 0) or the ReID
// engines' 64-lane operand (stem_pack_launch, layout 1).
int b2_op_stem_pack(int device, const void* img, int is_u8, int B, int H, int W, int layout, int Hu, int Wu, int split,
                    float* out, uint16_t* out_hi, uint16_t* out_lo) {
  B2_CHECK(img && out, "b2_op_stem_pack: null argument");
  B2_CHECK(layout == 0 || layout == 1, "b2_op_stem_pack: layout must be 0 (detector) or 1 (ReID)");
  B2_CHECK(layout == 0 || is_u8, "b2_op_stem_pack: the ReID layout takes uint8 crops only");
  B2_CHECK(B >= 1 && H >= 1 && W >= 1 && Hu >= 1 && Wu >= 1, "b2_op_stem_pack: needs positive sizes");
  const int lanes = layout == 0 ? 16 : 64;
  const size_t n_img = static_cast<size_t>(B) * H * W * 3;
  // the kernels index an image's pixels and an operand image's pixels with int
  B2_CHECK(static_cast<size_t>(H) * W <= INT_MAX && static_cast<size_t>(Hu) * Wu <= INT_MAX,
           "b2_op_stem_pack: frame or operand too large");
  B2_CUDA(cudaSetDevice(device));
  Arena a;
  const Planes op = a.planes(B, Hu, Wu, lanes, split != 0);
  uint8_t* d_img = a.alloc<uint8_t>(n_img * (is_u8 ? 1 : sizeof(float)));
  B2_CHECK(op.hi && d_img, "b2_op_stem_pack: out of device memory");
  B2_CUDA(cudaMemcpy(d_img, img, n_img * (is_u8 ? 1 : sizeof(float)), cudaMemcpyHostToDevice));
  const int rc = layout == 0 ? stem_pack16_launch(d_img, is_u8 != 0, B, H, W, op.hi, op.lo, Hu, Wu, nullptr)
                             : stem_pack_launch(d_img, B, H, W, op.hi, op.lo, Hu, Wu, nullptr);
  if (rc) return -1;
  B2_CUDA(cudaDeviceSynchronize());
  return return_planes(op, op.elems(), out, out_hi, out_lo);
}

// The distance GEMMs' operand conversion alone: cosine_normalize_rows (normalize != 0) or rows_to_planes.
int b2_op_distance_operand(int device, const float* x, int rows, int D, int ld, int normalize, float eps, uint16_t* out_hi,
                           uint16_t* out_lo, float* sqnorm, uint32_t* range_flag) {
  B2_CHECK(x && out_hi && out_lo, "b2_op_distance_operand: null argument");
  B2_CHECK(rows >= 1 && D >= 1 && ld >= D && eps >= 0.f, "b2_op_distance_operand: needs rows, D >= 1, ld >= D, eps >= 0");
  B2_CUDA(cudaSetDevice(device));
  const size_t n = static_cast<size_t>(rows) * ld;
  Arena a;
  __half *hi = a.alloc<__half>(n), *lo = a.alloc<__half>(n);
  float* d_x = upload_f32(a, x, static_cast<size_t>(rows) * D);
  float* d_sq = a.alloc<float>(rows);
  unsigned int* flag = a.alloc<unsigned int>(1);
  B2_CHECK(hi && lo && d_x && d_sq && flag, "b2_op_distance_operand: out of device memory");
  if (normalize ? cosine_normalize_rows(d_x, rows, D, eps, hi, lo, ld, nullptr)
                : rows_to_planes(d_x, rows, D, hi, lo, ld, d_sq, flag, nullptr))
    return -1;
  B2_CUDA(cudaDeviceSynchronize());
  B2_CUDA(cudaMemcpy(out_hi, hi, n * sizeof(__half), cudaMemcpyDeviceToHost));
  B2_CUDA(cudaMemcpy(out_lo, lo, n * sizeof(__half), cudaMemcpyDeviceToHost));
  if (sqnorm && !normalize) B2_CUDA(cudaMemcpy(sqnorm, d_sq, rows * sizeof(float), cudaMemcpyDeviceToHost));
  if (range_flag && !normalize) B2_CUDA(cudaMemcpy(range_flag, flag, sizeof(unsigned int), cudaMemcpyDeviceToHost));
  return 0;
}

// The distance GEMMs' epilogues alone, on host-given products: distance_finish (kind 0 cosine, 1 squared euclidean),
// cosine_segmin (kind 2) or pair_segmin (kind 3).
int b2_op_distance_epilogue(int device, int kind, const float* dots, int rows, int cols, int ld, const float* na2,
                            const float* nb2, const int32_t* seg_a, int n_a, const int32_t* seg_b, int n_b,
                            const uint8_t* gate, float fill, float* out) {
  B2_CHECK(dots && out, "b2_op_distance_epilogue: null argument");
  B2_CHECK(kind >= 0 && kind <= 3 && rows >= 1 && cols >= 1 && ld >= cols,
           "b2_op_distance_epilogue: needs kind 0..3, rows, cols >= 1 and ld >= cols");
  B2_CHECK((kind != 1 && kind != 3) || (na2 && nb2), "b2_op_distance_epilogue: the euclidean kinds need na2 and nb2");
  auto segs_ok = [](const int32_t* seg, int n, int limit) {
    if (!seg || n < 1 || seg[0] < 0) return false;
    for (int i = 0; i < n; ++i)
      if (seg[i + 1] < seg[i]) return false;
    return seg[n] <= limit;
  };
  B2_CHECK(kind < 2 || segs_ok(seg_a, n_a, rows), "b2_op_distance_epilogue: seg_a must be n_a + 1 non-decreasing row offsets "
                                                  "in [0, rows]");
  B2_CHECK(kind < 3 || segs_ok(seg_b, n_b, cols), "b2_op_distance_epilogue: seg_b must be n_b + 1 non-decreasing column "
                                                  "offsets in [0, cols]");
  B2_CUDA(cudaSetDevice(device));
  const size_t n_out = kind < 2 ? static_cast<size_t>(rows) * cols
                                : static_cast<size_t>(n_a) * (kind == 2 ? cols : n_b);
  Arena a;
  float* d_dots = upload_f32(a, dots, static_cast<size_t>(rows) * ld);
  float* d_na2 = upload_f32(a, na2, rows);
  float* d_nb2 = upload_f32(a, nb2, cols);
  int* d_seg = a.alloc<int>(static_cast<size_t>(n_a) + n_b + 2);
  uint8_t* d_gate = gate && kind == 3 ? a.alloc<uint8_t>(static_cast<size_t>(n_a) * n_b) : nullptr;
  float* d_out = a.alloc<float>(n_out);
  B2_CHECK(d_dots && (!na2 || d_na2) && (!nb2 || d_nb2) && d_seg && (!gate || kind != 3 || d_gate) && d_out,
           "b2_op_distance_epilogue: out of device memory");
  if (kind >= 2) B2_CUDA(cudaMemcpy(d_seg, seg_a, (n_a + 1) * sizeof(int), cudaMemcpyHostToDevice));
  if (kind == 3) B2_CUDA(cudaMemcpy(d_seg + n_a + 1, seg_b, (n_b + 1) * sizeof(int), cudaMemcpyHostToDevice));
  if (d_gate) B2_CUDA(cudaMemcpy(d_gate, gate, static_cast<size_t>(n_a) * n_b, cudaMemcpyHostToDevice));
  const int rc = kind < 2    ? distance_finish(d_dots, ld, rows, cols, kind, d_na2, d_nb2, d_out, nullptr)
                 : kind == 2 ? cosine_segmin(d_dots, ld, d_seg, n_a, cols, d_out, nullptr)
                             : pair_segmin(d_dots, ld, d_na2, d_nb2, d_seg, n_a, d_seg + n_a + 1, n_b, d_gate, fill, d_out,
                                           nullptr);
  if (rc) return -1;
  B2_CUDA(cudaDeviceSynchronize());
  B2_CUDA(cudaMemcpy(out, d_out, n_out * sizeof(float), cudaMemcpyDeviceToHost));
  return 0;
}

// The ReID crop resize alone (reid_crop_resize_launch).
int b2_op_reid_crop_resize(int device, const uint8_t* frames, int nf, int h, int w, const int32_t* boxes, int n, int out_h,
                           int out_w, uint8_t* out) {
  B2_CHECK(frames && boxes && out, "b2_op_reid_crop_resize: null argument");
  B2_CHECK(nf >= 1 && h >= 1 && w >= 1 && n >= 1, "b2_op_reid_crop_resize: needs nf, h, w, n >= 1");
  if (reid_boxes_check(boxes, n, nf, h, w, "b2_op_reid_crop_resize")) return -1;
  B2_CUDA(cudaSetDevice(device));
  const size_t nb_frames = static_cast<size_t>(nf) * h * w * 3, nb_out = static_cast<size_t>(n) * out_h * out_w * 3;
  Arena a;
  uint8_t* d_frames = a.alloc<uint8_t>(nb_frames, false);
  int32_t* d_boxes = a.alloc<int32_t>(static_cast<size_t>(n) * 5, false);
  uint8_t* d_out = a.alloc<uint8_t>(nb_out);
  B2_CHECK(d_frames && d_boxes && d_out, "b2_op_reid_crop_resize: out of device memory");
  B2_CUDA(cudaMemcpy(d_frames, frames, nb_frames, cudaMemcpyHostToDevice));
  B2_CUDA(cudaMemcpy(d_boxes, boxes, sizeof(int32_t) * 5 * n, cudaMemcpyHostToDevice));
  if (reid_crop_resize_launch(d_frames, h, w, d_boxes, n, d_out, out_h, out_w, nullptr)) return -1;
  B2_CUDA(cudaDeviceSynchronize());
  B2_CUDA(cudaMemcpy(out, d_out, nb_out, cudaMemcpyDeviceToHost));
  return 0;
}

// The resize alone (parity tests): host uint8 [n, src_h, src_w, 3] -> host float32 [n, dst_h, dst_w, 3].
int b2_resize_frames(int device, const uint8_t* frames_u8, int n, int src_h, int src_w, int dst_h, int dst_w,
                     float* out_host) {
  B2_CHECK(frames_u8 && out_host && n > 0 && src_h > 0 && src_w > 0 && dst_h > 0 && dst_w > 0, "b2_resize_frames: bad argument");
  B2_CUDA(cudaSetDevice(device));
  const size_t nb_src = static_cast<size_t>(n) * src_h * src_w * 3, nb_dst = static_cast<size_t>(n) * dst_h * dst_w * 3 * sizeof(float);
  Arena a;
  uint8_t* d_src = a.alloc<uint8_t>(nb_src, false);
  float* d_dst = a.alloc<float>(nb_dst / sizeof(float), false);
  B2_CHECK(d_src && d_dst, "b2_resize_frames: out of device memory");
  B2_CUDA(cudaMemcpy(d_src, frames_u8, nb_src, cudaMemcpyHostToDevice));
  if (resize_u8_launch(d_src, n, src_h, src_w, d_dst, dst_h, dst_w, nullptr)) return -1;
  B2_CUDA(cudaMemcpy(out_host, d_dst, nb_dst, cudaMemcpyDeviceToHost));
  return 0;
}

}  // extern "C"
