// Host-side core shared by the detector, ReID and EfficientDet engines: activation planes, the device arena, conv-layer
// records, weight lookup / BatchNorm folding / upload, the step list with its graph capture and per-step profiling, and
// stage readback.
#pragma once
#include <stdint.h>

#include <functional>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "common.h"

namespace b2 {

// Activation tensor in HBM: NHWC, fp16 "hi" plane plus (in split precision) an fp16 "lo" plane that holds
// (x - hi) * 2048, so x ~= hi + lo / 2048 to ~22 significant bits.  C is the stored (padded) channel count; creal the
// model's own count where the engine pads channels (EfficientDet), else 0.
struct Planes {
  __half* hi = nullptr;
  __half* lo = nullptr;   // nullptr when precision == fp16
  int B = 0, H = 0, W = 0, C = 0, creal = 0;
  size_t elems() const { return static_cast<size_t>(B) * H * W * C; }
  // images [b0, b0 + n): offsets follow this buffer's own H x W x C
  Planes images(int b0, int n) const {
    const size_t off = static_cast<size_t>(b0) * H * W * C;
    Planes p = *this;
    p.B = n;
    p.hi = hi ? hi + off : nullptr;
    p.lo = lo ? lo + off : nullptr;
    return p;
  }
};

// Owns device allocations; frees them when it goes away.  Every allocation carries 256 bytes of slack (vector loads and
// TMA boxes may touch past the last element) and is zero-filled on the legacy stream unless `zero` is false: a buffer
// allocated after the engine's streams have started work needs a device synchronise before its first use.
class Arena {
 public:
  Arena() = default;
  Arena(const Arena&) = delete;
  Arena& operator=(const Arena&) = delete;
  ~Arena();
  template <typename T>
  T* alloc(size_t n, bool zero = true) {
    return static_cast<T*>(raw(n * sizeof(T), zero));
  }
  // hi (+ lo in split precision) planes of B x H x W x C; hi == nullptr when out of memory
  Planes planes(int B, int H, int W, int C, bool split, int creal = 0);
  size_t requested() const { return requested_; }   // bytes asked for so far, failed requests included
  size_t failed() const { return failed_; }         // bytes of the requests that could not be allocated

 private:
  void* raw(size_t bytes, bool zero);
  std::vector<void*> ptrs_;
  size_t requested_ = 0, failed_ = 0;
};

struct PlanDeleter {
  void operator()(ConvPlan* p) const { conv_tc_plan_destroy(p); }
};
using PlanPtr = std::unique_ptr<ConvPlan, PlanDeleter>;

// One implicit-GEMM conv (or dense layer) of an engine: geometry, packed weights, operands and its tensor-core plans.
struct ConvLayer {
  std::string name;                 // checkpoint name (or scope) of the weights, used in error messages and step names
  std::string bn, bias;             // BatchNorm scope and bias name in the checkpoint, "" = none
  int layout = 0;                   // the engine's packing of the checkpoint weight
  int cin_real = 0;                 // input channels of the model (<= d.Cin where the engine pads channels)
  ConvDesc d;
  ConvWeights w;
  ConvIO io;
  PlanPtr plan;
  std::vector<PlanPtr> part_plan;   // the same layer over each part of the batch (detector's multi-stream passes)
  float* w_master = nullptr;        // optional fp32 copy of the packed weights, written by upload_conv
};

// Completes `d` for input `in` (d.in_H / d.in_W are the view, 0 = the whole buffer; d.in_ld 0 = in.C) writing `out`
// planes, or fp32 rows of stride `ldc_f32` into `out_f32` when that is set, plus `res` when given, and allocates the packed
// weights [Cout_pad][R*S*Cin] (a grouped conv: [Cout_pad][R*S*kGroupWindow], or with `dense_groups` the dense
// block-diagonal expansion the CUDA-core kernel reads).  Caller fills R, S, stride, dilation, pads, Cout, groups,
// epilogue and placement in `d`.
// With `shared` the layer runs those packed weights (another layer's, of the same K and Cout) and allocates none.
std::unique_ptr<ConvLayer> make_conv(Arena& a, bool split, const std::string& name, ConvDesc d, const Planes& in,
                                     const Planes& out, const Planes* res = nullptr, float* out_f32 = nullptr,
                                     int ldc_f32 = 0, bool dense_groups = false, const ConvWeights* shared = nullptr);
// Creates the full-batch plan of every layer.
int plan_convs(const std::vector<std::unique_ptr<ConvLayer>>& layers, bool split, int num_sms);

// A checkpoint as the caller passed it: name -> (data, element count).
struct WeightSet {
  std::map<std::string, std::pair<const float*, int64_t>> m;
  WeightSet() = default;
  WeightSet(const char* const* names, const float* const* data, const int64_t* numel, int n);
  void add(const std::string& n, const float* data, int64_t numel) { m[n] = std::make_pair(data, numel); }
  const float* get(const std::string& n, int64_t expect) const;   // nullptr + error when missing or of another size
  bool has(const std::string& n) const { return m.count(n) != 0; }
};

// Parameter names of a BatchNorm scope.
struct BnNames {
  const char *gamma, *beta, *mean, *var;
};
constexpr BnNames kTensorpackBn = {"/gamma", "/beta", "/mean/EMA", "/variance/EMA"};
constexpr BnNames kKerasBn = {"/gamma", "/beta", "/moving_mean", "/moving_variance"};
constexpr BnNames kTorchBn = {".weight", ".bias", ".running_mean", ".running_var"};

// Inference BatchNorm of `scope` as a per-channel scale / shift in double.  An empty scope is the identity.
int fold_bn(const WeightSet& ws, const std::string& scope, const BnNames& nm, double eps, int C, std::vector<double>& scale,
            std::vector<double>& shift);
// The epilogue bias of a conv whose output is BN(Wx + b): shift + b * scale (b may be null), Cout_pad entries.
std::vector<float> fold_bias(const std::vector<double>& scale, const std::vector<double>& shift, const float* b, int Cout,
                             int Cout_pad);

// A grouped conv's HWIO weight [R*S][Cin/groups][Cout], each output column o times scale[o] (scale may be null), into
// `packed` [Cout_pad][K] (zero elsewhere): K = R*S*kGroupWindow packs each 64-column window's diagonal group blocks
// (conv_tc), K = R*S*Cin the dense block-diagonal expansion (conv_simt).
void pack_grouped(const float* w, int RS, int Cin, int Cout, int groups, const double* scale, int K,
                  std::vector<float>& packed);

// Packed fp32 weights [Cout_pad][K] -> the layer's operand planes (and w_master), bias -> the layer's bias.  Refuses a
// weight the fp16 planes cannot represent and a non-finite bias.
int upload_conv(const ConvLayer& L, const std::vector<float>& packed, const std::vector<float>& bias, cudaStream_t st);
// Host fp32 -> device planes (n elements), and back.
int upload_planes(const float* host, __half* hi, __half* lo, size_t n, cudaStream_t st);
int download_planes(const __half* hi, const __half* lo, size_t n, float* host, cudaStream_t st);

// One entry of an engine's launch sequence.
struct Step {
  int phase = 0;
  int kind = 0;                 // the kind the engine's step-info call reports (0 = tensor-core conv)
  std::string name;
  double flops = 0, bytes = 0;  // algorithmic FLOPs, HBM bytes (operands once, at the stored precision)
  int launches = 1;
  std::function<int(cudaStream_t)> run;
  std::vector<std::function<int(cudaStream_t)>> parts;   // the step over each part of the batch (detector phases 0-2)
};
// Appends a step; the caller may add per-part launches to the returned step.
Step& add_step(std::vector<Step>& steps, int phase, int kind, const std::string& name, std::function<int(cudaStream_t)> run,
               double bytes = 0, double flops = 0, int launches = 1);
Step& add_conv_step(std::vector<Step>& steps, int phase, const ConvLayer* L);   // kind 0, launches L's plan
// Makes `device` current, checks it is an sm_90 part, reports its SM count and creates the engine's non-blocking stream.
int open_device(int device, const char* who, int* num_sms, cudaStream_t* stream);

// Runs the steps whose phase bit is set in `mask`.
int run_steps(const std::vector<Step>& steps, unsigned mask, cudaStream_t st);
int total_launches(const std::vector<Step>& steps);
// Per-step CUDA-event timing of eager launches, averaged over reps.
int profile_steps(const std::vector<Step>& steps, cudaStream_t st, int reps, float* ms_out, int cap, int* n_out);
int step_info(const std::vector<Step>& steps, int idx, char* name, int name_cap, double* flops, double* bytes, int* kind);
// Runs `enqueue` eagerly once (one-time lazy setup must not happen inside a capture), then captures it into `*out`.
int capture_graph(cudaStream_t st, const std::function<int()>& enqueue, cudaGraphExec_t* out);

// A named tensor the engine exposes for inspection: activation planes, or raw fp32 / int32 rows.
struct Stage {
  enum Kind { kPlanes = 0, kF32 = 1, kI32 = 2 } kind = kPlanes;
  Planes pl;
  void* ptr = nullptr;
  int64_t shape[4] = {1, 1, 1, 1};
  int64_t numel() const { return shape[0] * shape[1] * shape[2] * shape[3]; }
};
struct StageMap {
  std::map<std::string, Stage> m;
  void planes(const std::string& name, const Planes& p);
  void raw(const std::string& name, void* ptr, Stage::Kind kind, int64_t a, int64_t b, int64_t c, int64_t d);
  const Stage* find(const std::string& name) const;   // nullptr + error when unknown
};
// As fp32 / int32 (4 bytes per element) to host memory; waits for the stream first.
int stage_read(const Stage& s, cudaStream_t st, void* dst);
int stage_write(const Stage& s, cudaStream_t st, const void* src);
// Stage `name` of `stages` into dst (capacity bytes) with its shape; `who` names the calling entry point in errors.
int stage_get(const StageMap& stages, const char* name, cudaStream_t st, void* dst, int64_t capacity, int64_t shape[4],
              const char* who);

}  // namespace b2
