// Host-side core shared by the three engines (see engine_core.h).
#include <math.h>
#include <stdio.h>

#include "../../include/b200det.h"
#include "engine_core.h"
#include "kernels.h"

namespace b2 {

static thread_local std::string g_err;
void set_error(const std::string& msg) { g_err = msg; }
const char* last_error() { return g_err.c_str(); }

Arena::~Arena() {
  for (void* p : ptrs_) cudaFree(p);
}

void* Arena::raw(size_t bytes, bool zero) {
  void* p = nullptr;
  requested_ += bytes + 256;
  if (cudaMalloc(&p, bytes + 256) != cudaSuccess) {
    cudaGetLastError();   // an out-of-memory result is not sticky: keep it from surfacing at a later launch check
    failed_ += bytes + 256;
    return nullptr;
  }
  if (zero) cudaMemset(p, 0, bytes + 256);
  ptrs_.push_back(p);
  return p;
}

Planes Arena::planes(int B, int H, int W, int C, bool split, int creal) {
  Planes p;
  p.B = B; p.H = H; p.W = W; p.C = C; p.creal = creal;
  p.hi = alloc<__half>(p.elems());
  p.lo = split ? alloc<__half>(p.elems()) : nullptr;
  if (split && !p.lo) p.hi = nullptr;
  return p;
}

std::unique_ptr<ConvLayer> make_conv(Arena& a, bool split, const std::string& name, ConvDesc d, const Planes& in,
                                     const Planes& out, const Planes* res, float* out_f32, int ldc_f32,
                                     bool dense_groups, const ConvWeights* shared) {
  std::unique_ptr<ConvLayer> L(new ConvLayer());
  L->name = name;
  d.B = in.B; d.Cin = in.C;
  if (d.in_H == 0) { d.in_H = in.H; d.in_W = in.W; }
  d.in_pitch_H = in.H; d.in_pitch_W = in.W;
  if (d.in_ld == 0) d.in_ld = in.C;
  if (out_f32) {
    d.out_H = d.Ho(); d.out_W = d.Wo(); d.ldc = ldc_f32;
  } else {
    d.out_H = out.H; d.out_W = out.W; d.ldc = out.C;
  }
  if (res) { d.res_H = res->H; d.res_W = res->W; d.ldr = res->C; }
  L->d = d;
  L->w.Cout_pad = (d.Cout + 15) / 16 * 16;
  L->w.K = d.R * d.S * (d.groups > 1 && !dense_groups ? kGroupWindow : in.C);
  if (shared && shared->K == L->w.K && shared->Cout_pad == L->w.Cout_pad) {
    L->w = *shared;
  } else if (!shared) {
    L->w.w_hi = a.alloc<__half>(static_cast<size_t>(L->w.Cout_pad) * L->w.K);
    L->w.w_lo = split ? a.alloc<__half>(static_cast<size_t>(L->w.Cout_pad) * L->w.K) : nullptr;
    L->w.bias = a.alloc<float>(L->w.Cout_pad);
  }   // a mismatched `shared` leaves the weights null: plan_convs refuses the layer
  L->io.in_hi = in.hi; L->io.in_lo = in.lo;
  L->io.out_hi = out.hi; L->io.out_lo = out.lo; L->io.out_f32 = out_f32;
  if (res) { L->io.res_hi = res->hi; L->io.res_lo = res->lo; }
  return L;
}

int plan_convs(const std::vector<std::unique_ptr<ConvLayer>>& layers, bool split, int num_sms) {
  for (auto& L : layers) {
    B2_CHECK(L->w.w_hi && L->w.bias && (!split || L->w.w_lo), "out of device memory (weights of " + L->name + ")");
    L->plan.reset(conv_tc_plan_create(L->d, L->w, L->io, split, num_sms));
    if (!L->plan) {
      set_error("plan for " + L->name + ": " + last_error());
      return -1;
    }
  }
  return 0;
}

WeightSet::WeightSet(const char* const* names, const float* const* data, const int64_t* numel, int n) {
  for (int i = 0; i < n; ++i) m[names[i]] = std::make_pair(data[i], numel[i]);
}

const float* WeightSet::get(const std::string& n, int64_t expect) const {
  auto it = m.find(n);
  if (it == m.end()) { set_error("missing weight: " + n); return nullptr; }
  if (it->second.second != expect) {
    set_error("weight " + n + ": expected " + std::to_string(expect) + " values, got " + std::to_string(it->second.second));
    return nullptr;
  }
  return it->second.first;
}

int fold_bn(const WeightSet& ws, const std::string& scope, const BnNames& nm, double eps, int C, std::vector<double>& scale,
            std::vector<double>& shift) {
  scale.assign(C, 1.0);
  shift.assign(C, 0.0);
  if (scope.empty()) return 0;
  const float* g = ws.get(scope + nm.gamma, C);
  const float* b = ws.get(scope + nm.beta, C);
  const float* m = ws.get(scope + nm.mean, C);
  const float* v = ws.get(scope + nm.var, C);
  if (!g || !b || !m || !v) return -1;
  for (int i = 0; i < C; ++i) {
    scale[i] = static_cast<double>(g[i]) / sqrt(static_cast<double>(v[i]) + eps);
    shift[i] = static_cast<double>(b[i]) - static_cast<double>(m[i]) * scale[i];
  }
  return 0;
}

std::vector<float> fold_bias(const std::vector<double>& scale, const std::vector<double>& shift, const float* b, int Cout,
                             int Cout_pad) {
  std::vector<float> bias(Cout_pad, 0.f);
  for (int o = 0; o < Cout; ++o)
    bias[o] = static_cast<float>(b ? shift[o] + static_cast<double>(b[o]) * scale[o] : shift[o]);
  return bias;
}

void pack_grouped(const float* w, int RS, int Cin, int Cout, int groups, const double* scale, int K,
                  std::vector<float>& packed) {
  const int cg = Cin / groups, cgo = Cout / groups;
  const bool windowed = K != RS * Cin;
  const int kc = windowed ? kGroupWindow : Cin;   // input channels per tap in the packed row
  for (int o = 0; o < Cout; ++o) {
    // first input channel of o's group, relative to the channels o's packed row covers
    const int c0 = (o / cgo) * cg - (windowed ? o / kGroupWindow * kGroupWindow : 0);
    for (int t = 0; t < RS; ++t)
      for (int ci = 0; ci < cg; ++ci) {
        const float v = w[(static_cast<size_t>(t) * cg + ci) * Cout + o];
        packed[static_cast<size_t>(o) * K + static_cast<size_t>(t) * kc + c0 + ci] =
            scale ? static_cast<float>(v * scale[o]) : v;
      }
  }
}

namespace {

// Device scratch of one call, freed on every return path.
struct Scratch {
  void* p = nullptr;
  ~Scratch() { if (p) cudaFree(p); }
  float* f32() { return static_cast<float*>(p); }
};

}  // namespace

int upload_conv(const ConvLayer& L, const std::vector<float>& packed, const std::vector<float>& bias, cudaStream_t st) {
  const size_t n = packed.size();
  // the (hi, lo) operand planes are fp16: a folded weight beyond +-65504 (or a non-finite one) would become inf here and
  // NaN inside the MMA (inf * 0) -- refuse it at load time; activations are watched by the kernel's range monitor
  for (size_t i = 0; i < n; ++i)
    if (!(fabsf(packed[i]) <= 65504.f)) {
      set_error("weight of layer '" + L.name + "' outside the fp16-plane range (|w| > 65504 after BatchNorm folding, or not "
                "finite): this checkpoint is not representable in the (hi, lo) fp16 operand format");
      return -1;
    }
  for (size_t i = 0; i < bias.size(); ++i)
    if (!std::isfinite(bias[i])) {
      set_error("bias / folded BatchNorm shift of layer '" + L.name + "' is not finite");
      return -1;
    }
  Scratch tmp;
  B2_CUDA(cudaMalloc(&tmp.p, n * sizeof(float)));
  // same stream as the conversion kernel: a pageable cudaMemcpy on the legacy stream may return before its DMA lands,
  // and the engine streams are non-blocking (not ordered after the legacy stream)
  B2_CUDA(cudaMemcpyAsync(tmp.p, packed.data(), n * sizeof(float), cudaMemcpyHostToDevice, st));
  if (f32_to_planes(tmp.f32(), L.w.w_hi, L.w.w_lo, n, st)) return -1;
  if (L.w_master) B2_CUDA(cudaMemcpyAsync(L.w_master, tmp.p, n * sizeof(float), cudaMemcpyDeviceToDevice, st));
  B2_CUDA(cudaMemcpyAsync(L.w.bias, bias.data(), bias.size() * sizeof(float), cudaMemcpyHostToDevice, st));
  B2_CUDA(cudaStreamSynchronize(st));
  return 0;
}

int upload_planes(const float* host, __half* hi, __half* lo, size_t n, cudaStream_t st) {
  Scratch tmp;
  B2_CUDA(cudaMalloc(&tmp.p, n * sizeof(float)));
  B2_CUDA(cudaMemcpyAsync(tmp.p, host, n * sizeof(float), cudaMemcpyHostToDevice, st));
  if (f32_to_planes(tmp.f32(), hi, lo, n, st)) return -1;
  B2_CUDA(cudaStreamSynchronize(st));
  return 0;
}

int download_planes(const __half* hi, const __half* lo, size_t n, float* host, cudaStream_t st) {
  Scratch tmp;
  B2_CUDA(cudaMalloc(&tmp.p, n * sizeof(float)));
  if (planes_to_f32(hi, lo, tmp.f32(), n, st)) return -1;
  B2_CUDA(cudaMemcpyAsync(host, tmp.p, n * sizeof(float), cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  return 0;
}

Step& add_step(std::vector<Step>& steps, int phase, int kind, const std::string& name, std::function<int(cudaStream_t)> run,
               double bytes, double flops, int launches) {
  Step s;
  s.phase = phase;
  s.kind = kind;
  s.name = name;
  s.bytes = bytes;
  s.flops = flops;
  s.launches = launches;
  s.run = std::move(run);
  steps.push_back(std::move(s));
  return steps.back();
}

Step& add_conv_step(std::vector<Step>& steps, int phase, const ConvLayer* L) {
  return add_step(steps, phase, 0, L->name, [L](cudaStream_t st) { return conv_tc_launch(L->plan.get(), st); });
}

int open_device(int device, const char* who, int* num_sms, cudaStream_t* stream) {
  B2_CUDA(cudaSetDevice(device));
  cudaDeviceProp prop;
  B2_CUDA(cudaGetDeviceProperties(&prop, device));
  B2_CHECK(prop.major == 9 && prop.minor == 0, std::string(who) + ": this library is built for sm_90a (H100) only");
  *num_sms = prop.multiProcessorCount;
  B2_CUDA(cudaStreamCreateWithFlags(stream, cudaStreamNonBlocking));
  return 0;
}

int run_steps(const std::vector<Step>& steps, unsigned mask, cudaStream_t st) {
  for (const Step& s : steps)
    if ((mask >> s.phase) & 1u)
      if (s.run(st)) return -1;
  return 0;
}

int total_launches(const std::vector<Step>& steps) {
  int n = 0;
  for (const Step& s : steps) n += s.launches * (s.parts.empty() ? 1 : static_cast<int>(s.parts.size()));
  return n;
}

namespace {

struct Events {
  std::vector<cudaEvent_t> ev;
  ~Events() { for (cudaEvent_t e : ev) if (e) cudaEventDestroy(e); }
};

}  // namespace

int profile_steps(const std::vector<Step>& steps, cudaStream_t st, int reps, float* ms_out, int cap, int* n_out) {
  const int n = static_cast<int>(steps.size());
  B2_CHECK(cap >= n, "profile_steps: buffer too small");
  Events ev;
  ev.ev.assign(2 * n, nullptr);
  for (auto& e : ev.ev) B2_CUDA(cudaEventCreate(&e));
  std::vector<double> acc(n, 0.0);
  for (int r = 0; r < reps; ++r) {
    for (int i = 0; i < n; ++i) {
      B2_CUDA(cudaEventRecord(ev.ev[2 * i], st));
      if (steps[i].run(st)) return -1;
      B2_CUDA(cudaEventRecord(ev.ev[2 * i + 1], st));
    }
    B2_CUDA(cudaStreamSynchronize(st));
    for (int i = 0; i < n; ++i) {
      float ms = 0.f;
      B2_CUDA(cudaEventElapsedTime(&ms, ev.ev[2 * i], ev.ev[2 * i + 1]));
      acc[i] += ms;
    }
  }
  for (int i = 0; i < n; ++i) ms_out[i] = static_cast<float>(acc[i] / reps);
  *n_out = n;
  return 0;
}

int step_info(const std::vector<Step>& steps, int idx, char* name, int name_cap, double* flops, double* bytes, int* kind) {
  B2_CHECK(name && flops && bytes && kind, "step_info: null argument");
  B2_CHECK(idx >= 0 && idx < static_cast<int>(steps.size()), "step_info: index out of range");
  const Step& s = steps[idx];
  *kind = s.kind;
  *flops = s.flops;
  *bytes = s.bytes;
  snprintf(name, name_cap, "%s", s.name.c_str());
  return 0;
}

int capture_graph(cudaStream_t st, const std::function<int()>& enqueue, cudaGraphExec_t* out) {
  if (enqueue()) return -1;
  B2_CUDA(cudaStreamSynchronize(st));
  cudaGraph_t g = nullptr;
  B2_CUDA(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
  const int rc = enqueue();
  cudaError_t e = cudaStreamEndCapture(st, &g);
  if (rc) {
    if (g) cudaGraphDestroy(g);
    return -1;
  }
  B2_CUDA(e);
  e = cudaGraphInstantiate(out, g, 0);
  cudaGraphDestroy(g);
  B2_CUDA(e);
  return 0;
}

void StageMap::planes(const std::string& name, const Planes& p) {
  Stage s;
  s.kind = Stage::kPlanes;
  s.pl = p;
  s.shape[0] = p.B; s.shape[1] = p.H; s.shape[2] = p.W; s.shape[3] = p.C;
  m[name] = s;
}

void StageMap::raw(const std::string& name, void* ptr, Stage::Kind kind, int64_t a, int64_t b, int64_t c, int64_t d) {
  Stage s;
  s.kind = kind;
  s.ptr = ptr;
  s.shape[0] = a; s.shape[1] = b; s.shape[2] = c; s.shape[3] = d;
  m[name] = s;
}

const Stage* StageMap::find(const std::string& name) const {
  auto it = m.find(name);
  if (it == m.end()) {
    set_error("unknown stage: " + name);
    return nullptr;
  }
  return &it->second;
}

int stage_read(const Stage& s, cudaStream_t st, void* dst) {
  const size_t n = static_cast<size_t>(s.numel());
  B2_CUDA(cudaStreamSynchronize(st));
  if (s.kind == Stage::kPlanes) return download_planes(s.pl.hi, s.pl.lo, n, static_cast<float*>(dst), st);
  B2_CUDA(cudaMemcpyAsync(dst, s.ptr, n * 4, cudaMemcpyDeviceToHost, st));
  B2_CUDA(cudaStreamSynchronize(st));
  return 0;
}

int stage_write(const Stage& s, cudaStream_t st, const void* src) {
  const size_t n = static_cast<size_t>(s.numel());
  B2_CUDA(cudaStreamSynchronize(st));
  if (s.kind == Stage::kPlanes) return upload_planes(static_cast<const float*>(src), s.pl.hi, s.pl.lo, n, st);
  B2_CUDA(cudaMemcpyAsync(s.ptr, src, n * 4, cudaMemcpyHostToDevice, st));
  B2_CUDA(cudaStreamSynchronize(st));
  return 0;
}

int stage_get(const StageMap& stages, const char* name, cudaStream_t st, void* dst, int64_t capacity, int64_t shape[4],
              const char* who) {
  const Stage* s = stages.find(name);
  if (!s) return -1;
  for (int i = 0; i < 4; ++i) shape[i] = s->shape[i];
  B2_CHECK(capacity >= s->numel() * 4, std::string(who) + ": buffer too small");
  return stage_read(*s, st, dst);
}

}  // namespace b2

extern "C" {
const char* b2_last_error(void) { return b2::last_error(); }
int b2_version(void) { return 1; }
}  // extern "C"
