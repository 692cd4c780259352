// The per-call GEMM workspace (gemm_ws.h) and the tracker / ReID distance entry points that run on it.
#include <stdlib.h>

#include <algorithm>
#include <functional>
#include <mutex>

#include "../../include/b200det.h"
#include "gemm_ws.h"
#include "kernels.h"

namespace b2 {

GemmWs::~GemmWs() {
  if (!transient) return;
  release();
  if (stream) cudaStreamDestroy(stream);
}

void GemmWs::release() {
  plans.clear();
  void* ptrs[] = {d_a, d_b, d_dots, d_out, d_bias, d_na2, d_nb2, d_int, d_gate, d_range, a_hi, a_lo, b_hi, b_lo};
  for (void* q : ptrs) if (q) cudaFree(q);
  d_a = d_b = d_dots = d_out = d_bias = d_na2 = d_nb2 = nullptr;
  d_int = nullptr;
  d_gate = nullptr;
  d_range = nullptr;
  a_hi = a_lo = b_hi = b_lo = nullptr;
}

int GemmWs::reserve(int device, const GemmNeed& need) {
  if (!stream) {
    B2_CUDA(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, device));
    B2_CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
  }
  size_t* c[] = {&cap.a, &cap.b, &cap.Sp, &cap.Np, &cap.Dp, &cap.out, &cap.ints, &cap.gate};
  const size_t n[] = {need.a, need.b, need.Sp, need.Np, need.Dp, need.out, need.ints, need.gate};
  bool fits = true;
  for (int i = 0; i < 8; ++i) fits = fits && n[i] <= *c[i];
  if (fits) {
    B2_CUDA(cudaMemsetAsync(d_range, 0, sizeof(unsigned int), stream));
    return 0;
  }
  B2_CUDA(cudaStreamSynchronize(stream));
  release();
  for (int i = 0; i < 8; ++i) *c[i] = std::max<size_t>(n[i] > *c[i] ? n[i] * (transient ? 1 : 2) : *c[i], 1);
  B2_CUDA(cudaMalloc(&d_a, cap.a * 4));
  B2_CUDA(cudaMalloc(&d_b, cap.b * 4));
  B2_CUDA(cudaMalloc(&d_dots, cap.Sp * cap.Np * 4));
  B2_CUDA(cudaMalloc(&d_out, cap.out * 4));
  B2_CUDA(cudaMalloc(&d_bias, cap.Np * 4));
  B2_CUDA(cudaMalloc(&d_na2, cap.Sp * 4));
  B2_CUDA(cudaMalloc(&d_nb2, cap.Np * 4));
  B2_CUDA(cudaMalloc(&d_int, cap.ints * 4));
  B2_CUDA(cudaMalloc(&d_gate, cap.gate));
  B2_CUDA(cudaMalloc(&d_range, sizeof(unsigned int)));
  B2_CUDA(cudaMemsetAsync(d_range, 0, sizeof(unsigned int), stream));
  B2_CUDA(cudaMalloc(&a_hi, cap.Sp * cap.Dp * 2));
  B2_CUDA(cudaMalloc(&a_lo, cap.Sp * cap.Dp * 2));
  B2_CUDA(cudaMalloc(&b_hi, cap.Np * cap.Dp * 2));
  B2_CUDA(cudaMalloc(&b_lo, cap.Np * cap.Dp * 2));
  B2_CUDA(cudaMemsetAsync(d_bias, 0, cap.Np * 4, stream));
  B2_CUDA(cudaMemsetAsync(d_na2, 0, cap.Sp * 4, stream));
  B2_CUDA(cudaMemsetAsync(d_nb2, 0, cap.Np * 4, stream));
  B2_CUDA(cudaMemsetAsync(a_hi, 0, cap.Sp * cap.Dp * 2, stream));
  B2_CUDA(cudaMemsetAsync(a_lo, 0, cap.Sp * cap.Dp * 2, stream));
  B2_CUDA(cudaMemsetAsync(b_hi, 0, cap.Np * cap.Dp * 2, stream));
  B2_CUDA(cudaMemsetAsync(b_lo, 0, cap.Np * cap.Dp * 2, stream));
  B2_CUDA(cudaStreamSynchronize(stream));
  return 0;
}

int GemmWs::gemm(int Sp, int Np, int Dp, bool split) {
  const std::vector<int> key = {Sp, Np, Dp, split ? 1 : 0};
  auto it = plans.find(key);
  if (it == plans.end()) {
    ConvDesc d;
    d.B = 1; d.in_H = 1; d.in_W = Sp; d.Cin = Dp; d.in_pitch_H = 1; d.in_pitch_W = Sp; d.in_ld = Dp;
    d.Cout = Np; d.out_H = 1; d.out_W = Sp; d.ldc = Np;
    ConvWeights cw;
    cw.w_hi = b_hi; cw.w_lo = split ? b_lo : nullptr; cw.bias = d_bias; cw.Cout_pad = Np; cw.K = Dp;
    ConvIO io;
    io.in_hi = a_hi; io.in_lo = split ? a_lo : nullptr; io.out_f32 = d_dots;
    PlanPtr plan(conv_tc_plan_create(d, cw, io, split, num_sms));
    B2_CHECK(plan != nullptr, std::string("GEMM workspace plan: ") + last_error());
    it = plans.emplace(key, std::move(plan)).first;
  }
  return conv_tc_launch(it->second.get(), stream);
}

int GemmWs::download(float* out, size_t n, const char* who) {
  unsigned int range = 0;
  B2_CUDA(cudaMemcpyAsync(out, d_out, sizeof(float) * n, cudaMemcpyDeviceToHost, stream));
  B2_CUDA(cudaMemcpyAsync(&range, d_range, sizeof(unsigned int), cudaMemcpyDeviceToHost, stream));
  B2_CUDA(cudaStreamSynchronize(stream));
  B2_CHECK(range == 0, std::string(who) + ": input outside the fp16-plane range (a finite |x| >= 65520 rounds to inf in "
                       "the GEMM operand's hi plane); scale the embeddings down");
  return 0;
}

namespace {

// b2_cosine_cost / b2_distance_matrix are called once per frame (per cascade level) by the trackers: a call is three
// uploads, four launches and one download on the workspace's stream.  B2_NO_WS=1 (test hook) runs every call in a private
// workspace that is released when the call returns -- same code, no reuse; tests compare the two bit for bit.

std::map<int, GemmWs> g_dist_ws;   // the trackers' workspaces, one per device
std::mutex g_dist_ws_mutex;        // one call at a time per process (the trackers are single-threaded per stream)

// Runs `run` on the device's workspace, or on a private one under B2_NO_WS.
int on_dist_ws(int device, const std::function<int(GemmWs&)>& run) {
  std::lock_guard<std::mutex> lock(g_dist_ws_mutex);
  if (getenv("B2_NO_WS") != nullptr) {
    GemmWs w;
    w.transient = true;
    return run(w);
  }
  return run(g_dist_ws[device]);
}

// a [na][D] x b [nb][D] on the workspace, metric 0 cosine / 1 squared euclidean: the distance matrix [na][nb], or with
// `seg` ([T + 1] offsets of a's rows) the per-segment minimum of the cosine distance [T][nb].  Cosine rows are divided by
// max(|x|, eps).
int distance_run(GemmWs& w, int device, const float* a, int na, const float* b, int nb, int D, int metric, float eps,
                 bool split, const int32_t* seg, int T, float* out, const char* who) {
  const int Dp = (D + 63) / 64 * 64, Np = (nb + 15) / 16 * 16, Sp = (na + 127) / 128 * 128, rows = seg ? T : na;
  GemmNeed need;
  need.a = static_cast<size_t>(na) * D; need.b = static_cast<size_t>(nb) * D;
  need.Sp = Sp; need.Np = Np; need.Dp = Dp;
  need.out = static_cast<size_t>(rows) * nb; need.ints = seg ? T + 1 : 0;
  if (w.reserve(device, need)) return -1;
  cudaStream_t st = w.stream;
  B2_CUDA(cudaMemcpyAsync(w.d_a, a, sizeof(float) * na * D, cudaMemcpyHostToDevice, st));
  B2_CUDA(cudaMemcpyAsync(w.d_b, b, sizeof(float) * nb * D, cudaMemcpyHostToDevice, st));
  if (seg) B2_CUDA(cudaMemcpyAsync(w.d_int, seg, sizeof(int) * (T + 1), cudaMemcpyHostToDevice, st));
  if (metric == 0) {
    if (cosine_normalize_rows(w.d_a, na, D, eps, w.a_hi, w.a_lo, Dp, st) ||
        cosine_normalize_rows(w.d_b, nb, D, eps, w.b_hi, w.b_lo, Dp, st))
      return -1;
  } else {
    if (rows_to_planes(w.d_a, na, D, w.a_hi, w.a_lo, Dp, w.d_na2, w.d_range, st) ||
        rows_to_planes(w.d_b, nb, D, w.b_hi, w.b_lo, Dp, w.d_nb2, w.d_range, st))
      return -1;
  }
  if (w.gemm(Sp, Np, Dp, split)) return -1;
  if (seg ? cosine_segmin(w.d_dots, Np, w.d_int, T, nb, w.d_out, st)
          : distance_finish(w.d_dots, Np, na, nb, metric, w.d_na2, w.d_nb2, w.d_out, st))
    return -1;
  return w.download(out, static_cast<size_t>(rows) * nb, who);
}

}  // namespace
}  // namespace b2

using namespace b2;

extern "C" {

// ---- DeepSORT appearance cost ---------------------------------------------------------------
int b2_cosine_cost(int device, const float* gallery, const int32_t* seg_offsets, int T, const float* dets, int N,
                   int D, int precision, float* cost) {
  B2_CHECK(gallery && seg_offsets && dets && cost, "b2_cosine_cost: null argument");
  if (T <= 0 || N <= 0) return 0;
  B2_CHECK(D > 0 && seg_offsets[0] == 0, "b2_cosine_cost: seg_offsets must start at 0");
  for (int t = 0; t < T; ++t)
    B2_CHECK(seg_offsets[t + 1] >= seg_offsets[t], "b2_cosine_cost: seg_offsets must be non-decreasing");
  B2_CHECK(seg_offsets[T] > 0, "b2_cosine_cost: empty gallery");
  B2_CUDA(cudaSetDevice(device));
  const bool split = precision == 1;
  return on_dist_ws(device, [&](GemmWs& w) {
    return distance_run(w, device, gallery, seg_offsets[T], dets, N, D, 0, 0.f, split, seg_offsets, T, cost, "b2_cosine_cost");
  });
}

// ---- distance matrix (torchreid/distance.py:6-80) ------------------------------------------------
int b2_distance_matrix(int device, const float* a, int na, const float* b, int nb, int D, int metric, int precision,
                       float* out) {
  B2_CHECK(a && b && out, "b2_distance_matrix: null argument");
  B2_CHECK(metric == 0 || metric == 1, "b2_distance_matrix: metric must be 0 (cosine) or 1 (squared euclidean)");
  if (na <= 0 || nb <= 0) return 0;
  B2_CHECK(D > 0, "b2_distance_matrix: D must be positive");
  B2_CUDA(cudaSetDevice(device));
  const bool split = precision == 1;
  return on_dist_ws(device, [&](GemmWs& w) {
    return distance_run(w, device, a, na, b, nb, D, metric, 1e-12f, split, nullptr, 0, out, "b2_distance_matrix");
  });
}

}  // extern "C"
