// Multi-camera ReID track-pair costs (BASELINE config 5): for a pair of cameras, the appearance cost of every
// (track of camera 1, track of camera 2) pair = min over the tracks' crop embeddings of the squared euclidean distance,
// gated by the spatial (top-down trajectory) distance.
//
// Reference (Python loops, one sklearn euclidean_distances call per track pair): multi_video_reid.py:308-324
// compute_feature_dist, :260-305 compute_spatial_dist; the assignment that follows (:512) is b2_lapjv (csrc/tmot.cpp).
// Here: ONE tensor-core GEMM over the concatenated galleries ([Sa,D] x [Sb,D]^T on conv_tc_kernel) and one segmented
// min kernel; the trajectory distance is plain host code (float64, as the reference).
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <map>
#include <mutex>
#include <vector>

#include "../../include/b200det.h"
#include "gemm_ws.h"
#include "kernels.h"

namespace b2 {
namespace {

// One workspace per device (the pair costs of config 5 are computed pair after pair with similar shapes), apart from the
// trackers' so that the two kinds of callers do not wait on each other.
std::map<int, GemmWs> g_pair_ws;
std::mutex g_pair_mutex;

}  // namespace
}  // namespace b2

using namespace b2;

extern "C" {

// Shared body: `a` / `b` are host pointers (a_dev == 0: uploaded first) or device pointers -- b may be PEER memory of
// another GPU opened through b2_gallery_open: rows_to_planes then reads it over NVLink while converting to the fp16 operand
// planes, i.e. the "exchange" is the operand load of the GEMM's first stage, no staged copy of the peer gallery exists.
// Operand rows beyond Sa / Sb (padding up to the plan's shape) hold leftovers of earlier calls, NaN or inf included: they
// only produce products nobody reads.
static int pair_cost_impl(int device, const float* a, bool a_dev, const int32_t* seg_a, int N, const float* b, bool b_dev,
                          const int32_t* seg_b, int M, int D, const uint8_t* gate, float fill, int precision, float* out) {
  B2_CHECK(N >= 0 && M >= 0 && D > 0, "b2_track_pair_cost: bad argument");
  if (N == 0 || M == 0) return 0;
  B2_CHECK(a && seg_a && b && seg_b && out, "b2_track_pair_cost: null argument");
  const int Sa = seg_a[N], Sb = seg_b[M];
  B2_CHECK(seg_a[0] == 0 && seg_b[0] == 0, "b2_track_pair_cost: segment offsets must start at 0");
  for (int i = 0; i < N; ++i) B2_CHECK(seg_a[i + 1] >= seg_a[i], "b2_track_pair_cost: seg_a not monotone");
  for (int j = 0; j < M; ++j) B2_CHECK(seg_b[j + 1] >= seg_b[j], "b2_track_pair_cost: seg_b not monotone");
  if (Sa == 0 || Sb == 0) {
    for (size_t k = 0; k < static_cast<size_t>(N) * M; ++k) out[k] = fill;
    return 0;
  }
  B2_CUDA(cudaSetDevice(device));
  const bool split = precision == 1;
  const int Dp = (D + 63) / 64 * 64, Np = (Sb + 15) / 16 * 16, Sp = (Sa + 127) / 128 * 128;
  std::lock_guard<std::mutex> lock(g_pair_mutex);
  GemmWs own;   // B2_NO_WS=1 (test hook): a private workspace per call, as for b2_distance_matrix
  own.transient = true;
  GemmWs& w = getenv("B2_NO_WS") != nullptr ? own : g_pair_ws[device];
  GemmNeed need;
  need.a = a_dev ? 0 : static_cast<size_t>(Sa) * D;
  need.b = b_dev ? 0 : static_cast<size_t>(Sb) * D;
  need.Sp = Sp; need.Np = Np; need.Dp = Dp;
  need.out = static_cast<size_t>(N) * M;
  need.ints = static_cast<size_t>(N) + M + 2;
  need.gate = static_cast<size_t>(N) * M;
  if (w.reserve(device, need)) return -1;
  cudaStream_t st = w.stream;
  const float* d_a = a;
  const float* d_b = b;
  if (!a_dev) {
    B2_CUDA(cudaMemcpyAsync(w.d_a, a, sizeof(float) * Sa * D, cudaMemcpyHostToDevice, st));
    d_a = w.d_a;
  }
  if (!b_dev) {
    B2_CUDA(cudaMemcpyAsync(w.d_b, b, sizeof(float) * Sb * D, cudaMemcpyHostToDevice, st));
    d_b = w.d_b;
  }
  int* d_sa = w.d_int;
  int* d_sb = w.d_int + N + 1;
  B2_CUDA(cudaMemcpyAsync(d_sa, seg_a, sizeof(int) * (N + 1), cudaMemcpyHostToDevice, st));
  B2_CUDA(cudaMemcpyAsync(d_sb, seg_b, sizeof(int) * (M + 1), cudaMemcpyHostToDevice, st));
  if (gate) B2_CUDA(cudaMemcpyAsync(w.d_gate, gate, static_cast<size_t>(N) * M, cudaMemcpyHostToDevice, st));
  if (rows_to_planes(d_a, Sa, D, w.a_hi, w.a_lo, Dp, w.d_na2, w.d_range, st) ||
      rows_to_planes(d_b, Sb, D, w.b_hi, w.b_lo, Dp, w.d_nb2, w.d_range, st))
    return -1;
  if (w.gemm(Sp, Np, Dp, split)) return -1;
  if (pair_segmin(w.d_dots, Np, w.d_na2, w.d_nb2, d_sa, N, d_sb, M, gate ? w.d_gate : nullptr, fill, w.d_out, st)) return -1;
  return w.download(out, static_cast<size_t>(N) * M, a_dev ? "b2_track_pair_cost_dev" : "b2_track_pair_cost");
}

int b2_track_pair_cost(int device, const float* a, const int32_t* seg_a, int N, const float* b, const int32_t* seg_b,
                       int M, int D, const uint8_t* gate, float fill, int precision, float* out) {
  return pair_cost_impl(device, a, false, seg_a, N, b, false, seg_b, M, D, gate, fill, precision, out);
}

int b2_track_pair_cost_dev(int device, const float* a_dev, const int32_t* seg_a, int N, const float* b_dev,
                           const int32_t* seg_b, int M, int D, const uint8_t* gate, float fill, int precision, float* out) {
  return pair_cost_impl(device, a_dev, true, seg_a, N, b_dev, true, seg_b, M, D, gate, fill, precision, out);
}

// ---- galleries in device memory that other processes of the node can map (one process per GPU, SURVEY 8e) ----
int b2_gallery_create(int device, const float* feats_host, int rows, int D, float** dev_out, uint8_t handle_out[64]) {
  B2_CHECK(dev_out && handle_out && rows >= 0 && D > 0 && (rows == 0 || feats_host), "b2_gallery_create: bad argument");
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t is 64 bytes");
  *dev_out = nullptr;
  B2_CUDA(cudaSetDevice(device));
  float* p = nullptr;
  B2_CUDA(cudaMalloc(&p, std::max<size_t>(static_cast<size_t>(rows) * D, 1) * sizeof(float)));
  cudaError_t e = rows ? cudaMemcpy(p, feats_host, static_cast<size_t>(rows) * D * sizeof(float), cudaMemcpyHostToDevice)
                       : cudaSuccess;
  cudaIpcMemHandle_t h;
  if (e == cudaSuccess) e = cudaIpcGetMemHandle(&h, p);
  if (e != cudaSuccess) {
    cudaFree(p);
    B2_CUDA(e);
  }
  memcpy(handle_out, &h, 64);
  *dev_out = p;
  return 0;
}

int b2_gallery_open(int device, const uint8_t handle[64], float** peer_out) {
  B2_CHECK(handle && peer_out, "b2_gallery_open: null argument");
  *peer_out = nullptr;
  B2_CUDA(cudaSetDevice(device));
  cudaIpcMemHandle_t h;
  memcpy(&h, handle, 64);
  void* p = nullptr;
  B2_CUDA(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));   // enables P2P (NVLink) access to the owner GPU
  *peer_out = static_cast<float*>(p);
  return 0;
}

int b2_gallery_close(int device, float* peer) {
  if (!peer) return 0;
  B2_CUDA(cudaSetDevice(device));
  B2_CUDA(cudaIpcCloseMemHandle(peer));
  return 0;
}

int b2_gallery_free(int device, float* dev) {
  if (!dev) return 0;
  B2_CUDA(cudaSetDevice(device));
  B2_CUDA(cudaFree(dev));
  return 0;
}

// multi_video_reid.py:260-305 compute_spatial_dist: trajectories as (frame, x, y) rows grouped per track; for every
// track pair the mean point distance over the frames both tracks have (camera-2 frames shifted by frame_offset), kept
// if <= tol, else 9999.  A frame that occurs twice in a track keeps its LAST point (dict semantics, :269-275).
int b2_track_spatial_dist(const int32_t* frames1, const double* pts1, const int32_t* seg1, int N, const int32_t* frames2,
                          const double* pts2, const int32_t* seg2, int M, int frame_offset, double tol, double* out) {
  B2_CHECK(N >= 0 && M >= 0, "b2_track_spatial_dist: bad argument");
  if (N == 0 || M == 0) return 0;
  B2_CHECK(frames1 && pts1 && seg1 && frames2 && pts2 && seg2 && out, "b2_track_spatial_dist: null argument");
  std::vector<std::map<int, const double*>> t2(M);
  for (int j = 0; j < M; ++j)
    for (int k = seg2[j]; k < seg2[j + 1]; ++k) t2[j][frames2[k] + frame_offset] = pts2 + 2 * k;
  for (int i = 0; i < N; ++i) {
    std::map<int, const double*> t1;
    for (int k = seg1[i]; k < seg1[i + 1]; ++k) t1[frames1[k]] = pts1 + 2 * k;
    for (int j = 0; j < M; ++j) {
      double sum = 0;
      int cnt = 0;
      for (const auto& kv : t1) {
        auto it = t2[j].find(kv.first);
        if (it == t2[j].end()) continue;
        const double dx = kv.second[0] - it->second[0], dy = kv.second[1] - it->second[1];
        sum += sqrt(dx * dx + dy * dy);
        ++cnt;
      }
      double v = 9999.0;
      if (cnt > 0) {
        const double mean = sum / cnt;
        if (mean <= tol) v = mean;
      }
      out[static_cast<size_t>(i) * M + j] = v;
    }
  }
  return 0;
}

}  // extern "C"
